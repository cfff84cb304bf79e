// Shared host/device descriptors for the convolution launches of the se(3)-TrackNet conv stack.
//
// Every conv on the path (reference se3_tracknet.py:57-78; 7x7 s2 stem, 3x3 s1, 3x3 s2) is
// described the same way: an NHWC activation tensor, a list of filter "taps", each tap a
// displacement in input pixels plus `k_per_tap` contiguous input channels, and a K-major weight
// matrix W[g*Cout + co][tap*k_per_tap + c] with the eval-mode BatchNorm folded in.
//
//  * 3x3:  9 taps (dy,dx) in {-1,0,1}^2, k_per_tap = Cin (channels of one pixel)
//  * stem: 7 taps (one per filter ROW r), k_per_tap = 32 = 8 pixels x 4 channels of the
//          zero-padded NHWC4 input starting at x = 2*ox (7 real filter columns + 1 zero column)
//
// Two wgmma kernels (conv_wgmma.cu) cover the 14 launches' worth of layers:
//  * conv_resident_kernel: Cout = 64 layers (the two stems, the six 64-channel 3x3 convs); the whole weight
//    matrix lives in shared memory; one launch per layer, static tile ranges.
//  * conv_trunk_kernel: the Cout >= 256 layers (convAB1, convAB2.*, {trans,rot}_conv1, {trans,rot}_conv2.*) as ONE
//    launch: a persistent CTA per SM pulls (layer, image, tile) work units from a global counter and per-image
//    completion counters carry the layer-to-layer dependencies, so no SM idles at a layer boundary.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace se3tn {

constexpr int kMaxTaps = 9;
constexpr int kBlockM = 128;          // M tile: two warpgroups x wgmma M = 64
constexpr int kChunkBytes = 128;      // one SWIZZLE_128B row of K: 32 tf32 words / 32 x [bf16 hi, bf16 lo] / 64 bf16

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SELU = 2 };
enum { KIND_S1 = 0, KIND_S2 = 1, KIND_STEM = 2 };            // conv kinds (compile-time unit tables in conv_wgmma.cu)
// The wgmma kernels take their precision as an SE3TN_PREC_* value (include/se3tn.h); the byte layout of each mode's
// activations and weights is defined in storage.cuh.

struct Tap {
    int16_t dy, dx;      // input-pixel displacement of this tap relative to (oy*stride, ox*stride)
};

// geometry of one conv for the FFMA cross-check kernel (conv_direct.cu) -- fp32 NHWC, 4 bytes per channel
struct ConvGeom {
    int Hin, Win, in_cstride, in_coff;
    int Ho, Wo, stride;
    int cin;             // K floats per tap per group
    int cout;            // per group
    int groups;
    int num_taps;
    int n_img;
    Tap taps[kMaxTaps];
    int out_cstride, out_coff;
    int res_cstride, res_coff;
    int act;
};

struct ConvPtrs {
    const float* in;
    const float* w;      // [groups*cout][num_taps*cin]
    const float* bias;   // [groups*cout]
    const float* res;    // nullable, NHWC
    float* out;
};

constexpr int kLayersPerSet = 14;     // stride of the per-set device tables: one row per conv layer
constexpr int kPoolSlices = 8;        // fused average pool: column sums per 16-row slice of the last layer's 11x11 tile

// ---- wgmma kernels ----------------------------------------------------------------------------------------
// One layer as the device sees it.  Channel counts are in CHANNELS; byte strides follow from the precision.
struct LayerDesc {
    CUtensorMap amap[4];   // activation views: S1 one map; S2 four parity views (py*2+px); stem two (even / odd input rows)
    CUtensorMap bmap;      // weights of weight set `single_wid` (multi-set launches take theirs from gbmaps)
    const float* bias;     // [groups*cout] fp32 (single-set)
    uint8_t* out;          // NHWC output buffer (image 0)
    const uint8_t* res;    // residual input (nullable), same storage format as out
    float* pool_part;      // non-null: fused AdaptiveAvgPool2d(1): column sums [image][kPoolSlices][out_c] instead of the activation
    int kind;              // KIND_*
    int chunks;            // 128-byte K chunks per pixel per group (cin * bytes / 128)
    int cin_words;         // 32-bit words of K per tap per group (weight-matrix K offset of a tap = tap * cin_words)
    int in_gstride_words;  // word offset between groups
    int cout;              // per group
    int groups;
    int n_tiles;           // cout / BN
    int tiles_x, tiles_y;  // 11x11 output tiles per image
    int Ho, Wo;
    int act;
    int out_c, out_coff;   // channels per pixel of the output buffer, channel offset of this layer's channel 0
    int res_c;             // channels per pixel of the residual buffer
    int li;                // row of the per-set tables (layer index)
    // SE3TN_PREC_FP8 (a weight set's fp8 block, kFp8BlockFloats: scales, then per-layer mul tables): scale indices of the
    // e4m3 output and residual (-1: not e4m3), plus ch / q_grp_ch when q_grp_ch > 0 (the heads' per-group scales); offset
    // of this layer's mul[co] = s_in * s_w[co] table
    int q_out, q_res, q_grp_ch, fp8_mul;
    // trunk scheduling
    int unit_base;         // first global work-unit index of this layer (units are K-split pieces when TrunkParams::ksplit > 1)
    int base_unit0;        // index of this layer's first UNSPLIT unit among all unsplit units of the launch (split-K scratch / counters)
    int units_per_image;   // tiles_x * tiles_y * n_tiles * groups (unsplit)
    int dep_layer;         // index (within the launch) of the layer whose per-image completion this layer waits for; -1: none
    unsigned dep_target;   // value done[dep_layer][image] reaches when that image is complete (one signal per warp of the owning consumer warpgroup and K piece: 4 x ksplit x units per image)
};

constexpr int kTrunkMaxLayers = 6;

// A weight set's SE3TN_PREC_FP8 block (floats): the SE3TN_FP8_SCALES activation scales (padded to 16 floats), then per trunk
// layer its mul[co] = s_in(co) * s_w[co], rows 256, 256, 256, 1024, 1024, 1024.  At a fixed device address for the set's life.
constexpr int kFp8MulBase = 16;
constexpr int kFp8TrunkRows[kTrunkMaxLayers] = {256, 256, 256, 1024, 1024, 1024};
constexpr int kFp8BlockFloats = kFp8MulBase + 256 * 3 + 1024 * 3;

struct TrunkParams {
    LayerDesc layer[kTrunkMaxLayers];
    int n_layers;
    int total_units;
    int img_first, n_img;          // absolute image range [img_first, img_first + n_img)
    int max_batch;                 // row length of the done[] table
    unsigned* sched;               // [0] next work unit; then done[layer][image] counters (zeroed before the launch)
    const int* img_wid;            // nullable: weight-set id per absolute image index
    const CUtensorMap* gbmaps;     // per-set weight maps, entry [wid * kLayersPerSet + li]
    const float* const* gbias;     // per-set bias pointers, same indexing
    unsigned long long* trace;     // nullable (SE3TN_TRACE)
    // latency mode (a handful of tracks): every unit's K loop is cut into `ksplit` pieces run by different CTAs (units are dealt
    // round robin so that they are); each piece dumps its fp32 accumulator to `partial`, then finishes ITS share of the unit's
    // 32-column blocks: it waits for the other pieces' dumps, sums all pieces in a fixed order and runs the normal epilogue.  1 = off.
    int ksplit;
    float* partial;                // [unsplit unit][piece][4 warp slices][64-row half][32-column block][float4 0..3][lane]
    unsigned* slice_cnt;           // [unsplit unit][4 warp slices] number of pieces that have dumped the slice (zeroed before the launch)
    const float* fp8;              // SE3TN_PREC_FP8: the fp8 block of the single set
    const float* const* gfp8;      // SE3TN_PREC_FP8, multi-set: fp8 block per set id
};

struct ResidentParams {
    LayerDesc L;
    int img_first, n_img;
    int m_tiles;                   // n_img * tiles_x * tiles_y
    int step_x, step_y, off_x, off_y;   // tile origin in A-map coordinates = tile index * step + off (stem: pooled 5x5 blocks)
    const int* img_wid;
    const CUtensorMap* gbmaps;
    const float* const* gbias;
    const float* fp8;              // SE3TN_PREC_FP8 (the layers that write CAT in e4m3): as TrunkParams
    const float* const* gfp8;
    unsigned long long* trace;
    unsigned long long* tile_trace;    // SE3TN_TRACE: this launch's [SE3TN_TRACE_TILES][4] per-tile stamps (include/se3tn.h)
};

cudaError_t launch_conv_resident(const ResidentParams& p, int kind, int prec, int num_sms, bool pdl, cudaStream_t stream);
cudaError_t launch_conv_trunk(const TrunkParams& p, int prec, int num_sms, bool pdl, cudaStream_t stream);
// latency mode: at most kSplitMaxImages images, ksplit = kSplitK pieces, 128-channel units (at most 8 per image and layer)
constexpr int kSplitMaxImages = 4, kSplitK = 4, kSplitMaxUnits = kSplitMaxImages * 8 * kTrunkMaxLayers;
// 32-bit words of scheduler state a trunk launch needs: next-unit counter + done[layers][max_batch] + split-K slice counters
inline size_t trunk_sched_words(int max_batch) { return 1 + static_cast<size_t>(kTrunkMaxLayers) * max_batch + static_cast<size_t>(kSplitMaxUnits) * 4; }
inline size_t trunk_partial_floats() { return static_cast<size_t>(kSplitMaxUnits) * kSplitK * 128 * 128; }

cudaError_t launch_conv_direct(const ConvGeom& g, const ConvPtrs& p, cudaStream_t stream);

}  // namespace se3tn
