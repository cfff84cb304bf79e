// libse3tn: context, per-object weight sets, TMA tensor maps and the launch schedule of the
// se(3)-TrackNet hot path behind the C ABI declared in include/se3tn.h.
#include "../../include/se3tn.h"
#include "conv_common.h"
#include "aux_kernels.h"
#include "augment.h"
#include "metrics.h"
#include "overlay.h"
#include "render.h"
#include <dlfcn.h>
#include "depth_fill.h"
#include "fit.h"
#include "icp.h"
#include "hypotheses.h"
#include "init.h"
#include "reinit.h"
#include "storage.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

using namespace se3tn;

namespace {

// --------------------------------------------------------------------------------------------
// Network schedule: 14 conv layers cover the reference's 17 convs (se3_tracknet.py:57-78): the two heads' first convs
// are one layer with concatenated output channels, their basic blocks one grouped layer each.  Layers 0-7 are one
// conv_resident_kernel launch each; layers 8-13 are ONE conv_trunk_kernel launch.
// --------------------------------------------------------------------------------------------
enum Buf { B_X0A, B_X0B, B_Y1A, B_Y1B, B_P1A, B_P1B, B_T1, B_T2, B_U, B_CAT, B_F1, B_T4, B_F2, B_H1, B_H2, B_H3, B_COUNT };

constexpr size_t kBufFloats[B_COUNT] = {
    kStemImgFloats, kStemImgFloats,                 // X0A, X0B  (182 x 184 x 4)
    88 * 88 * 64, 88 * 88 * 64,                     // Y1A, Y1B  (fp32 mode only: the tensor-core stems pool in their epilogue)
    44 * 44 * 64, 44 * 44 * 64,                     // P1A, P1B
    44 * 44 * 64, 44 * 44 * 64, 44 * 44 * 64,       // T1, T2, U
    44 * 44 * 128,                                  // CAT
    22 * 22 * 256, 22 * 22 * 256, 22 * 22 * 256,    // F1, T4, F2
    11 * 11 * 1024, 11 * 11 * 1024, 11 * 11 * 1024  // H1, H2, H3
};

enum Kind { K_STEM, K_S1, K_S2 };

struct LayerSpec {
    Kind kind;
    Buf in, out, res;            // res == B_COUNT: none
    int Hin, Win, in_c;          // input spatial + channels per pixel of the input buffer
    int cin, cout, groups;       // per group
    int out_c, out_coff;         // channels per pixel of the output buffer, channel offset
    int act;
    int block_n;
};

constexpr Buf NONE = B_COUNT;
const LayerSpec kLayers[14] = {
    // kind   in     out    res    Hin  Win  in_c  cin  cout groups out_c coff act       BN
    {K_STEM, B_X0A, B_Y1A, NONE,  182, 184,   4,   32,   64, 1,    64,   0, ACT_SELU,  64},   // convA1
    {K_STEM, B_X0B, B_Y1B, NONE,  182, 184,   4,   32,   64, 1,    64,   0, ACT_SELU,  64},   // convB1
    {K_S1,   B_P1A, B_T1,  NONE,   44,  44,  64,   64,   64, 1,    64,   0, ACT_RELU,  64},   // convA2.conv1
    {K_S1,   B_T1,  B_CAT, B_P1A,  44,  44,  64,   64,   64, 1,   128,   0, ACT_RELU,  64},   // convA2.conv2 (+id) -> cat[0:64]
    {K_S1,   B_P1B, B_T2,  NONE,   44,  44,  64,   64,   64, 1,    64,   0, ACT_RELU,  64},   // convB2.conv1
    {K_S1,   B_T2,  B_U,   B_P1B,  44,  44,  64,   64,   64, 1,    64,   0, ACT_RELU,  64},   // convB2.conv2 (+id)
    {K_S1,   B_U,   B_T2,  NONE,   44,  44,  64,   64,   64, 1,    64,   0, ACT_RELU,  64},   // convB3.conv1
    {K_S1,   B_T2,  B_CAT, B_U,    44,  44,  64,   64,   64, 1,   128,  64, ACT_RELU,  64},   // convB3.conv2 (+id) -> cat[64:128]
    {K_S2,   B_CAT, B_F1,  NONE,   44,  44, 128,  128,  256, 1,   256,   0, ACT_SELU, 128},   // convAB1
    {K_S1,   B_F1,  B_T4,  NONE,   22,  22, 256,  256,  256, 1,   256,   0, ACT_RELU, 128},   // convAB2.conv1
    {K_S1,   B_T4,  B_F2,  B_F1,   22,  22, 256,  256,  256, 1,   256,   0, ACT_RELU, 128},   // convAB2.conv2 (+id) = 'feature'
    {K_S2,   B_F2,  B_H1,  NONE,   22,  22, 256,  256, 1024, 1,  1024,   0, ACT_SELU, 128},   // trans_conv1 ++ rot_conv1
    {K_S1,   B_H1,  B_H2,  NONE,   11,  11, 1024, 512,  512, 2,  1024,   0, ACT_RELU, 128},   // {trans,rot}_conv2.conv1
    {K_S1,   B_H2,  B_H3,  B_H1,   11,  11, 1024, 512,  512, 2,  1024,   0, ACT_RELU, 128},   // {trans,rot}_conv2.conv2 (+id)
};
constexpr int kFirstTrunkLayer = 8;

inline int layer_taps(const LayerSpec& L) { return L.kind == K_STEM ? 7 : 9; }
inline int layer_ktot(const LayerSpec& L) { return layer_taps(L) * L.cin; }
inline int layer_rows(const LayerSpec& L) { return L.cout * L.groups; }
inline int layer_Ho(const LayerSpec& L) { return L.kind == K_STEM ? 88 : (L.kind == K_S2 ? L.Hin / 2 : L.Hin); }
inline int res_channels(const LayerSpec& L) { return L.res == B_H1 ? 1024 : (L.res == B_F1 ? 256 : 64); }

constexpr size_t kFcFloats = 6 * 512 + 6;

size_t blob_floats() {
    size_t n = 0;
    for (const LayerSpec& L : kLayers) n += static_cast<size_t>(layer_rows(L)) * layer_ktot(L) + layer_rows(L);
    return n + kFcFloats;
}

// Per-precision state is indexed by the SE3TN_PREC_* value; the fp32 FFMA mode has no entry of its own there.
constexpr int kNumPrecs = 6;
constexpr int kTensorPrecs[] = {SE3TN_PREC_TF32, SE3TN_PREC_BF16X3, SE3TN_PREC_BF16, SE3TN_PREC_FP16};   // every layer's weights in that format
constexpr int kWgmmaPrecs[] = {SE3TN_PREC_TF32, SE3TN_PREC_BF16X3, SE3TN_PREC_BF16, SE3TN_PREC_FP8, SE3TN_PREC_FP16};   // per-set weight-map tables
constexpr float kFp16Max = 65504.f;   // the largest finite fp16 value (SE3TN_PREC_FP16 saturates there)

// SE3TN_PREC_FP8 scale indices (include/se3tn.h order) of trunk layer l's input, output and residual (-1: none).  H1 and H2
// (indices 4 and 6) have one scale per 512-channel head group: + ch / 512.
constexpr int kFp8In[6] = {0, 1, 2, 3, 4, 6}, kFp8Out[6] = {1, 2, 3, 4, 6, -1}, kFp8Res[6] = {-1, -1, 1, -1, -1, 4};
constexpr int kFp8HeadCh = 512;
inline bool fp8_in_grouped(int l) { return kFp8In[l] >= 4; }
inline bool fp8_out_grouped(int l) { return l >= 3; }          // H1, H2, and the last layer's residual H1
inline int fp8_mul_off(int l) { int o = kFp8MulBase; for (int i = 0; i < l; ++i) o += kFp8TrunkRows[i]; return o; }
constexpr int kFp8WRows = 256 * 3 + 1024 * 3;                   // trunk weight rows: one s_w each

// 2^ceil(log2(amax / 448)), 1 for amax == 0 (aux_kernels.cu pow2_scale_dev, exactly)
float pow2_scale(double amax) {
    if (!(amax > 0.0)) return 1.f;
    int ex;
    const double m = std::frexp(amax, &ex);
    return std::ldexp(1.f, ex - 9 + (m > 0.875 ? 1 : 0));
}
bool is_pow2_scale(float s) {
    if (!(std::isfinite(s) && s > 0.f) || !std::isnormal(s)) return false;
    int ex;
    return std::frexp(s, &ex) == 0.5f;
}

// Owned CUDA resources, released with their owner (every entry point makes the context's device current first).
struct CudaRelease {
    void operator()(void* p) const { cudaFree(p); }                  // device memory
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
    void operator()(cudaGraphExec_t g) const { cudaGraphExecDestroy(g); }
};
struct CudaFreeHost { void operator()(uint8_t* p) const { cudaFreeHost(p); } };   // pinned host memory
template <typename T> using DevBuf = std::unique_ptr<T[], CudaRelease>;
using PinBuf = std::unique_ptr<uint8_t[], CudaFreeHost>;
template <typename H> using Handle = std::unique_ptr<std::remove_pointer_t<H>, CudaRelease>;

template <typename T> cudaError_t dev_alloc(DevBuf<T>& b, size_t n) {
    void* p = nullptr;
    const cudaError_t e = cudaMalloc(&p, n * sizeof(T));
    if (e == cudaSuccess) b.reset(static_cast<T*>(p));
    return e;
}

// Makes b hold at least n elements (a PinBuf holds bytes).  A larger buffer replaces b, and cap (how many b holds) changes,
// only once it exists; the caller makes sure no queued work still uses the old buffer.
template <typename B, typename N> cudaError_t grow(B& b, N& cap, N n) {
    if (n <= cap) return cudaSuccess;
    cudaError_t e;
    if constexpr (std::is_same_v<B, PinBuf>) {
        void* p = nullptr;
        if ((e = cudaHostAlloc(&p, n, cudaHostAllocDefault)) == cudaSuccess) b.reset(static_cast<uint8_t*>(p));
    } else e = dev_alloc(b, n);
    if (e == cudaSuccess) cap = n;
    return e;
}

inline size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// Every form of one weight set that the kernels read.
struct DeviceWeights {
    DevBuf<float> blob;             // exact fp32 blob (biases, fc and the fp32 mode's conv weights)
    DevBuf<uint8_t> conv[kNumPrecs];   // tensor-core modes: conv weights in that mode's format (storage.cuh) at w_off * bytes per channel
    DevBuf<uint8_t> stack;          // 8 x [128][288 words]: resident layers with hi / lo rows stacked along N (conv_wgmma.cu STACK)
    DevBuf<float> perm;             // 64-channel layers: rows in the accumulator fragment's channel order, tf32 words
    size_t w_off[14], b_off[14];
    size_t fc_off;
    CUtensorMap bmap[kNumPrecs][kLayersPerSet];   // the weight map the kernel of each layer wants, per precision
    DevBuf<float> fp8;              // SE3TN_PREC_FP8 block (conv_common.h kFp8BlockFloats): activation scales, mul tables
    DevBuf<float> fp8_sw;           // the trunk's per-row weight scales s_w, layer after layer
    std::vector<float> fp8_sw_host;  // the same on the host (the mul tables are formed here)
};

struct WeightSet {
    std::unique_ptr<DeviceWeights> dev;   // null: not loaded
    float mean32[8], std32[8];
    double mean64[8], std64[8];
    int stats_f64 = 0;
    bool has_stats = false;
    float fp8_scales[SE3TN_FP8_SCALES];   // SE3TN_PREC_FP8 activation scales, valid with has_fp8 (dropped by a reload)
    bool has_fp8 = false;
    bool fp16_fits = false;               // every conv weight SE3TN_PREC_FP16 holds in fp16 is within its range (set by a load)
};

// One CAD model of the rasteriser in device memory; view() is the kernels' non-owning MeshDev.
struct Mesh {
    DevBuf<float> pos, nrm; DevBuf<uint8_t> col; DevBuf<int> faces; int nv = 0, nf = 0;
    MeshDev view() const { return {pos.get(), nrm.get(), col.get(), faces.get(), nv, nf}; }
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

std::string g_create_error;

struct F64Bits {   // a double held as its bits: a double member would make StepKey's bytes ambiguous (0.0 == -0.0)
    uint64_t bits = 0;
    F64Bits() = default;
    F64Bits(double d) { memcpy(&bits, &d, sizeof d); }
    operator double() const { double d; memcpy(&d, &bits, sizeof d); return d; }
};

// Everything the kernels of one track or validation step are given that can differ from one call to the next.  Its bytes,
// compared with memcmp, are the key of the step's CUDA graph (run_step), and step_launches takes its arguments from nowhere
// else: an argument missing here could not be read by the launches, so a replayed graph never runs on stale ones.
enum : uint8_t { kStepTrack = 0, kStepEval = 1, kStepPairs = 2 };   // StepKey::kind
// se3tn_eval_pairs_augmented's chain (se3tn_augment as the kernels take it); all zero in every other step
struct AugKey {
    uint64_t seed;
    F64Bits hsv_prob, hsv_noise[3], bright_lo, bright_hi, noise_prob, noise_rgb, noise_depth, blur_prob, cover_prob;
    int32_t stages;                            // bit 0 HSVJitter, 1 ChangeBright, 2 GaussianNoise, 3 GaussianBlur, 4 BlackCover; 0: none
    int32_t blur_half_max;                     // max_kernel_size // 2
    aug::Config config() const {
        aug::Config c{};
        c.seed = seed; c.hsv = stages & 1; c.bright = (stages >> 1) & 1; c.noise = (stages >> 2) & 1; c.blur = (stages >> 3) & 1;
        c.cover = (stages >> 4) & 1; c.blur_half_max = blur_half_max;
        c.hsv_prob = hsv_prob; for (int k = 0; k < 3; ++k) c.hsv_noise[k] = hsv_noise[k];
        c.bright_lo = bright_lo; c.bright_hi = bright_hi; c.noise_prob = noise_prob; c.noise_rgb = noise_rgb; c.noise_depth = noise_depth;
        c.blur_prob = blur_prob; c.cover_prob = cover_prob;
        return c;
    }
};
// A hypothesis step's expansion and choice (se3tn_track_opts.hyp); all zero in every other step.  The step's own tracks (StepKey::n = n x S) are the
// expanded rows in context scratch; these are the caller's n tracks and the call's results.
struct HypKey {
    int32_t S, pad;                            // hypotheses per track (0: not a hypothesis step); pad is always 0
    uint64_t seed;
    F64Bits max_t, max_r;                      // metres, degrees
    const double* poses_in; const int64_t* keys; const int32_t* wid_in; const double* width_in;
    double* poses_out; float* trans_out; float* rot_out; int32_t* choice; int32_t* fit_out;
};
// A render step's depth refinement after the last round (se3tn_track_opts.icp); all zero when ICP is off, so every other
// step's key keeps its bytes.
struct IcpKey {
    int32_t iterations, tau, min_inliers, pad; // iterations 0: no ICP; pad is always 0
    double* poses;                             // icp_poses (M x n x 16) or NULL
    double* stats;                             // out_icp (n x kIcpCols) or NULL
};
struct StepKey {
    uint8_t kind, mixed;                       // kStepTrack, kStepEval (se3tn_eval_pairs) or kStepPairs (se3tn_perturb_pairs); the tracks use more than one weight set
    uint8_t fill, fill_extrapolate;            // track step: its se3tn_track_opts fill, all zero when off (zero in a validation step)
    uint16_t fill_blur, iterations;            // iterations: the track step's rounds, 1 without opts (zero in a validation step)
    int32_t n, precision, first_wid;           // first_wid: the first track's weight set
    int32_t H, W, render_mode, render_H, render_W;   // the frame; input A drawn in the step (SE3TN_RENDER_*, camera size) or -1, 0, 0
    int32_t fit_tau, fit_pad;                  // track step that renders input A: opts->fit_tau_mm (0: no fit check); fit_pad is always 0
    F64Bits K[4], tn, rn, fill_max_depth;
    AugKey aug;                                // validation step: the augmentation of input B (aug.stages 0: none)
    const uint8_t* aug_seg; const int64_t* pair_index; uint8_t* aug_rgb; uint16_t* aug_depth;   // its maskB (NULL: depthB > 100), keys, output
    const uint8_t* frame_rgb; const uint16_t* frame_depth; const double* object_width;   // track step
    const double* poses_in;                    // track step: the previous poses; validation step: A_in_cam
    const double* B_in_cam; const uint8_t* rgbB; const uint16_t* depthB;                 // validation step: inputs; pair step: rgbB / depthB outputs
    const uint8_t* rgbA; const uint16_t* depthA; const int32_t* wid_dev;                  // wid_dev NULL: every track uses set 0 (pair step: mesh ids)
    float* out_trans; float* out_rot; double* poses_out;                                  // poses_out: track step
    float* sq; double* labels; float* sums;                                               // validation step
    const uint8_t* seg; const int32_t* class_ids; uint8_t* segB; int32_t* seg_count;      // pair step
    double* round_poses;                       // track step that renders input A: each round's poses (se3tn_track_render) or NULL
    int32_t* fit_rows;                         // fit_tau > 0: the rows of the fit check, n x kFitCols
    HypKey hyp;                                // track step with opts->hyp
    IcpKey icp;                                // track step with opts->icp
};
static_assert(std::has_unique_object_representations_v<StepKey>, "a graph key is compared byte for byte: no padding, no floating point");

}  // namespace

struct se3tn_ctx {
    int device = 0;
    int max_batch = 0;
    int num_sms = 0;
    uint8_t* workspace = nullptr;    // the caller's, or own_workspace
    DevBuf<uint8_t> own_workspace;   // set only when the library allocated the workspace
    float* buf[B_COUNT] = {};
    CUtensorMap amap4[14][4];        // activation views, 4 bytes per channel (TF32 / BF16X3; also the stems' input in every mode)
    CUtensorMap amap2[14][4];        // activation views, 2 bytes per channel (PREC_BF16 / PREC_FP16, layers 2..13; PREC_FP8, layers 2..7)
    CUtensorMap amap1[14][4];        // activation views, 1 byte per channel (PREC_FP8, trunk layers 8..13)
    DevBuf<float> fp8_scratch;       // se3tn_calibrate_fp8: 8 maxima (as bits), then trans / rot of max_batch pairs (first use)
    int pdl = 1;                     // SE3TN_PDL=0 disables programmatic dependent launch between the kernels of a step
    std::map<int, Mesh> meshes;      // CAD models of the rasteriser, keyed by mesh id
    DevBuf<MeshDev> d_meshes; int mesh_rows = 0; bool meshes_dirty = false;   // device table of their views, rebuilt when a model changes
    DevBuf<uint8_t> render_proj, render_unif; size_t render_proj_bytes = 0; int render_max_nv = 0;   // rasteriser workspace
    DevBuf<uint8_t> in_a; size_t in_a_bytes = 0;   // se3tn_track_render's input A, rgbA | depthA for max_batch tracks (allocated on first use)
    DevBuf<float> loss_sq; size_t loss_sq_floats = 0;   // se3tn_eval_pairs' loss terms when the caller wants none back: max_batch x 6 (allocated on first use)
    // augmented validation steps: the draws (max_batch x SE3TN_AUG_PARAMS doubles), then augmented rgbB | depthB for max_batch
    // pairs (allocated at that size by the first augmented call, never moved after)
    DevBuf<uint8_t> aug; size_t aug_bytes = 0;
    DevBuf<int> pair_bbox; int pair_bbox_ints = 0;     // se3tn_perturb_pairs' crop windows, max_batch x 8 (allocated on first use, never moved)
    DevBuf<unsigned> cover_z; size_t cover_z_words = 0;   // se3tn_visibility's nearest-z planes, rows x H x W (grows on demand; never in a captured step)
    DevBuf<unsigned> append_done; int append_done_words = 0;   // se3tn_append_pairs' CTA counter, zero between launches (allocated on first use)
    DevBuf<uint8_t> metrics; size_t metrics_bytes = 0;   // se3tn_add_adi_sets' staged offsets and ids, or se3tn_vocap_sets' scratch (grows on demand)
    DevBuf<uint8_t> fill; size_t fill_bytes = 0;   // depth hole-filling scratch a | b | lut | minmax in one block, then the filled frame of a track step that fills, so all exist or none (grows on demand)
    // the fit check's block: the device route's rows (max_batch x kFitCols int32), then the fit's rendered depth for max_batch
    // tracks; allocated by the first step with the check on, never moved after (captured steps hold both addresses)
    DevBuf<uint8_t> fit; size_t fit_bytes = 0;
    // a hypothesis step's expanded tracks: poses (max_batch x 16), widths, ids, network outputs (max_batch x 3 each); allocated
    // by the first hypothesis step, never moved after
    DevBuf<uint8_t> hyp; size_t hyp_bytes = 0;
    // the ICP block: the sums (max_batch x kIcpSums doubles), then the ICP render's depth and triangle ids of
    // max_batch tracks; allocated by the first ICP step, never moved after
    DevBuf<uint8_t> icp; size_t icp_bytes = 0;
    // se3tn_init_poses' scratch (InitLayout); grows on demand after a stream synchronisation, never captured in a graph
    DevBuf<uint8_t> init; size_t init_bytes = 0;
    // se3tn_fit_poses' rendered depth (n x 176 x 176 uint16); grows on demand after a stream synchronisation, never captured
    DevBuf<uint8_t> fit_poses; size_t fit_poses_bytes = 0;
    DevBuf<float> pool_part;        // [max_batch][kPoolSlices][1024] column sums from the last conv's epilogue
    DevBuf<unsigned> sched;          // trunk kernel: next-unit counter + done[6][max_batch] + split-K slice counters; zero between steps (head_pooled_kernel clears it)
    DevBuf<float> partial;           // split-K scratch of the latency mode (n <= 4): trunk_partial_floats()
    bool sched_dirty = false;        // a step failed between the trunk launch and the head launch: clear before the next one
    DevBuf<unsigned long long> trace;   // SE3TN_TRACE=1: [14 slots][256 CTAs][8] globaltimer stamps of the last forward (conv_wgmma.cu trace_stamp)
    EncodeTiledFn encode = nullptr;
    std::map<int, WeightSet> weights;
    // device copies of per-set stats, rebuilt when a set changes: [max_id+1][8]
    DevBuf<float> d_mean32, d_std32; DevBuf<double> d_mean64, d_std64;
    int stats_rows = 0; bool stats_dirty = true; int stats_f64 = 0;
    // per-weight-set device tables for multi-set launches, rebuilt when a set is (re)loaded: entry [wid*14 + layer]
    DevBuf<CUtensorMap> d_bmaps[kNumPrecs];   // per tensor-core precision
    DevBuf<const float*> d_bias, d_fc;        // d_fc[wid] -> [6][512] weights then [6] biases
    DevBuf<const float*> d_fp8;               // d_fp8[wid] -> the set's SE3TN_PREC_FP8 block
    int table_rows = 0; bool tables_dirty = true;
    int launches = 0;
    bool profiling = false;
    // CUDA graphs of whole steps (step_launches), keyed by their StepKey.  Besides the key, a step's launches read only context
    // state whose every change drops these graphs (or that is fixed for the context's life: workspace, scheduler, activation
    // tensor maps): the weight sets and their device tables (se3tn_load_weights), the statistics (se3tn_set_stats), the meshes
    // and rasteriser workspace (se3tn_set_mesh), the depth-fill block (reserve_fill) and the host-IO buffers (track_host_step).
    // The fit check's block never moves once allocated (render_into_scratch).
    int use_graphs = 1;              // SE3TN_GRAPH=0: plain stream launches; set to 0 at run time if capture is not possible
    bool last_was_graph = false;
    struct StepGraph { StepKey key; Handle<cudaGraphExec_t> exec; int launches; unsigned long long last_use; };
    std::vector<StepGraph> graphs; unsigned long long graph_clock = 0;
    Handle<cudaStream_t> cap_stream;   // steps are captured on this private stream (the caller's may be the legacy default stream, which cannot be captured) and replayed on the caller's
    Handle<cudaEvent_t> ev[2][SE3TN_PROFILE_SLOTS];   // start, end of each profiling slot
    bool ev_used[SE3TN_PROFILE_SLOTS] = {};
    // se3tn_track_host: context-owned pinned staging and device-side inputs / outputs (stable addresses -> the step's graph is reused)
    struct HostIO {
        PinBuf pin; size_t pin_bytes = 0;                      // pinned host staging: inputs, then outputs
        DevBuf<uint8_t> dev; size_t dev_bytes = 0;             // device: frame rgb | frame depth | poses | widths | rgbA | depthA | ids | out poses | out trans | out rot
        int H = 0, W = 0, n_cap = 0;
    } hio;
    std::string err;
};

namespace {

int fail(se3tn_ctx* c, int code, const std::string& msg) {
    if (c) c->err = msg; else g_create_error = msg;
    return code;
}
#define CU_TRY(ctx, expr)                                                                        \
    do { cudaError_t e_ = (expr);                                                                \
         if (e_ != cudaSuccess) return fail((ctx), SE3TN_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); } while (0)

// Every entry point works on the context's device and leaves the caller's current device as it found it.
struct DeviceGuard {
    int prev = -1, dev;
    explicit DeviceGuard(int d) : dev(d) { if (cudaGetDevice(&prev) != cudaSuccess) prev = -1; if (prev != dev) cudaSetDevice(dev); }
    ~DeviceGuard() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
};

struct ProfScope {
    se3tn_ctx* c; int slot; cudaStream_t s;
    ProfScope(se3tn_ctx* c_, int slot_, cudaStream_t s_) : c(c_), slot(slot_), s(s_) {
        if (c->profiling) { cudaEventRecord(c->ev[0][slot].get(), s); }
    }
    ~ProfScope() { if (c->profiling) { cudaEventRecord(c->ev[1][slot].get(), s); c->ev_used[slot] = true; } }
};

size_t workspace_floats(int max_batch) {
    size_t n = 0;
    for (int b = 0; b < B_COUNT; ++b) {
        size_t f = kBufFloats[b] * static_cast<size_t>(max_batch);
        n += (f + 255) & ~size_t(255);           // keep every buffer 1 KB aligned
    }
    return n;
}

// rank-4 tensor map over 32-bit words, SWIZZLE_128B, box inner = 32 words
int make_map4(se3tn_ctx* c, CUtensorMap* m, const void* base, const cuuint64_t dims[4], const cuuint64_t strides_bytes[3],
              const cuuint32_t box[4], CUtensorMapL2promotion l2, const char* what) {
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = c->encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), dims, strides_bytes, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, l2, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char msg[512];
        snprintf(msg, sizeof msg, "cuTensorMapEncodeTiled(%s) failed: CUresult %d dims {%llu,%llu,%llu,%llu} strides {%llu,%llu,%llu} box {%u,%u,%u,%u}",
                 what, (int)r, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3],
                 (unsigned long long)strides_bytes[0], (unsigned long long)strides_bytes[1], (unsigned long long)strides_bytes[2],
                 box[0], box[1], box[2], box[3]);
        return fail(c, SE3TN_ERR_CUDA, msg);
    }
    return SE3TN_OK;
}

// weight matrix [rows][inner words] -> boxes of 32 words x box_rows
int make_map2(se3tn_ctx* c, CUtensorMap* m, const void* base, cuuint64_t inner, cuuint64_t rows, cuuint32_t box_rows, const char* what) {
    const cuuint64_t dims[2] = {inner, rows};
    const cuuint64_t strides[1] = {inner * sizeof(float)};
    const cuuint32_t box[2] = {32, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUresult r = c->encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char msg[256];
        snprintf(msg, sizeof msg, "cuTensorMapEncodeTiled(%s) failed: CUresult %d dims {%llu,%llu} box {32,%u}", what, (int)r,
                 (unsigned long long)inner, (unsigned long long)rows, box_rows);
        return fail(c, SE3TN_ERR_CUDA, msg);
    }
    return SE3TN_OK;
}

// Activation-side tensor maps: built once per context (they depend only on the workspace layout).  Boxes are extended
// by the vertical filter extent so the vertical taps become descriptor row shifts inside one shared-memory tile
// (conv_wgmma.cu).  bpc = bytes per channel of the storage format (stems: always their 16-byte-per-pixel input).
int build_activation_maps(se3tn_ctx* c, int bpc, CUtensorMap (*out)[4]) {
    const cuuint64_t N = static_cast<cuuint64_t>(c->max_batch);
    for (int li = 0; li < 14; ++li) {
        const LayerSpec& L = kLayers[li];
        const uint8_t* base = reinterpret_cast<const uint8_t*>(c->buf[L.in]);
        char what[64];
        if (bpc == 1 && li < kFirstTrunkLayer) continue;   // e4m3 activations: the trunk's inputs only
        if (L.kind == K_STEM) {
            if (bpc != 4) continue;
            // even / odd input-row views of the zero-padded NHWC4 stem input; x is the overlapping
            // 8-pixel window view (stride 2 pixels = 32 B, extent 128 B)
            const cuuint64_t rowpitch = static_cast<cuuint64_t>(kStemW) * 4 * sizeof(float);
            const cuuint64_t strides[3] = {8 * sizeof(float), 2 * rowpitch, static_cast<cuuint64_t>(kStemH) * rowpitch};
            for (int odd = 0; odd < 2; ++odd) {
                const cuuint64_t dims[4] = {32, 88, odd ? 90u : 91u, N};
                const cuuint32_t box[4] = {32, 11, odd ? 13u : 14u, 1};
                snprintf(what, sizeof what, "layer %d stem %s rows", li, odd ? "odd" : "even");
                int rc = make_map4(c, &out[li][odd], base + odd * rowpitch, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, what);
                if (rc) return rc;
            }
        } else if (L.kind == K_S1) {
            const cuuint64_t Cb = static_cast<cuuint64_t>(L.in_c) * bpc, W = L.Win, H = L.Hin;
            const cuuint64_t dims[4] = {Cb / 4, W, H, N};
            const cuuint64_t strides[3] = {Cb, W * Cb, H * W * Cb};
            const cuuint32_t box[4] = {32, 11, 13, 1};
            snprintf(what, sizeof what, "layer %d s1 (%d B/ch)", li, bpc);
            int rc = make_map4(c, &out[li][0], base, dims, strides, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, what);
            if (rc) return rc;
        } else {
            // stride 2: four parity views (py, px) of the input, each a dense half-resolution tensor
            const cuuint64_t Cb = static_cast<cuuint64_t>(L.in_c) * bpc, W = L.Win, H = L.Hin;
            const cuuint64_t dims[4] = {Cb / 4, W / 2, H / 2, N};
            const cuuint64_t strides[3] = {2 * Cb, 2 * W * Cb, H * W * Cb};
            for (int py = 0; py < 2; ++py)
                for (int px = 0; px < 2; ++px) {
                    const cuuint32_t box[4] = {32, 11, py ? 12u : 11u, 1};
                    snprintf(what, sizeof what, "layer %d s2 parity %d%d (%d B/ch)", li, py, px, bpc);
                    int rc = make_map4(c, &out[li][py * 2 + px], base + (static_cast<size_t>(py) * W + px) * Cb, dims, strides, box,
                                       CU_TENSOR_MAP_L2_PROMOTION_L2_128B, what);
                    if (rc) return rc;
                }
        }
    }
    return SE3TN_OK;
}

// geometry of one conv for the fp32 FFMA kernel
void fill_geom(const LayerSpec& L, int n, ConvGeom& g) {
    memset(&g, 0, sizeof g);
    g.Hin = L.Hin; g.Win = L.Win; g.in_cstride = L.in_c; g.in_coff = 0;
    g.Ho = layer_Ho(L); g.Wo = g.Ho;
    g.stride = (L.kind == K_S1) ? 1 : 2;
    g.cin = L.cin; g.cout = L.cout; g.groups = L.groups;
    g.num_taps = layer_taps(L);
    g.n_img = n;
    if (L.kind == K_STEM) {
        // tap r: padded input row 2*oy + r, 32 contiguous floats from padded x = 2*ox
        for (int r = 0; r < 7; ++r) { g.taps[r].dy = (int16_t)r; g.taps[r].dx = 0; }
    } else {
        for (int r = 0; r < 3; ++r)
            for (int s = 0; s < 3; ++s) { g.taps[r * 3 + s].dy = (int16_t)(r - 1); g.taps[r * 3 + s].dx = (int16_t)(s - 1); }
    }
    g.out_cstride = L.out_c; g.out_coff = L.out_coff;
    g.res_cstride = (L.res != NONE) ? res_channels(L) : 0;
    g.res_coff = 0;
    g.act = L.act;
}

// one layer as the wgmma kernels see it (conv_common.h LayerDesc)
void fill_layer_desc(const se3tn_ctx* c, const DeviceWeights& w, int li, int precision, LayerDesc& d) {
    const LayerSpec& L = kLayers[li];
    const int row = li;                            // row of the per-set tables
    memset(&d, 0, sizeof d);
    const bool stem = (L.kind == K_STEM);
    const int bpc = prec_bytes_per_channel(layer_input_prec(li, precision));   // of this layer's input
    const CUtensorMap (*amaps)[4] = bpc == 1 ? c->amap1 : (bpc == 2 ? c->amap2 : c->amap4);
    for (int m = 0; m < 4; ++m) d.amap[m] = amaps[li][m];
    d.bmap = w.bmap[precision][row];
    d.bias = w.blob.get() + w.b_off[li];
    d.kind = stem ? KIND_STEM : (L.kind == K_S2 ? KIND_S2 : KIND_S1);
    d.chunks = L.cin * bpc / kChunkBytes; d.cin_words = L.cin * bpc / 4; d.in_gstride_words = d.cin_words;
    if (stem) {
        d.out = reinterpret_cast<uint8_t*>(c->buf[li == 0 ? B_P1A : B_P1B]);   // fused MaxPool2d(3,2,1): the pooled tensor is written directly
        d.out_c = 64; d.out_coff = 0; d.Ho = d.Wo = 44;
        d.tiles_x = d.tiles_y = 9;                 // pooled 5x5 blocks
    } else {
        d.out = reinterpret_cast<uint8_t*>(c->buf[L.out]);
        d.out_c = L.out_c; d.out_coff = L.out_coff; d.Ho = d.Wo = layer_Ho(L);
        d.tiles_x = d.tiles_y = d.Ho / 11;
    }
    d.res = (L.res != NONE) ? reinterpret_cast<const uint8_t*>(c->buf[L.res]) : nullptr;
    d.res_c = (L.res != NONE) ? res_channels(L) : 0;
    d.cout = L.cout; d.groups = L.groups; d.n_tiles = L.cout / L.block_n;
    d.act = L.act; d.li = row;
    d.units_per_image = d.tiles_x * d.tiles_y * d.n_tiles * d.groups;
    d.dep_layer = -1; d.dep_target = 0; d.unit_base = 0;
    d.q_out = d.q_res = -1; d.q_grp_ch = 0; d.fp8_mul = 0;
    if (precision == SE3TN_PREC_FP8) {
        if (li >= kFirstTrunkLayer) {
            const int l = li - kFirstTrunkLayer;
            d.q_out = kFp8Out[l]; d.q_res = kFp8Res[l]; d.q_grp_ch = fp8_out_grouped(l) ? kFp8HeadCh : 0; d.fp8_mul = fp8_mul_off(l);
        } else if (L.out == B_CAT) {
            d.q_out = 0;                           // the two layers that write CAT encode it to e4m3 themselves
        }
    }
}

int sync_stats(se3tn_ctx* c, cudaStream_t s) {
    if (!c->stats_dirty) return SE3TN_OK;
    int max_id = -1, f64 = -1;
    for (auto& kv : c->weights) if (kv.second.has_stats) {
        if (kv.first > max_id) max_id = kv.first;
        if (f64 < 0) f64 = kv.second.stats_f64;
        else if (f64 != kv.second.stats_f64) return fail(c, SE3TN_ERR_STATE, "all weight sets must use the same mean/std dtype");
    }
    if (max_id < 0) return fail(c, SE3TN_ERR_STATE, "se3tn_set_stats has not been called");
    const int rows = max_id + 1;
    if (rows > c->stats_rows) {                    // grow: the old tables stay in place until all new ones exist
        DevBuf<float> m32, s32; DevBuf<double> m64, s64;
        CU_TRY(c, dev_alloc(m32, rows * 8)); CU_TRY(c, dev_alloc(s32, rows * 8));
        CU_TRY(c, dev_alloc(m64, rows * 8)); CU_TRY(c, dev_alloc(s64, rows * 8));
        c->d_mean32 = std::move(m32); c->d_std32 = std::move(s32); c->d_mean64 = std::move(m64); c->d_std64 = std::move(s64);
        c->stats_rows = rows;
    }
    std::vector<float> m32(rows * 8, 0.f), s32(rows * 8, 1.f);
    std::vector<double> m64(rows * 8, 0.0), s64(rows * 8, 1.0);
    for (auto& kv : c->weights) if (kv.second.has_stats && kv.first >= 0) {
        memcpy(&m32[kv.first * 8], kv.second.mean32, sizeof(float) * 8); memcpy(&s32[kv.first * 8], kv.second.std32, sizeof(float) * 8);
        memcpy(&m64[kv.first * 8], kv.second.mean64, sizeof(double) * 8); memcpy(&s64[kv.first * 8], kv.second.std64, sizeof(double) * 8);
    }
    // synchronous copies from stack-lifetime host vectors (rare: only when stats change)
    CU_TRY(c, cudaStreamSynchronize(s));
    CU_TRY(c, cudaMemcpy(c->d_mean32.get(), m32.data(), rows * 8 * sizeof(float), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(c->d_std32.get(), s32.data(), rows * 8 * sizeof(float), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(c->d_mean64.get(), m64.data(), rows * 8 * sizeof(double), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(c->d_std64.get(), s64.data(), rows * 8 * sizeof(double), cudaMemcpyHostToDevice));
    c->stats_f64 = f64; c->stats_dirty = false;
    return SE3TN_OK;
}

int sync_tables(se3tn_ctx* c, cudaStream_t s) {
    if (!c->tables_dirty) return SE3TN_OK;
    int max_id = -1;
    for (auto& kv : c->weights) if (kv.second.dev && kv.first > max_id) max_id = kv.first;
    if (max_id < 0) return fail(c, SE3TN_ERR_STATE, "no weight set loaded");
    const int rows = max_id + 1;
    CU_TRY(c, cudaStreamSynchronize(s));
    if (rows > c->table_rows) {                    // grow: the old tables stay in place until all new ones exist
        DevBuf<CUtensorMap> maps[kNumPrecs]; DevBuf<const float*> bias, fc, fp8;
        for (int p : kWgmmaPrecs) CU_TRY(c, dev_alloc(maps[p], rows * kLayersPerSet));
        CU_TRY(c, dev_alloc(bias, rows * kLayersPerSet));
        CU_TRY(c, dev_alloc(fc, rows));
        CU_TRY(c, dev_alloc(fp8, rows));
        for (int p : kWgmmaPrecs) c->d_bmaps[p] = std::move(maps[p]);
        c->d_bias = std::move(bias); c->d_fc = std::move(fc); c->d_fp8 = std::move(fp8);
        c->table_rows = rows;
    }
    const size_t entries = static_cast<size_t>(rows) * kLayersPerSet;
    std::vector<CUtensorMap> maps(kNumPrecs * entries);    // [precision][entry], zeroed for ids without weights
    std::vector<const float*> bias(entries, nullptr), fc(rows, nullptr), fp8(rows, nullptr);
    for (auto& kv : c->weights) {
        if (!kv.second.dev || kv.first < 0) continue;
        const DeviceWeights& w = *kv.second.dev;
        for (int li = 0; li < kLayersPerSet; ++li) {
            const size_t e = static_cast<size_t>(kv.first) * kLayersPerSet + li;
            for (int p : kWgmmaPrecs) maps[p * entries + e] = w.bmap[p][li];
            bias[e] = w.blob.get() + w.b_off[li];
        }
        fc[kv.first] = w.blob.get() + w.fc_off;
        fp8[kv.first] = w.fp8.get();
    }
    for (int p : kWgmmaPrecs)
        CU_TRY(c, cudaMemcpy(c->d_bmaps[p].get(), &maps[p * entries], entries * sizeof(CUtensorMap), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(c->d_bias.get(), bias.data(), bias.size() * sizeof(float*), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(c->d_fc.get(), fc.data(), fc.size() * sizeof(float*), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(c->d_fp8.get(), fp8.data(), fp8.size() * sizeof(float*), cudaMemcpyHostToDevice));
    c->tables_dirty = false;
    return SE3TN_OK;
}

// Rebuilds the device table of mesh views and the rasteriser workspace after se3tn_set_mesh.  Synchronous copies and
// allocations: like sync_stats / sync_tables it runs before a step is captured, never inside the capture.
int sync_meshes(se3tn_ctx* c, cudaStream_t s) {
    if (!c->meshes_dirty) return SE3TN_OK;
    const int rows = c->meshes.rbegin()->first + 1;
    CU_TRY(c, cudaStreamSynchronize(s));
    CU_TRY(c, grow(c->d_meshes, c->mesh_rows, rows));
    std::vector<MeshDev> tab(rows, c->meshes.begin()->second.view());   // unused ids alias the first model
    int max_nv = 0;
    for (auto& kv : c->meshes) { tab[kv.first] = kv.second.view(); max_nv = std::max(max_nv, kv.second.nv); }
    CU_TRY(c, cudaMemcpy(c->d_meshes.get(), tab.data(), sizeof(MeshDev) * rows, cudaMemcpyHostToDevice));
    CU_TRY(c, grow(c->render_proj, c->render_proj_bytes, static_cast<size_t>(c->max_batch) * max_nv * render_projected_bytes_per_vertex()));   // max_batch x largest model
    if (!c->render_unif) CU_TRY(c, dev_alloc(c->render_unif, static_cast<size_t>(c->max_batch) * render_uniform_bytes()));
    c->render_max_nv = max_nv;
    c->meshes_dirty = false;
    return SE3TN_OK;
}

// What the head kernel does besides trans / rot, in the tensor-core modes: the pose update (K6) of the same n tracks and / or
// the loss terms of a validation step.  The fp32 FFMA mode's head does neither; its caller launches them on their own.
struct HeadArgs { const double* pose_in = nullptr; double* pose_out = nullptr; float tn = 0.f, rn = 0.f; LossArgs loss; };

// The conv stack on images [first, first+n) of the context buffers.  img_wid (device, indexed by absolute image
// index) non-null: every image uses its own weight set in the same launches (tensor-core modes; the caller has run
// sync_tables); `weight_id` is then only a representative loaded set.
int run_network(se3tn_ctx* c, int weight_id, int first, int n, int precision,
                float* out_trans, float* out_rot, float* out_feature, cudaStream_t s, const int* img_wid = nullptr,
                const HeadArgs& head = HeadArgs()) {
    auto it = c->weights.find(weight_id);
    if (it == c->weights.end() || !it->second.dev) return fail(c, SE3TN_ERR_STATE, "weight set " + std::to_string(weight_id) + " not loaded");
    const DeviceWeights& w = *it->second.dev;
    if (precision < SE3TN_PREC_TF32 || precision > SE3TN_PREC_FP16) return fail(c, SE3TN_ERR_INVALID, "unknown precision");
    const bool tensor = precision != SE3TN_PREC_FP32;
    auto bufp = [&](Buf b) { return c->buf[b] + kBufFloats[b] * static_cast<size_t>(first); };
    const float* fcw = w.blob.get() + w.fc_off;
    if (!tensor) {
        // ---- fp32 FFMA cross-check mode: 14 direct convs + 2 max-pools + head ----
        if (img_wid) return fail(c, SE3TN_ERR_INVALID, "multi-weight-set launches need a tensor-core precision");
        for (int li = 0; li < 14; ++li) {
            const LayerSpec& L = kLayers[li];
            ConvGeom g; fill_geom(L, n, g);
            ConvPtrs p;
            p.in = bufp(L.in); p.out = bufp(L.out); p.res = (L.res != NONE) ? bufp(L.res) : nullptr;
            p.w = w.blob.get() + w.w_off[li]; p.bias = w.blob.get() + w.b_off[li];
            { ProfScope ps(c, li, s); CU_TRY(c, launch_conv_direct(g, p, s)); }
            ++c->launches;
            if (li == 0) { ProfScope ps(c, 14, s); CU_TRY(c, launch_maxpool(bufp(B_Y1A), bufp(B_P1A), n, 88, 88, 64, s)); ++c->launches; }
            if (li == 1) { ProfScope ps(c, 15, s); CU_TRY(c, launch_maxpool(bufp(B_Y1B), bufp(B_P1B), n, 88, 88, 64, s)); ++c->launches; }
        }
        { ProfScope ps(c, 16, s); CU_TRY(c, launch_head(bufp(B_H3), fcw, fcw + 6 * 512, out_trans, out_rot, n, 121, s)); }
        ++c->launches;
        if (out_feature) { CU_TRY(c, launch_nhwc_to_nchw(bufp(B_F2), out_feature, n, 22 * 22, 256, precision, s)); ++c->launches; }
        return SE3TN_OK;
    }
    // ---- tensor-core modes: 8 resident-weight launches + 1 trunk launch + head ----
    const CUtensorMap* gbmaps = img_wid ? c->d_bmaps[precision].get() : nullptr;
    const float* const* gbias = img_wid ? c->d_bias.get() : nullptr;
    const bool fp8 = precision == SE3TN_PREC_FP8;
    const float* fp8_block = fp8 ? w.fp8.get() : nullptr;
    const float* const* gfp8 = fp8 && img_wid ? c->d_fp8.get() : nullptr;
    if (c->sched_dirty) { CU_TRY(c, cudaMemsetAsync(c->sched.get(), 0, trunk_sched_words(c->max_batch) * sizeof(unsigned), s)); c->sched_dirty = false; }
    for (int li = 0; li < kFirstTrunkLayer; ++li) {
        ResidentParams rp;
        fill_layer_desc(c, w, li, precision, rp.L);
        rp.img_first = first; rp.n_img = n;
        rp.m_tiles = n * rp.L.tiles_x * rp.L.tiles_y;
        if (kLayers[li].kind == K_STEM) { rp.step_x = rp.step_y = 10; rp.off_x = rp.off_y = -1; }   // 11x11 conv outputs from (10*t - 1): the 5x5 pooled block's window
        else { rp.step_x = rp.step_y = 11; rp.off_x = rp.off_y = 0; }
        rp.img_wid = img_wid; rp.gbmaps = gbmaps; rp.gbias = gbias; rp.fp8 = fp8_block; rp.gfp8 = gfp8;
        // SE3TN_PREC_FP8: the stems and 64-channel layers are the bf16 mode's, but the two that write CAT encode it to e4m3
        const int lp = fp8 && kLayers[li].out != B_CAT ? SE3TN_PREC_BF16 : precision;
        rp.trace = c->trace ? c->trace.get() + static_cast<size_t>(li) * 256 * 8 : nullptr;
        rp.tile_trace = c->trace ? c->trace.get() + 14 * 256 * 8 + static_cast<size_t>(li) * SE3TN_TRACE_TILES * 4 : nullptr;
        { ProfScope ps(c, li, s); CU_TRY(c, launch_conv_resident(rp, rp.L.kind, lp, c->num_sms, c->pdl != 0, s)); }
        ++c->launches;
    }
    {
        TrunkParams tp;
        memset(&tp, 0, sizeof tp);
        // latency mode: a handful of tracks keep only 8 CTAs per layer busy, and the six layers of an image are a serial chain:
        // cut every unit's K loop into kSplitK pieces (conv_trunk_kernel).  Its fp32 sums are grouped differently, so results agree
        // with the throughput mode to rounding, not bit for bit; within the mode (n = 1..4) they do not depend on n.
        int ksplit = (n <= kSplitMaxImages) ? kSplitK : 1;
        for (int l = 0; l < 14 - kFirstTrunkLayer; ++l) {
            fill_layer_desc(c, w, kFirstTrunkLayer + l, precision, tp.layer[l]);
            while (tp.layer[l].chunks % ksplit) ksplit /= 2;       // 2-byte storage: convAB1 has only two 128-byte chunks per pixel,
                                                                   // 1-byte (fp8) one: no latency mode there
        }
        int base = 0, base0 = 0;
        for (int l = 0; l < 14 - kFirstTrunkLayer; ++l) {
            LayerDesc& d = tp.layer[l];
            d.unit_base = base; base += n * d.units_per_image * ksplit;
            d.base_unit0 = base0; base0 += n * d.units_per_image;
            // completion signals per unit: one per warp of the owning consumer warpgroup in every K piece (each piece finishes
            // 4 / ksplit of every warp's 32-column blocks)
            if (l > 0) { d.dep_layer = l - 1; d.dep_target = 4u * static_cast<unsigned>(ksplit) * static_cast<unsigned>(tp.layer[l - 1].units_per_image); }
        }
        if (ksplit > 1 && base0 > kSplitMaxUnits) return fail(c, SE3TN_ERR_STATE, "split-K scratch too small");
        tp.ksplit = ksplit; tp.partial = c->partial.get();
        tp.slice_cnt = c->sched.get() + 1 + static_cast<size_t>(kTrunkMaxLayers) * c->max_batch;
        tp.layer[5].pool_part = c->pool_part.get();   // AdaptiveAvgPool2d(1) fused into the last conv's epilogue (indexed by absolute image)
        tp.n_layers = 6; tp.total_units = base;
        tp.img_first = first; tp.n_img = n; tp.max_batch = c->max_batch;
        tp.sched = c->sched.get(); tp.img_wid = img_wid; tp.gbmaps = gbmaps; tp.gbias = gbias; tp.fp8 = fp8_block; tp.gfp8 = gfp8;
        tp.trace = c->trace ? c->trace.get() + static_cast<size_t>(kFirstTrunkLayer) * 256 * 8 : nullptr;
        c->sched_dirty = true;                     // cleared again by the head kernel below
        { ProfScope ps(c, kFirstTrunkLayer, s); CU_TRY(c, launch_conv_trunk(tp, precision, c->num_sms, c->pdl != 0, s)); }
        ++c->launches;
    }
    {
        ProfScope ps(c, 16, s);
        CU_TRY(c, launch_head_pooled(c->pool_part.get() + static_cast<size_t>(first) * kPoolSlices * 1024, fcw, fcw + 6 * 512, out_trans, out_rot, n, 121,
                                     img_wid ? img_wid + first : nullptr, img_wid ? c->d_fc.get() : nullptr,
                                     head.pose_in, head.pose_out, head.tn, head.rn, head.loss,
                                     c->sched.get(), static_cast<int>(trunk_sched_words(c->max_batch)), s));
        c->sched_dirty = false;
    }
    ++c->launches;
    if (out_feature) { CU_TRY(c, launch_nhwc_to_nchw(reinterpret_cast<const uint8_t*>(c->buf[B_F2]) + static_cast<size_t>(first) * 22 * 22 * 256 * prec_bytes_per_channel(precision), out_feature, n, 22 * 22, 256,
                                                       precision, s, fp8 ? fp8_block + kFp8In[3] : nullptr)); ++c->launches; }   // F2's scale
    return SE3TN_OK;
}

// Launches shared by the public entry points and step_launches.  They check and sync nothing: their callers have checked the
// arguments and brought the statistics / meshes up to date, outside any capture.
// K0: preprocess (a frame and input A) or normalize (ready-made crops), with the context's statistics, into the stem buffers
int queue_preprocess(se3tn_ctx* c, PreprocessArgs a, int n, cudaStream_t s) {
    a.mean32 = c->d_mean32.get(); a.std32 = c->d_std32.get(); a.mean64 = c->d_mean64.get(); a.std64 = c->d_std64.get();
    a.stats_f64 = c->stats_f64; a.stats_rows = c->stats_rows;
    a.stemA = c->buf[B_X0A]; a.stemB = c->buf[B_X0B];
    { ProfScope ps(c, 17, s); CU_TRY(c, launch_preprocess(a, n, s)); }
    ++c->launches;
    return SE3TN_OK;
}

RenderArgs render_args(const se3tn_ctx* c, const double* K, const double* poses, const double* object_width, const int32_t* mesh_ids,
                       int mode, int H, int W, uint8_t* rgbA, uint16_t* depthA) {
    RenderArgs a;
    a.poses = poses; a.object_width = object_width; a.mesh_ids = mesh_ids; a.meshes = c->d_meshes.get(); a.n_meshes = c->mesh_rows;
    a.fx = K[0]; a.fy = K[1]; a.cx = K[2]; a.cy = K[3];
    a.rgb = rgbA; a.depth = depthA;
    a.mode = mode == SE3TN_RENDER_PYRENDER ? 1 : 0; a.vw = W; a.vh = H;
    a.projected = c->render_proj.get(); a.uniforms = c->render_unif.get(); a.max_nv = c->render_max_nv;
    return a;
}

int queue_render(se3tn_ctx* c, const double* K, const double* poses, const double* object_width, const int32_t* mesh_ids, int n,
                 int mode, int H, int W, uint8_t* rgbA, uint16_t* depthA, cudaStream_t s, bool pdl = true) {
    const RenderArgs a = render_args(c, K, poses, object_width, mesh_ids, mode, H, W, rgbA, depthA);
    { ProfScope ps(c, 20, s); CU_TRY(c, launch_render(a, n, s, pdl)); }
    c->launches += 2;
    return SE3TN_OK;
}

constexpr size_t kStackBytes = 8 * 128 * 288 * sizeof(float);   // DeviceWeights::stack
constexpr size_t kPermFloats = 6 * 64 * 576;                     // DeviceWeights::perm

// Device bytes of the DeviceWeights prepare_weights builds: what one loaded weight set holds.
size_t weight_set_bytes() {
    const size_t floats = blob_floats();
    size_t bytes = floats * sizeof(float) + floats;                // the fp32 blob, the fp8 conv weights
    for (int p : kTensorPrecs) bytes += floats * prec_bytes_per_channel(p);
    return bytes + (kFp8BlockFloats + kFp8WRows + kPermFloats) * sizeof(float) + kStackBytes;
}

// Every form of a weight blob the kernels read, built into `w` (which owns all of it, so a failure leaves nothing behind).
// Its allocations are the ones weight_set_bytes counts.
int prepare_weights(se3tn_ctx* c, DeviceWeights& w, const float* blob) {
    const size_t floats = blob_floats();
    CU_TRY(c, dev_alloc(w.blob, floats));
    for (int p : kTensorPrecs) CU_TRY(c, dev_alloc(w.conv[p], floats * prec_bytes_per_channel(p)));
    CU_TRY(c, dev_alloc(w.conv[SE3TN_PREC_FP8], floats));
    CU_TRY(c, dev_alloc(w.fp8, kFp8BlockFloats));
    CU_TRY(c, dev_alloc(w.fp8_sw, kFp8WRows));
    CU_TRY(c, dev_alloc(w.stack, kStackBytes));
    CU_TRY(c, dev_alloc(w.perm, kPermFloats));
    DevBuf<float> perm_tmp;                        // one 64-channel layer's fp32 weights with permuted rows
    CU_TRY(c, dev_alloc(perm_tmp, 64 * 576));
    CU_TRY(c, cudaDeviceSynchronize());
    CU_TRY(c, cudaMemcpy(w.blob.get(), blob, floats * sizeof(float), cudaMemcpyHostToDevice));
    size_t off = 0;
    for (int li = 0; li < 14; ++li) {
        const LayerSpec& L = kLayers[li];
        const int rows = layer_rows(L), ktot = layer_ktot(L);
        w.w_off[li] = off; off += static_cast<size_t>(rows) * ktot;
        w.b_off[li] = off; off += rows;
        const float* wsrc = w.blob.get() + w.w_off[li];
        auto conv_dst = [&](int p) { return w.conv[p].get() + w.w_off[li] * prec_bytes_per_channel(p); };
        char what[64];
        int rc = SE3TN_OK;
        if (li >= kFirstTrunkLayer) {
            // trunk layers: natural row order, tiles of {32 words, block_n rows} streamed through the weight ring
            snprintf(what, sizeof what, "layer %d weights", li);
            for (int p : kTensorPrecs) {
                CU_TRY(c, launch_encode_weights(p, wsrc, conv_dst(p), rows, ktot, 0));
                if (!rc) rc = make_map2(c, &w.bmap[p][li], conv_dst(p), ktot * prec_bytes_per_channel(p) / 4, rows, L.block_n, what);
            }
            // e4m3 with a power-of-two scale per row (SE3TN_PREC_FP8)
            int sw_off = 0;
            for (int l = 0; l < li - kFirstTrunkLayer; ++l) sw_off += kFp8TrunkRows[l];
            CU_TRY(c, launch_encode_weights_fp8(wsrc, conv_dst(SE3TN_PREC_FP8), w.fp8_sw.get() + sw_off, rows, ktot, 0));
            if (!rc) rc = make_map2(c, &w.bmap[SE3TN_PREC_FP8][li], conv_dst(SE3TN_PREC_FP8), ktot / 4, rows, L.block_n, what);
        } else {
            // resident-weight layers.  Stems keep the natural row order; the 64-channel 3x3 layers use the row order of the
            // accumulator fragment (all precisions).  BF16X3: hi / lo rows stacked along N.
            const bool stem = (L.kind == K_STEM);
            void* w_tf32 = conv_dst(SE3TN_PREC_TF32);
            if (!stem) {
                if (ktot != 576 || rows != 64) return fail(c, SE3TN_ERR_STATE, "resident layer shape");
                CU_TRY(c, launch_permute_rows64(wsrc, perm_tmp.get(), 576, 0));
                wsrc = perm_tmp.get(); w_tf32 = w.perm.get() + static_cast<size_t>(li - 2) * 64 * 576;
            }
            snprintf(what, sizeof what, "layer %d resident weights", li);
            CU_TRY(c, launch_encode_weights(SE3TN_PREC_TF32, wsrc, w_tf32, 64, ktot, 0));
            rc = make_map2(c, &w.bmap[SE3TN_PREC_TF32][li], w_tf32, ktot, 64, 64, what);
            uint8_t* sdst = w.stack.get() + static_cast<size_t>(li) * 128 * 288 * sizeof(float);
            CU_TRY(c, launch_split_stack_weights(wsrc, sdst, stem, 0));
            if (!rc) rc = make_map2(c, &w.bmap[SE3TN_PREC_BF16X3][li], sdst, stem ? 224 : 288, 128, 128, what);
            for (int p : {SE3TN_PREC_BF16, SE3TN_PREC_FP16}) {   // the 2-byte formats
                if (stem) w.bmap[p][li] = w.bmap[stem_input_prec(p)][li];   // the stem's input format decides
                else {
                    CU_TRY(c, launch_encode_weights(p, wsrc, conv_dst(p), 64, ktot, 0));   // permuted rows
                    if (!rc) rc = make_map2(c, &w.bmap[p][li], conv_dst(p), 288, 64, 64, what);
                }
            }
            w.bmap[SE3TN_PREC_FP8][li] = w.bmap[resident_prec(SE3TN_PREC_FP8)][li];   // SE3TN_PREC_FP8 runs these as bf16
        }
        if (rc) return rc;
    }
    w.fc_off = off;
    CU_TRY(c, cudaDeviceSynchronize());            // a kernel that failed above fails the load
    w.fp8_sw_host.resize(kFp8WRows);
    CU_TRY(c, cudaMemcpy(w.fp8_sw_host.data(), w.fp8_sw.get(), kFp8WRows * sizeof(float), cudaMemcpyDeviceToHost));
    CU_TRY(c, cudaMemset(w.fp8.get(), 0, kFp8BlockFloats * sizeof(float)));   // no scales yet (WeightSet::has_fp8)
    CU_TRY(c, cudaDeviceSynchronize());
    return SE3TN_OK;
}

// A set's SE3TN_PREC_FP8 block from its activation scales: the scales, and mul[co] = s_in(co) * s_w[co] per trunk layer
// (powers of two: exact).  The block keeps its address, so captured steps read the new values.  The device is synchronised
// first: no queued step reads the block while it changes.
int upload_fp8(se3tn_ctx* c, WeightSet& ws, const float* scales) {
    const DeviceWeights& w = *ws.dev;
    std::vector<float> blk(kFp8BlockFloats, 0.f);
    for (int i = 0; i < SE3TN_FP8_SCALES; ++i) blk[i] = scales[i];
    int sw = 0;
    for (int l = 0; l < kTrunkMaxLayers; ++l) {
        float* mul = blk.data() + fp8_mul_off(l);
        for (int co = 0; co < kFp8TrunkRows[l]; ++co)
            mul[co] = scales[kFp8In[l] + (fp8_in_grouped(l) ? co / kFp8HeadCh : 0)] * w.fp8_sw_host[sw + co];
        sw += kFp8TrunkRows[l];
    }
    CU_TRY(c, cudaDeviceSynchronize());
    CU_TRY(c, cudaMemcpy(w.fp8.get(), blk.data(), blk.size() * sizeof(float), cudaMemcpyHostToDevice));
    memcpy(ws.fp8_scales, scales, sizeof ws.fp8_scales);
    ws.has_fp8 = true;
    return SE3TN_OK;
}

// Whether every conv weight that SE3TN_PREC_FP16 holds in fp16 (layers 2-13; the stems hold bf16x3) is within fp16's range
bool fp16_weights_fit(const float* blob) {
    size_t off = 0;
    for (const LayerSpec& L : kLayers) {
        const size_t nw = static_cast<size_t>(layer_rows(L)) * layer_ktot(L);
        if (L.kind != K_STEM)
            for (size_t i = 0; i < nw; ++i)
                if (std::fabs(blob[off + i]) > kFp16Max) return false;
        off += nw + layer_rows(L);
    }
    return true;
}

// What a step in `precision` needs of every set it uses besides its weights: SE3TN_PREC_FP8 the set's activation scales,
// SE3TN_PREC_FP16 conv weights within fp16's range (a checkpoint's weights are not saturated silently)
int check_prec(se3tn_ctx* c, const char* fn, int wid, int precision) {
    auto it = c->weights.find(wid);
    if (it == c->weights.end() || !it->second.dev) return SE3TN_OK;
    if (precision == SE3TN_PREC_FP8 && !it->second.has_fp8)
        return fail(c, SE3TN_ERR_STATE, std::string(fn) + ": weight set " + std::to_string(wid) +
                                         " has no fp8 activation scales (se3tn_calibrate_fp8 / se3tn_set_fp8_scales)");
    if (precision == SE3TN_PREC_FP16 && !it->second.fp16_fits)
        return fail(c, SE3TN_ERR_STATE, std::string(fn) + ": weight set " + std::to_string(wid) +
                                         " has a conv weight above 65504 in magnitude, outside fp16's range");
    return SE3TN_OK;
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
extern "C" {

size_t se3tn_workspace_bytes(int max_batch) {
    if (max_batch <= 0) return 0;
    return workspace_floats(max_batch) * sizeof(float);
}

size_t se3tn_weight_set_bytes(void) { return weight_set_bytes(); }

const char* se3tn_last_error(se3tn_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

int se3tn_create(int device, int max_batch, void* workspace, se3tn_ctx** out) {
    if (!out || max_batch <= 0) return fail(nullptr, SE3TN_ERR_INVALID, "se3tn_create: bad arguments");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || device < 0 || device >= ndev)
        return fail(nullptr, SE3TN_ERR_CUDA, std::string("se3tn_create: no such CUDA device: ") + cudaGetErrorString(e));
    cudaDeviceProp prop;
    CU_TRY(nullptr, cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, SE3TN_ERR_UNSUPPORTED, "se3tn_create: device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) +
                                                    ", this library is sm_90a only (no fallback path)");
    DeviceGuard guard(device);
    std::unique_ptr<se3tn_ctx> ctx(new se3tn_ctx());   // released by any early return below, while the device is still current
    se3tn_ctx* c = ctx.get();
    c->device = device; c->max_batch = max_batch; c->num_sms = prop.multiProcessorCount;
    if (const char* ov = getenv("SE3TN_PDL")) c->pdl = atoi(ov) != 0;
    if (const char* ov = getenv("SE3TN_GRAPH")) c->use_graphs = atoi(ov) != 0;
    if (const char* ov = getenv("SE3TN_TRACE"); ov && atoi(ov) != 0 && dev_alloc(c->trace, SE3TN_TRACE_WORDS) == cudaSuccess)
        cudaMemset(c->trace.get(), 0, SE3TN_TRACE_WORDS * sizeof(unsigned long long));

    void* fn = nullptr; cudaDriverEntryPointQueryResult qres;
    e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
        return fail(nullptr, SE3TN_ERR_CUDA, "se3tn_create: cuTensorMapEncodeTiled entry point unavailable");
    c->encode = reinterpret_cast<EncodeTiledFn>(fn);

    const size_t bytes = se3tn_workspace_bytes(max_batch);
    if (workspace) {
        if (reinterpret_cast<uintptr_t>(workspace) % 1024) return fail(nullptr, SE3TN_ERR_INVALID, "se3tn_create: workspace must be 1024-byte aligned");
        c->workspace = static_cast<uint8_t*>(workspace);
    } else {
        e = dev_alloc(c->own_workspace, bytes);
        if (e != cudaSuccess) return fail(nullptr, SE3TN_ERR_NOMEM, std::string("se3tn_create: cudaMalloc(workspace): ") + cudaGetErrorString(e));
        c->workspace = c->own_workspace.get();
    }
    e = dev_alloc(c->pool_part, static_cast<size_t>(max_batch) * kPoolSlices * 1024);
    if (e != cudaSuccess) return fail(nullptr, SE3TN_ERR_NOMEM, std::string("se3tn_create: pool buffer: ") + cudaGetErrorString(e));
    e = dev_alloc(c->partial, trunk_partial_floats());
    if (e == cudaSuccess) e = dev_alloc(c->sched, trunk_sched_words(max_batch));
    if (e == cudaSuccess) e = cudaMemset(c->sched.get(), 0, trunk_sched_words(max_batch) * sizeof(unsigned));
    if (e != cudaSuccess) return fail(nullptr, SE3TN_ERR_NOMEM, std::string("se3tn_create: scheduler state: ") + cudaGetErrorString(e));
    // zero once: the stem buffers' 3-pixel halo is the conv padding and is never written again
    e = cudaMemset(c->workspace, 0, bytes);
    if (e != cudaSuccess) return fail(nullptr, SE3TN_ERR_CUDA, std::string("se3tn_create: cudaMemset: ") + cudaGetErrorString(e));
    float* p = reinterpret_cast<float*>(c->workspace);
    for (int b = 0; b < B_COUNT; ++b) {
        c->buf[b] = p;
        p += (kBufFloats[b] * static_cast<size_t>(max_batch) + 255) & ~size_t(255);
    }
    int rc = build_activation_maps(c, 4, c->amap4);
    if (!rc) rc = build_activation_maps(c, 2, c->amap2);
    if (!rc) rc = build_activation_maps(c, 1, c->amap1);
    if (rc) return fail(nullptr, rc, c->err);
    // the memsets above ran on the NULL stream: later launches may use non-blocking streams, which do not wait for it
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return fail(nullptr, SE3TN_ERR_CUDA, std::string("se3tn_create: ") + cudaGetErrorString(e));
    *out = ctx.release();
    return SE3TN_OK;
}

void se3tn_destroy(se3tn_ctx* c) {
    if (!c) return;
    DeviceGuard guard(c->device);
    delete c;                                      // the context owns every resource it holds
}

int se3tn_load_weights(se3tn_ctx* c, int weight_id, const float* blob, size_t n_floats) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!blob || weight_id < 0) return fail(c, SE3TN_ERR_INVALID, "se3tn_load_weights: bad arguments");
    const size_t expect = blob_floats();
    if (n_floats != expect || expect != SE3TN_WEIGHT_BLOB_FLOATS)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_load_weights: blob has " + std::to_string(n_floats) + " floats, expected " + std::to_string(expect));
    DeviceGuard guard(c->device);
    // the id counts as loaded only once every form of the new weights is ready: a failed load leaves it not loaded
    WeightSet& ws = c->weights[weight_id];
    ws.dev.reset();
    ws.has_fp8 = false;                            // fp8 activation scales belong to the weights they were calibrated on
    ws.fp16_fits = fp16_weights_fit(blob);
    c->tables_dirty = true;
    c->graphs.clear();                             // captured steps hold the old tensor maps / table pointers
    std::unique_ptr<DeviceWeights> w(new DeviceWeights());
    const int rc = prepare_weights(c, *w, blob);
    if (rc) return rc;
    ws.dev = std::move(w);
    return SE3TN_OK;
}

int se3tn_set_stats(se3tn_ctx* c, int weight_id, const void* mean8, const void* std8, int is_f64) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!mean8 || !std8 || weight_id < 0) return fail(c, SE3TN_ERR_INVALID, "se3tn_set_stats: bad arguments");
    WeightSet& ws = c->weights[weight_id];
    for (int i = 0; i < 8; ++i) {
        if (is_f64) {
            ws.mean64[i] = static_cast<const double*>(mean8)[i]; ws.std64[i] = static_cast<const double*>(std8)[i];
            ws.mean32[i] = static_cast<float>(ws.mean64[i]); ws.std32[i] = static_cast<float>(ws.std64[i]);
        } else {
            ws.mean32[i] = static_cast<const float*>(mean8)[i]; ws.std32[i] = static_cast<const float*>(std8)[i];
            ws.mean64[i] = ws.mean32[i]; ws.std64[i] = ws.std32[i];
        }
    }
    ws.stats_f64 = is_f64 ? 1 : 0; ws.has_stats = true;
    c->stats_dirty = true;
    c->graphs.clear();
    return SE3TN_OK;
}

int se3tn_preprocess(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                     const double* K, const double* poses, const double* object_width,
                     const uint8_t* rgbA, const uint16_t* depthA, const int32_t* weight_ids, int n,
                     int precision, float* out_A, float* out_B, uint8_t* crop_rgb, uint16_t* crop_depth, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !K || !poses || !object_width || !rgbA || !depthA || H <= 0 || W <= 0)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_preprocess: null/invalid argument");
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, "se3tn_preprocess: n exceeds max_batch");
    if ((out_A == nullptr) != (out_B == nullptr)) return fail(c, SE3TN_ERR_INVALID, "se3tn_preprocess: out_A/out_B must both be given or both NULL");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    int rc = sync_stats(c, s); if (rc) return rc;
    PreprocessArgs a{};
    a.frame_rgb = frame_rgb; a.frame_depth = frame_depth; a.H = H; a.W = W;
    a.fx = K[0]; a.fy = K[1]; a.cx = K[2]; a.cy = K[3];
    a.poses = poses; a.object_width = object_width; a.rgbA = rgbA; a.depthA = depthA; a.weight_ids = weight_ids;
    a.precision = precision; a.nchwA = out_A; a.nchwB = out_B; a.crop_rgb = crop_rgb; a.crop_depth = crop_depth;
    return queue_preprocess(c, a, n, s);
}

int se3tn_normalize(se3tn_ctx* c, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                    const double* poses, const int32_t* weight_ids, int n, int precision, float* out_A, float* out_B, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!rgbA || !depthA || !rgbB || !depthB || !poses) return fail(c, SE3TN_ERR_INVALID, "se3tn_normalize: null argument");
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, "se3tn_normalize: n exceeds max_batch");
    if ((out_A == nullptr) != (out_B == nullptr)) return fail(c, SE3TN_ERR_INVALID, "se3tn_normalize: out_A/out_B must both be given or both NULL");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    int rc = sync_stats(c, s); if (rc) return rc;
    PreprocessArgs a{};
    a.frame_rgb = rgbB; a.frame_depth = depthB; a.H = kImg; a.W = kImg; a.b_precropped = 1;
    a.poses = poses; a.rgbA = rgbA; a.depthA = depthA; a.weight_ids = weight_ids;
    a.precision = precision; a.nchwA = out_A; a.nchwB = out_B;
    return queue_preprocess(c, a, n, s);
}

int se3tn_compute_bbox(se3tn_ctx* c, const double* poses, const double* K, const double* widths, const double* scale,
                       int32_t* out_bbox, int n, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!poses || !K || !widths || !scale || !out_bbox || n < 0) return fail(c, SE3TN_ERR_INVALID, "se3tn_compute_bbox: null/invalid argument");
    DeviceGuard guard(c->device);
    CU_TRY(c, launch_bbox(poses, K, widths, scale, out_bbox, n, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

int se3tn_crop_bbox(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const int32_t* bbox, int n,
                    int out_h, int out_w, uint8_t* crop_rgb, uint16_t* crop_depth, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !bbox || !crop_rgb || !crop_depth || H <= 0 || W <= 0 || out_h <= 0 || out_w <= 0 || n < 0)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_crop_bbox: null/invalid argument");
    DeviceGuard guard(c->device);
    CU_TRY(c, launch_crop(frame_rgb, frame_depth, H, W, bbox, n, out_h, out_w, crop_rgb, crop_depth, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

int se3tn_forward(se3tn_ctx* c, int weight_id, const float* A, const float* B, int n,
                  float* out_trans, float* out_rot, float* out_feature, int precision, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!A || !B || !out_trans || !out_rot) return fail(c, SE3TN_ERR_INVALID, "se3tn_forward: null argument");
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, "se3tn_forward: n exceeds max_batch");
    if (n == 0) return SE3TN_OK;
    { const int rc = check_prec(c, "se3tn_forward", weight_id, precision); if (rc) return rc; }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    c->launches = 0;
    { ProfScope ps(c, 19, s);
      CU_TRY(c, launch_nchw_to_stem(A, c->buf[B_X0A], n, precision, s));
      CU_TRY(c, launch_nchw_to_stem(B, c->buf[B_X0B], n, precision, s)); }
    c->launches += 2;
    return run_network(c, weight_id, 0, n, precision, out_trans, out_rot, out_feature, s);
}

int se3tn_forward_preprocessed(se3tn_ctx* c, int weight_id, int first, int n,
                               float* out_trans, float* out_rot, float* out_feature, int precision, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!out_trans || !out_rot) return fail(c, SE3TN_ERR_INVALID, "se3tn_forward_preprocessed: null argument");
    if (first < 0 || n < 0 || first + n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, "se3tn_forward_preprocessed: range exceeds max_batch");
    if (n == 0) return SE3TN_OK;
    { const int rc = check_prec(c, "se3tn_forward_preprocessed", weight_id, precision); if (rc) return rc; }
    DeviceGuard guard(c->device);
    return run_network(c, weight_id, first, n, precision, out_trans, out_rot, out_feature, static_cast<cudaStream_t>(stream));
}

int se3tn_set_fp8_scales(se3tn_ctx* c, int weight_id, const float* scales, int n_scales) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!scales || n_scales != SE3TN_FP8_SCALES) return fail(c, SE3TN_ERR_INVALID, "se3tn_set_fp8_scales: need SE3TN_FP8_SCALES scales");
    auto it = c->weights.find(weight_id);
    if (weight_id < 0 || it == c->weights.end() || !it->second.dev)
        return fail(c, SE3TN_ERR_STATE, "se3tn_set_fp8_scales: weight set " + std::to_string(weight_id) + " not loaded");
    for (int i = 0; i < SE3TN_FP8_SCALES; ++i)
        if (!is_pow2_scale(scales[i]))
            return fail(c, SE3TN_ERR_INVALID, "se3tn_set_fp8_scales: scale " + std::to_string(i) + " (" + std::to_string(scales[i]) +
                                              ") is not a finite positive power of two");
    DeviceGuard guard(c->device);
    return upload_fp8(c, it->second, scales);
}

int se3tn_get_fp8_scales(se3tn_ctx* c, int weight_id, float* scales, int n_scales) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!scales || n_scales != SE3TN_FP8_SCALES) return fail(c, SE3TN_ERR_INVALID, "se3tn_get_fp8_scales: need room for SE3TN_FP8_SCALES scales");
    auto it = c->weights.find(weight_id);
    if (weight_id < 0 || it == c->weights.end() || !it->second.dev || !it->second.has_fp8)
        return fail(c, SE3TN_ERR_STATE, "se3tn_get_fp8_scales: weight set " + std::to_string(weight_id) + " has no fp8 activation scales");
    memcpy(scales, it->second.fp8_scales, sizeof(float) * SE3TN_FP8_SCALES);
    return SE3TN_OK;
}

int se3tn_calibrate_fp8(se3tn_ctx* c, int weight_id, const float* A, const float* B, int n, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!A || !B || n <= 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, "se3tn_calibrate_fp8: null input or n outside [1, max_batch]");
    auto it = c->weights.find(weight_id);
    if (weight_id < 0 || it == c->weights.end() || !it->second.dev)
        return fail(c, SE3TN_ERR_STATE, "se3tn_calibrate_fp8: weight set " + std::to_string(weight_id) + " not loaded");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    const size_t scratch = 16 + 6 * static_cast<size_t>(c->max_batch);
    if (!c->fp8_scratch) CU_TRY(c, dev_alloc(c->fp8_scratch, scratch));
    unsigned* amax = reinterpret_cast<unsigned*>(c->fp8_scratch.get());
    float* tr = c->fp8_scratch.get() + 16;
    // the bf16x3 forward leaves every e4m3 tensor of the mode in the buffers, stored in bf16x3
    int rc = se3tn_forward(c, weight_id, A, B, n, tr, tr + 3 * c->max_batch, nullptr, SE3TN_PREC_BF16X3, stream);
    if (rc) return rc;
    AmaxArgs a{};
    auto tensor = [&](int i, Buf b, int pixels, int C, int c0, int nc) { a.t[i] = {reinterpret_cast<const uint8_t*>(c->buf[b]), pixels, C, c0, nc}; };
    tensor(0, B_CAT, 44 * 44, 128, 0, 128);
    tensor(1, B_F1, 22 * 22, 256, 0, 256); tensor(2, B_T4, 22 * 22, 256, 0, 256); tensor(3, B_F2, 22 * 22, 256, 0, 256);
    for (int g = 0; g < 2; ++g) {
        tensor(4 + g, B_H1, 11 * 11, 1024, g * kFp8HeadCh, kFp8HeadCh);
        tensor(6 + g, B_H2, 11 * 11, 1024, g * kFp8HeadCh, kFp8HeadCh);
    }
    a.n_tensors = SE3TN_FP8_SCALES; a.n = n;
    CU_TRY(c, cudaMemsetAsync(amax, 0, SE3TN_FP8_SCALES * sizeof(unsigned), s));
    CU_TRY(c, launch_amax_bf16x3(a, amax, s));
    unsigned bits[SE3TN_FP8_SCALES];
    CU_TRY(c, cudaMemcpyAsync(bits, amax, sizeof bits, cudaMemcpyDeviceToHost, s));
    CU_TRY(c, cudaStreamSynchronize(s));
    float scales[SE3TN_FP8_SCALES];
    for (int i = 0; i < SE3TN_FP8_SCALES; ++i) {
        float m; memcpy(&m, &bits[i], sizeof m);
        if (!std::isfinite(m)) return fail(c, SE3TN_ERR_INVALID, "se3tn_calibrate_fp8: the activations of tensor " + std::to_string(i) + " are not finite");
        scales[i] = pow2_scale(static_cast<double>(m) * SE3TN_FP8_HEADROOM);
    }
    return upload_fp8(c, it->second, scales);
}

int se3tn_pose_update(se3tn_ctx* c, const double* poses_in, const float* trans, const float* rot,
                      double tn, double rn, double* poses_out, int n, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!poses_in || !trans || !rot || !poses_out || n < 0) return fail(c, SE3TN_ERR_INVALID, "se3tn_pose_update: null/invalid argument");
    DeviceGuard guard(c->device);
    { ProfScope ps(c, 18, static_cast<cudaStream_t>(stream)); CU_TRY(c, launch_pose_update(poses_in, trans, rot, static_cast<float>(tn), static_cast<float>(rn), poses_out, n, static_cast<cudaStream_t>(stream))); }
    ++c->launches;
    return SE3TN_OK;
}

int se3tn_so3_log(se3tn_ctx* c, const double* poses_a, const double* poses_b, double tn, double rn,
                  double* trans_label, double* rot_label, int n, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!poses_a || !poses_b || !trans_label || !rot_label || n < 0) return fail(c, SE3TN_ERR_INVALID, "se3tn_so3_log: null/invalid argument");
    DeviceGuard guard(c->device);
    CU_TRY(c, launch_so3_log(poses_a, poses_b, tn, rn, trans_label, rot_label, n, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

} // extern "C"

namespace {

// Input A drawn inside the step (se3tn_track_render): se3tn_render_ex's mode and camera image size (0 x 0 in the vispy mode,
// which ignores them).
struct RenderSpec { int mode, H, W; };

int render_spec(se3tn_ctx* c, const char* fn, int mode, int H, int W, RenderSpec& r) {
    if (mode != SE3TN_RENDER_VISPY && mode != SE3TN_RENDER_PYRENDER) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": unknown render mode");
    const bool pyr = mode == SE3TN_RENDER_PYRENDER;
    if (pyr && (H <= 0 || W <= 0 || H > 65536 || W > 65536)) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": render_H / render_W out of range");
    r = {mode, pyr ? H : 0, pyr ? W : 0};
    return SE3TN_OK;
}

// Host-side checks of one step, before anything is queued.  Every id a track uses needs weights AND channel statistics
// (se3tn_set_stats is per weight id), so that the preprocess kernel never normalises with another set's (or no) statistics.
// A step that renders input A also needs a model for every id: the rasteriser would otherwise draw model 0 in its place.
// *multi: the tracks use more than one weight set.
int check_step(se3tn_ctx* c, const char* fn, const int32_t* wid_host, const int32_t* wid_dev, int n, bool render, bool* multi,
               int precision) {
    if ((wid_host == nullptr) != (wid_dev == nullptr))
        return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": weight_ids_host and weight_ids_dev must both be given or both NULL");
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": n exceeds max_batch");
    *multi = false;
    for (int i = 0; i < n; ++i) {
        const int wid = wid_host ? wid_host[i] : 0;
        auto it = c->weights.find(wid);
        if (wid < 0 || it == c->weights.end() || !it->second.dev) return fail(c, SE3TN_ERR_STATE, "weight set " + std::to_string(wid) + " not loaded");
        if (!it->second.has_stats) return fail(c, SE3TN_ERR_STATE, "weight set " + std::to_string(wid) + " has no mean/std (se3tn_set_stats)");
        if (render && !c->meshes.count(wid))
            return fail(c, SE3TN_ERR_STATE, std::string(fn) + ": id " + std::to_string(wid) + " (track " + std::to_string(i) + ") has no mesh (se3tn_set_mesh)");
        { const int rc = check_prec(c, fn, wid, precision); if (rc) return rc; }
        if (wid != (wid_host ? wid_host[0] : 0)) *multi = true;
        if (!wid_host) break;                       // all tracks use set 0
    }
    return SE3TN_OK;
}

// The depth-fill block for an H x W frame: scratch a | b | lut | minmax, then, when a track step fills the frame, the filled
// uint16 frame.  Captured steps hold the block's addresses, so they are dropped, once the stream has drained, before the block
// is replaced; grow installs the new block only once it exists.
size_t fill_plane_bytes(int H, int W) { return align256(static_cast<size_t>(H) * W * sizeof(float)); }
size_t fill_lut_bytes() { return align256((kFillLutEntries + 1) * sizeof(float)); }
size_t fill_scratch_bytes(int H, int W) { return 2 * fill_plane_bytes(H, W) + fill_lut_bytes() + 2 * sizeof(unsigned); }

int reserve_fill(se3tn_ctx* c, int H, int W, bool filled_frame, cudaStream_t s) {
    const size_t bytes = filled_frame ? align256(fill_scratch_bytes(H, W)) + static_cast<size_t>(H) * W * sizeof(uint16_t) : fill_scratch_bytes(H, W);
    if (bytes <= c->fill_bytes) return SE3TN_OK;
    CU_TRY(c, cudaStreamSynchronize(s));
    c->graphs.clear();
    CU_TRY(c, grow(c->fill, c->fill_bytes, bytes));
    return SE3TN_OK;
}

FillScratch fill_scratch(se3tn_ctx* c, int H, int W) {
    uint8_t* f = c->fill.get();
    const size_t plane = fill_plane_bytes(H, W), lut = fill_lut_bytes();
    return {reinterpret_cast<float*>(f), reinterpret_cast<float*>(f + plane), reinterpret_cast<float*>(f + 2 * plane),
            reinterpret_cast<unsigned*>(f + 2 * plane + lut)};
}

uint16_t* filled_frame(se3tn_ctx* c, int H, int W) { return reinterpret_cast<uint16_t*>(c->fill.get() + align256(fill_scratch_bytes(H, W))); }

// A step as run_step takes it: the key, and the ids on the host.  Only host code reads those: check_step, first_wid / mixed,
// and the fp32 mode's runs of equal ids, which are never captured.
struct Step : StepKey { const int32_t* wid_host; };

// What every track step takes from its scalar arguments and its ids (checked by check_step: `mixed`), added to what track_opts
// wrote; the caller adds the device pointers.
void track_step(Step& st, int H, int W, const double* K, const int32_t* wid_host, bool mixed, int n, double tn, double rn, int precision) {
    st.n = n; st.precision = precision; st.H = H; st.W = W;
    for (int i = 0; i < 4; ++i) st.K[i] = K[i];
    st.tn = tn; st.rn = rn;
    st.wid_host = wid_host; st.first_wid = wid_host ? wid_host[0] : 0; st.mixed = mixed;
    st.render_mode = -1;
}

// The fit check's block: the device route's rows, then the fit's rendered depth of max_batch tracks.
size_t fit_rows_bytes(int max_batch) { return align256(static_cast<size_t>(max_batch) * kFitCols * sizeof(int32_t)); }
int32_t* fit_rows(se3tn_ctx* c) { return reinterpret_cast<int32_t*>(c->fit.get()); }
uint16_t* fit_depth(se3tn_ctx* c) { return reinterpret_cast<uint16_t*>(c->fit.get() + fit_rows_bytes(c->max_batch)); }

// A track step that draws input A first.  It lands in context scratch for max_batch tracks, allocated by the first such step:
// its address never changes after, so captured steps stay valid.  With the fit check on, the step also runs the fit into the
// context's rows (the host route points them at its own output block); their block is allocated the same way, by the first step
// with the check on.
int render_into_scratch(se3tn_ctx* c, const RenderSpec& r, Step& st) {
    const size_t img = static_cast<size_t>(kImg) * kImg, rgb_bytes = align256(static_cast<size_t>(c->max_batch) * img * 3);
    CU_TRY(c, grow(c->in_a, c->in_a_bytes, rgb_bytes + static_cast<size_t>(c->max_batch) * img * 2));
    st.render_mode = r.mode; st.render_H = r.H; st.render_W = r.W;
    st.rgbA = c->in_a.get(); st.depthA = reinterpret_cast<uint16_t*>(c->in_a.get() + rgb_bytes);
    if (st.fit_tau) {
        CU_TRY(c, grow(c->fit, c->fit_bytes, fit_rows_bytes(c->max_batch) + static_cast<size_t>(c->max_batch) * img * sizeof(uint16_t)));
        st.fit_rows = fit_rows(c);
    }
    return SE3TN_OK;
}

// A hypothesis step's scratch: the expanded tracks' poses | widths | ids | trans | rot, max_batch rows each.
struct HypScratch { double* poses; double* width; int32_t* wid; float* trans; float* rot; };
int reserve_hyp(se3tn_ctx* c, HypScratch* x) {
    const size_t mb = static_cast<size_t>(c->max_batch);
    const size_t o_w = align256(mb * 16 * sizeof(double)), o_id = o_w + align256(mb * sizeof(double)),
                 o_tr = o_id + align256(mb * sizeof(int32_t)), o_ro = o_tr + align256(mb * 3 * sizeof(float));
    CU_TRY(c, grow(c->hyp, c->hyp_bytes, o_ro + mb * 3 * sizeof(float)));
    uint8_t* b = c->hyp.get();
    *x = {reinterpret_cast<double*>(b), reinterpret_cast<double*>(b + o_w), reinterpret_cast<int32_t*>(b + o_id),
          reinterpret_cast<float*>(b + o_tr), reinterpret_cast<float*>(b + o_ro)};
    return SE3TN_OK;
}

// The ICP block: sums | the ICP render's depth | its triangle ids, max_batch tracks each.
size_t icp_sums_bytes(int max_batch) { return align256(static_cast<size_t>(max_batch) * kIcpSums * sizeof(double)); }
size_t icp_depth_bytes(int max_batch) { return align256(static_cast<size_t>(max_batch) * kImg * kImg * sizeof(uint16_t)); }
double* icp_sums(se3tn_ctx* c) { return reinterpret_cast<double*>(c->icp.get()); }
uint16_t* icp_depth(se3tn_ctx* c) { return reinterpret_cast<uint16_t*>(c->icp.get() + icp_sums_bytes(c->max_batch)); }
int32_t* icp_tri(se3tn_ctx* c) {
    return reinterpret_cast<int32_t*>(c->icp.get() + icp_sums_bytes(c->max_batch) + icp_depth_bytes(c->max_batch));
}

static_assert(sizeof(se3tn_icp_opts) == 16, "se3tn_icp_opts is 16 bytes without padding: _lib.IcpOpts mirrors it");
static_assert(kIcpCols == SE3TN_ICP_COLS, "se3tn_track_arrays' out_icp columns");
// opts->icp checked and written into st.icp, and the block allocated on the current device: a block that cannot be allocated
// refuses the call and leaves the context as it was.
int icp_opts(se3tn_ctx* c, const char* fn, const se3tn_icp_opts* o, Step& st) {
    const std::string f(fn);
    if (o->iterations < 1 || o->iterations > SE3TN_MAX_ICP_ITERATIONS)
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->icp->iterations is " + std::to_string(o->iterations) + ", not in [1, " +
                    std::to_string(SE3TN_MAX_ICP_ITERATIONS) + "]");
    if (o->tau_mm < 1 || o->tau_mm > 1000) return fail(c, SE3TN_ERR_INVALID, f + ": opts->icp->tau_mm must be in [1, 1000]");
    if (o->min_inliers < 6 || o->min_inliers > kImg * kImg)
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->icp->min_inliers must be in [6, " + std::to_string(kImg * kImg) + "]");
    if (o->reserved) return fail(c, SE3TN_ERR_INVALID, f + ": opts->icp->reserved must be 0");
    const size_t bytes = icp_sums_bytes(c->max_batch) + icp_depth_bytes(c->max_batch) + static_cast<size_t>(c->max_batch) * kImg * kImg * sizeof(int32_t);
    if (grow(c->icp, c->icp_bytes, bytes) != cudaSuccess) {
        cudaGetLastError();
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->icp: its scratch (" + std::to_string(bytes) + " bytes) cannot be allocated");
    }
    st.icp.iterations = o->iterations; st.icp.tau = o->tau_mm; st.icp.min_inliers = o->min_inliers;
    return SE3TN_OK;
}

static_assert(sizeof(se3tn_hypothesis_opts) == 32, "se3tn_hypothesis_opts is 32 bytes without padding: _lib.HypothesisOpts mirrors it");
static_assert(kHypDraws == SE3TN_HYP_DRAWS, "se3tn_draw_hypotheses' out_draws columns");
// The se3tn_hypothesis_opts `name` checked for n tracks and written into st.hyp's scalars.  Refused before anything is queued.
int hypothesis_opts(se3tn_ctx* c, const char* fn, const char* name, const se3tn_hypothesis_opts* h, int n, Step& st) {
    const std::string f = std::string(fn) + ": " + name;
    if (!h) return fail(c, SE3TN_ERR_INVALID, f + " is NULL");
    if (h->hypotheses < 1 || h->hypotheses > SE3TN_MAX_HYPOTHESES)
        return fail(c, SE3TN_ERR_INVALID, f + "->hypotheses is " + std::to_string(h->hypotheses) + ", not in [1, " +
                    std::to_string(SE3TN_MAX_HYPOTHESES) + "]");
    if (h->reserved) return fail(c, SE3TN_ERR_INVALID, f + "->reserved must be 0");
    if (!(std::isfinite(h->max_translation) && h->max_translation > 0.0 && h->max_translation <= 1.0))
        return fail(c, SE3TN_ERR_INVALID, f + "->max_translation must be finite and in (0, 1] m");
    if (!(h->max_rotation_deg > 0.0 && h->max_rotation_deg <= 180.0))
        return fail(c, SE3TN_ERR_INVALID, f + "->max_rotation_deg must be in (0, 180]");
    if (n < 0 || static_cast<long long>(n) * h->hypotheses > c->max_batch)
        return fail(c, SE3TN_ERR_INVALID, f + "->hypotheses x n = " + std::to_string(static_cast<long long>(n) * h->hypotheses) +
                    " exceeds max_batch " + std::to_string(c->max_batch));
    st.hyp.S = h->hypotheses; st.hyp.seed = static_cast<uint64_t>(h->seed);
    st.hyp.max_t = h->max_translation; st.hyp.max_r = h->max_rotation_deg;
    return SE3TN_OK;
}

// A tracking call's se3tn_track_opts (NULL: the defaults) checked and written into its step, so the key holds them: the fill,
// the rounds, the fit check, ICP (its block allocated) and the hypotheses.  renders: the step draws input A; n: its tracks.
// se3tn_track_batch / se3tn_track_host take input A from the caller: a later round, ICP or a hypothesis could not redraw it at
// another pose, and the fit check and ICP could not draw a model the weight id need not have.  ICP inside a hypothesis step is
// refused here, the one place that decides which extras a step runs.  Refused before anything is queued.
static_assert(sizeof(se3tn_track_opts) == 48, "se3tn_track_opts is 48 bytes without padding: _lib.TrackOpts mirrors it");
int track_opts(se3tn_ctx* c, const char* fn, const se3tn_track_opts* o, bool renders, int n, Step& st) {
    st.iterations = 1;
    if (!o) return SE3TN_OK;
    const std::string f(fn);
    if (o->fill_depth) {                           // off: the fill fields stay zero, whatever the caller left in them
        if (o->fill_blur != SE3TN_BLUR_BILATERAL && o->fill_blur != SE3TN_BLUR_GAUSSIAN)
            return fail(c, SE3TN_ERR_INVALID, f + ": opts->fill_blur is " + std::to_string(o->fill_blur) + ", not an SE3TN_BLUR_*");
        const float md = static_cast<float>(o->fill_max_depth);   // what the kernels compute with
        if (!(std::isfinite(md) && md > 0.f)) return fail(c, SE3TN_ERR_INVALID, f + ": opts->fill_max_depth must be finite and > 0");
        st.fill = 1; st.fill_max_depth = o->fill_max_depth; st.fill_extrapolate = o->fill_extrapolate != 0;
        st.fill_blur = static_cast<uint16_t>(o->fill_blur);
    }
    if (o->iterations < 1 || o->iterations > SE3TN_MAX_REFINE_ITERATIONS)
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->iterations must be in [1, " + std::to_string(SE3TN_MAX_REFINE_ITERATIONS) + "]");
    if (o->fit_tau_mm < 0 || o->fit_tau_mm > 1000) return fail(c, SE3TN_ERR_INVALID, f + ": opts->fit_tau_mm must be 0 or in [1, 1000]");
    if (o->reserved) return fail(c, SE3TN_ERR_INVALID, f + ": opts->reserved must be 0");
    if (!renders && o->iterations != 1)
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->iterations is " + std::to_string(o->iterations) + "; input A from the caller "
                    "cannot be redrawn, which needs se3tn_track_render[_host]");
    if (!renders && o->fit_tau_mm)
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->fit_tau_mm is set; input A from the caller, and the fit check draws each "
                    "track's model, which needs se3tn_track_render[_host]");
    if (!renders && (o->icp || o->hyp))
        return fail(c, SE3TN_ERR_INVALID, f + (o->icp ? ": opts->icp" : ": opts->hyp") + " is set; input A from the caller cannot "
                    "be redrawn, which needs se3tn_track_render[_host]");
    if (o->icp && o->hyp)
        return fail(c, SE3TN_ERR_INVALID, f + ": opts->icp and opts->hyp are both set; ICP inside a hypothesis step is not supported");
    st.iterations = static_cast<uint16_t>(o->iterations);
    st.fit_tau = o->fit_tau_mm;
    if (o->hyp) {
        const int rc = hypothesis_opts(c, fn, "opts->hyp", o->hyp, n, st);
        if (rc) return rc;
        if (!st.fit_tau)
            return fail(c, SE3TN_ERR_INVALID, f + ": opts->fit_tau_mm must be set with opts->hyp: the choice ranks the hypotheses by "
                        "the fit check's rows");
    }
    if (!o->icp) return SE3TN_OK;
    DeviceGuard guard(c->device);
    return icp_opts(c, fn, o->icp, st);
}

int run_step(se3tn_ctx* c, const Step& st, cudaStream_t s);

// A checked hypothesis step over device arrays: st holds the options and, in st.hyp, the caller's n tracks and outputs.  The
// step's own n x S tracks are the context's scratch (their poses in hyp_poses when the caller wants them); the host ids are
// repeated as the rows repeat them, for first_wid and the fp32 mode's runs of equal ids.
int run_hypotheses(se3tn_ctx* c, Step& st, const RenderSpec& r, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                   const double* K, const int32_t* wid_host, bool multi, int n, double tn, double rn, int precision,
                   double* hyp_poses, double* round_poses, cudaStream_t s) {
    HypScratch x;
    int rc = reserve_hyp(c, &x);
    if (rc) return rc;
    const int S = st.hyp.S;
    std::vector<int32_t> ids(wid_host ? static_cast<size_t>(n) * S : 0);
    for (size_t row = 0; row < ids.size(); ++row) ids[row] = wid_host[row / S];
    track_step(st, H, W, K, wid_host ? ids.data() : nullptr, multi, n * S, tn, rn, precision);
    st.frame_rgb = frame_rgb; st.frame_depth = frame_depth;
    st.poses_out = hyp_poses ? hyp_poses : x.poses;         // every round refines the expanded starts in place
    st.poses_in = st.poses_out;
    st.object_width = x.width; st.wid_dev = st.hyp.wid_in ? x.wid : nullptr;
    st.out_trans = x.trans; st.out_rot = x.rot; st.round_poses = round_poses;
    if ((rc = render_into_scratch(c, r, st))) return rc;
    return run_step(c, st, s);
}

// The conv stack over a step's n tracks.  Tensor-core modes: one forward in which every track picks its own weight set when the
// ids are mixed, its head doing `head` too.  fp32: one FFMA forward per run of equal ids, `head` left to the caller.
int run_tracks(se3tn_ctx* c, const Step& st, const HeadArgs& head, cudaStream_t s) {
    if (st.precision != SE3TN_PREC_FP32)
        return run_network(c, st.first_wid, 0, st.n, st.precision, st.out_trans, st.out_rot, nullptr, s, st.mixed ? st.wid_dev : nullptr, head);
    for (int first = 0; first < st.n;) {
        const int wid = st.wid_host ? st.wid_host[first] : 0;
        int last = first + 1;
        while (last < st.n && (st.wid_host ? st.wid_host[last] : 0) == wid) ++last;
        const int rc = run_network(c, wid, first, last - first, st.precision, st.out_trans + first * 3, st.out_rot + first * 3, nullptr, s);
        if (rc) return rc;
        first = last;
    }
    return SE3TN_OK;
}

// se3tn_eval_pairs_augmented's scratch: the draws, then augmented rgbB | depthB of max_batch pairs
double* aug_params(se3tn_ctx* c) { return reinterpret_cast<double*>(c->aug.get()); }
size_t aug_params_bytes(int max_batch) { return align256(static_cast<size_t>(max_batch) * SE3TN_AUG_PARAMS * sizeof(double)); }
uint8_t* aug_rgb(se3tn_ctx* c) { return c->aug.get() + aug_params_bytes(c->max_batch); }
uint16_t* aug_depth(se3tn_ctx* c) {
    return reinterpret_cast<uint16_t*>(aug_rgb(c) + align256(static_cast<size_t>(c->max_batch) * kImg * kImg * 3));
}
int reserve_aug(se3tn_ctx* c) {
    const size_t img = static_cast<size_t>(c->max_batch) * kImg * kImg;
    CU_TRY(c, grow(c->aug, c->aug_bytes, aug_params_bytes(c->max_batch) + align256(img * 3) + img * 2));
    return SE3TN_OK;
}

// se3tn_augment checked and turned into a step's AugKey.  n: the pairs of the call (n > max_batch is refused).
int check_augment(se3tn_ctx* c, const char* fn, const se3tn_augment* a, int n, AugKey* out) {
    const std::string f(fn);
    if (!a) return fail(c, SE3TN_ERR_INVALID, f + ": NULL augmentation");
    if (a->depth_missing) return fail(c, SE3TN_ERR_UNSUPPORTED, f + ": DepthMissing is not supported (commented out in the reference's train.py)");
    if (n <= 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, f + ": n must be in [1, max_batch]");
    const int32_t flags[5] = {a->hsv_jitter, a->change_bright, a->gaussian_noise, a->gaussian_blur, a->black_cover};
    AugKey k{};
    for (int i = 0; i < 5; ++i) {
        if (flags[i] != 0 && flags[i] != 1) return fail(c, SE3TN_ERR_INVALID, f + ": stage flags must be 0 or 1");
        k.stages |= flags[i] << i;
    }
    if (!k.stages) return fail(c, SE3TN_ERR_INVALID, f + ": no stage enabled (se3tn_eval_pairs evaluates the pairs as they are)");
    const double probs[4] = {a->hsv_prob, a->noise_prob, a->blur_prob, a->cover_prob};
    for (double p : probs)
        if (!(p >= 0.0 && p <= 1.0)) return fail(c, SE3TN_ERR_INVALID, f + ": probabilities must lie in [0, 1]");
    const double mags[5] = {a->hsv_noise[0], a->hsv_noise[1], a->hsv_noise[2], a->bright_mag[0], a->bright_mag[1]};
    for (double m : mags)
        if (!std::isfinite(m)) return fail(c, SE3TN_ERR_INVALID, f + ": magnitudes must be finite");
    if (!(std::isfinite(a->noise_rgb) && std::isfinite(a->noise_depth) && a->noise_rgb >= 0.0 && a->noise_depth >= 0.0))
        return fail(c, SE3TN_ERR_INVALID, f + ": noise magnitudes must be finite and >= 0");
    const int half = a->blur_max_kernel / 2;
    if (a->gaussian_blur && (a->blur_max_kernel < 0 || half < 1 || half > 3))
        return fail(c, SE3TN_ERR_INVALID, f + ": blur_max_kernel " + std::to_string(a->blur_max_kernel) +
                    " draws k outside {3, 5, 7}");
    k.seed = a->seed;
    k.hsv_prob = a->hsv_prob; for (int i = 0; i < 3; ++i) k.hsv_noise[i] = a->hsv_noise[i];
    k.bright_lo = a->bright_mag[0]; k.bright_hi = a->bright_mag[1];
    k.noise_prob = a->noise_prob; k.noise_rgb = a->noise_rgb; k.noise_depth = a->noise_depth;
    k.blur_prob = a->blur_prob; k.cover_prob = a->cover_prob;
    k.blur_half_max = a->gaussian_blur ? half : 0;
    *out = k;
    return SE3TN_OK;
}

// Every output of an augmentation call must be disjoint from its inputs: a CTA's reads of input B (the blur's halo rows) may come
// after another CTA has written its own rows.  Pairs of (pointer, bytes).
int check_disjoint(se3tn_ctx* c, const char* fn, std::initializer_list<std::pair<const void*, size_t>> outs,
                   std::initializer_list<std::pair<const void*, size_t>> ins, const char* why = "in-place augmentation is not supported") {
    auto overlap = [](const std::pair<const void*, size_t>& a, const std::pair<const void*, size_t>& b) {
        const uintptr_t x = reinterpret_cast<uintptr_t>(a.first), y = reinterpret_cast<uintptr_t>(b.first);
        return a.first && b.first && x < y + b.second && y < x + a.second;
    };
    for (auto o = outs.begin(); o != outs.end(); ++o) {
        for (const auto& i : ins)
            if (overlap(*o, i)) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": an output overlaps an input (" + why + ")");
        for (auto o2 = o + 1; o2 != outs.end(); ++o2)
            if (overlap(*o, *o2)) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": two outputs overlap");
    }
    return SE3TN_OK;
}

// The launches of one step on stream s, captured or not: render (if set) -> fill (if on) -> preprocess (track) or normalize
// (validation) -> conv stack -> the fp32 pose update (track) or the loss (validation: pair_loss in fp32, the reduction of the
// head's terms otherwise).  A track step that renders input A repeats render -> preprocess -> conv stack -> pose update
// st.iterations times on the same (filled) frame: round 0 reads poses_in, every later round reads and writes poses_out in place,
// exactly as a chain of single-round steps would.  With st.fit_tau, the fit check follows the last round: render (depth only)
// at poses_out -> fit_kernel, which writes st.fit_rows and nothing the rounds read.  Arguments come from `st` alone, context
// state only as the graph cache's comment in se3tn_ctx lists.
int step_launches(se3tn_ctx* c, const Step& st, cudaStream_t s) {
    c->launches = 0;
    const double K[4] = {st.K[0], st.K[1], st.K[2], st.K[3]};
    const bool fp32 = st.precision == SE3TN_PREC_FP32;
    int rc;
    if (st.kind == kStepPairs) {                   // se3tn_perturb_pairs: compute_bbox -> render A (pyrender mode) -> crop B with its seg
        const double scale[3] = {1000.0, 1000.0, 1000.0};     // produce_train_pair_data.py:118
        CU_TRY(c, launch_bbox(st.poses_in, K, st.object_width, scale, c->pair_bbox.get(), st.n, s));
        ++c->launches;
        rc = queue_render(c, K, st.poses_in, st.object_width, st.wid_dev, st.n, SE3TN_RENDER_PYRENDER, st.H, st.W,
                          const_cast<uint8_t*>(st.rgbA), const_cast<uint16_t*>(st.depthA), s);
        if (rc) return rc;
        CU_TRY(c, launch_crop_seg(st.frame_rgb, st.frame_depth, st.seg, st.H, st.W, c->pair_bbox.get(), st.class_ids, st.n, kImg, kImg,
                                  const_cast<uint8_t*>(st.rgbB), const_cast<uint16_t*>(st.depthB), st.segB, st.seg_count, s));
        ++c->launches;
        return SE3TN_OK;
    }
    if (st.hyp.S) {                                // hypothesis step: the n x S starts, ids and widths every later launch reads
        HypArgs h{};
        h.poses_in = st.hyp.poses_in; h.keys = st.hyp.keys; h.n = st.n / st.hyp.S; h.S = st.hyp.S; h.seed = st.hyp.seed;
        h.max_t = st.hyp.max_t; h.max_r_deg = st.hyp.max_r; h.wid_in = st.hyp.wid_in; h.width_in = st.hyp.width_in;
        h.poses = const_cast<double*>(st.poses_in); h.wid = const_cast<int32_t*>(st.wid_dev); h.width = const_cast<double*>(st.object_width);
        CU_TRY(c, launch_hypotheses(h, s));
        ++c->launches;
    }
    if (st.render_mode >= 0) {                     // track i draws mesh weight_ids[i] (0 without ids): one network and one model per object
        // after the expansion, a plain launch: preprocess_kernel reads the ids before its griddepcontrol.wait, and the chain of
        // PDL launches behind this render starts only once the expansion has completed
        rc = queue_render(c, K, st.poses_in, st.object_width, st.wid_dev, st.n, st.render_mode, st.render_H, st.render_W,
                          const_cast<uint8_t*>(st.rgbA), const_cast<uint16_t*>(st.depthA), s, st.hyp.S == 0);
        if (rc) return rc;
    }
    const uint16_t* depth = st.frame_depth;
    if (st.fill) {                                 // fill_depth(frame_depth) into the block run_step sized; the caller's frame is only read
        const bool gaussian = st.fill_blur == SE3TN_BLUR_GAUSSIAN;
        uint16_t* filled = filled_frame(c, st.H, st.W);
        CU_TRY(c, launch_fill_depth(st.frame_depth, st.H, st.W, static_cast<float>(st.fill_max_depth), st.fill_extrapolate != 0, gaussian,
                                    fill_scratch(c, st.H, st.W), filled, nullptr, s));
        c->launches += fill_depth_launches(st.fill_extrapolate != 0, gaussian);
        depth = filled;
    }
    // preprocess_kernel is launched with programmatic stream serialization, so it may start while the launch in front of it
    // (render_kernel, or the last fill kernel, both of which execute griddepcontrol.launch_dependents) is still running.  It
    // reads rgbA / depthA and the frame only after griddepcontrol.wait (aux_kernels.cu, grid_dep_wait()), which returns once
    // that launch has completed and its writes are visible: keep every read of input A and of the frame behind that wait.
    // The fill kernels themselves are plain launches, so the first one starts after the render has completed.
    PreprocessArgs a{};
    a.rgbA = st.rgbA; a.depthA = st.depthA; a.weight_ids = st.wid_dev; a.precision = st.precision;
    HeadArgs head;
    if (st.kind == kStepTrack) {
        a.frame_rgb = st.frame_rgb; a.frame_depth = depth; a.H = st.H; a.W = st.W; a.object_width = st.object_width;
        a.fx = K[0]; a.fy = K[1]; a.cx = K[2]; a.cy = K[3];
        head.pose_out = st.poses_out;
        head.tn = static_cast<float>(st.tn); head.rn = static_cast<float>(st.rn);
    } else {                                       // both depths are offset by A's z (reference datasets.py:136 -> data_augmentation.py:134-144)
        a.frame_rgb = st.rgbB; a.frame_depth = st.depthB; a.H = kImg; a.W = kImg; a.b_precropped = 1;
        if (st.aug.stages) {                       // input B augmented first; the normalize launch waits for it (grid_dep_wait)
            const aug::Config cfg = st.aug.config();
            double* params = aug_params(c);
            CU_TRY(c, launch_augment_draws(cfg, st.depthB, st.aug_seg, st.pair_index, st.n, params, s));
            CU_TRY(c, launch_augment_pixels(cfg, st.rgbB, st.depthB, st.pair_index, params, st.n, st.aug_rgb, st.aug_depth, s));
            c->launches += 2;
            a.frame_rgb = st.aug_rgb; a.frame_depth = st.aug_depth;
        }
        head.loss.poses_a = st.poses_in; head.loss.poses_b = st.B_in_cam; head.loss.tn = st.tn; head.loss.rn = st.rn;
        head.loss.sq = st.sq; head.loss.labels = st.labels;
    }
    const int rounds = st.kind == kStepTrack && st.render_mode >= 0 ? st.iterations : 1;
    for (int round = 0; round < rounds; ++round) {
        const double* poses = round == 0 ? st.poses_in : st.poses_out;
        if (round > 0) {
            // render_project_kernel (PDL) may start under the previous round's head / pose-update kernel, which writes these
            // poses; it reads them, and writes the projected vertices the previous round's render_kernel read, only after its
            // griddepcontrol.wait, which returns once that kernel -- and so, through each kernel's own wait, every earlier
            // launch of the step -- has completed.
            rc = queue_render(c, K, poses, st.object_width, st.wid_dev, st.n, st.render_mode, st.render_H, st.render_W,
                              const_cast<uint8_t*>(st.rgbA), const_cast<uint16_t*>(st.depthA), s);
            if (rc) return rc;
        }
        a.poses = poses;
        if (st.kind == kStepTrack) head.pose_in = poses;
        if ((rc = queue_preprocess(c, a, st.n, s))) return rc;
        if ((rc = run_tracks(c, st, head, s))) return rc;
        if (st.kind == kStepTrack) {
            if (fp32) {                            // otherwise the head kernel has updated the poses
                ProfScope ps(c, 18, s);
                CU_TRY(c, launch_pose_update(poses, st.out_trans, st.out_rot, head.tn, head.rn, st.poses_out, st.n, s));
                ++c->launches;
            }
            // the poses after round + 1, what a (round + 1)-round step leaves in poses_out; the next round's render waits for the copy
            if (st.round_poses)
                CU_TRY(c, cudaMemcpyAsync(st.round_poses + static_cast<size_t>(round) * st.n * 16, st.poses_out,
                                          sizeof(double) * 16 * static_cast<size_t>(st.n), cudaMemcpyDeviceToDevice, s));
            continue;
        } else {
            ProfScope ps(c, 21, s);
            if (fp32) CU_TRY(c, launch_pair_loss(st.out_trans, st.out_rot, nullptr, nullptr, head.loss, st.n, st.sums, s));
            else CU_TRY(c, launch_loss_reduce(st.sq, st.n, st.sums, s));
        }
        ++c->launches;
    }
    if (st.icp.iterations) {
        // M ICP iterations at poses_out, each render (depth + triangle ids, into the ICP block) -> accumulate -> solve, the solve
        // updating poses_out in place.  Every launch is PDL: each reads what the launch before it wrote only after its
        // griddepcontrol.wait, as the rounds' renders do.  The copies into icp_poses are ordered like round_poses'.
        RenderArgs ra = render_args(c, K, st.poses_out, st.object_width, st.wid_dev, st.render_mode, st.render_H, st.render_W,
                                    nullptr, icp_depth(c));
        ra.tri = icp_tri(c);
        IcpArgs ia{};
        ia.poses = st.poses_out; ia.object_width = st.object_width; ia.mesh_ids = st.wid_dev; ia.meshes = c->d_meshes.get();
        ia.n_meshes = c->mesh_rows; ia.fx = K[0]; ia.fy = K[1]; ia.cx = K[2]; ia.cy = K[3];
        ia.frame_depth = depth; ia.H = st.H; ia.W = st.W; ia.tri = icp_tri(c); ia.tau = st.icp.tau; ia.min_inliers = st.icp.min_inliers;
        ia.sums = icp_sums(c); ia.stats = st.icp.stats;
        for (int it = 0; it < st.icp.iterations; ++it) {
            CU_TRY(c, launch_render(ra, st.n, s));
            CU_TRY(c, launch_icp(ia, st.n, s));
            c->launches += 4;
            if (st.icp.poses)
                CU_TRY(c, cudaMemcpyAsync(st.icp.poses + static_cast<size_t>(it) * st.n * 16, st.poses_out,
                                          sizeof(double) * 16 * static_cast<size_t>(st.n), cudaMemcpyDeviceToDevice, s));
        }
    }
    if (st.fit_tau) {
        // the fit check at poses_out: render_project_kernel (PDL) reads the poses the last round's head / pose update wrote only
        // after its griddepcontrol.wait, as a later round's render does, and fit_kernel reads the depth drawn here, the poses and
        // the frame only after its own.  Depth only, into the fit's scratch: the step's input A keeps the last round's.  No
        // profiling slot: slot 20 keeps timing the last round's render.
        const RenderArgs ra = render_args(c, K, st.poses_out, st.object_width, st.wid_dev, st.render_mode, st.render_H, st.render_W,
                                          nullptr, fit_depth(c));
        CU_TRY(c, launch_render(ra, st.n, s));
        c->launches += 2;
        FitArgs fa;
        fa.poses = st.poses_out; fa.object_width = st.object_width; fa.fx = K[0]; fa.fy = K[1]; fa.cx = K[2]; fa.cy = K[3];
        fa.frame_depth = depth; fa.H = st.H; fa.W = st.W; fa.rendered = fit_depth(c); fa.tau = st.fit_tau; fa.rows = st.fit_rows;
        CU_TRY(c, launch_fit(fa, st.n, s));
        ++c->launches;
    }
    if (st.hyp.S) {                                // the choice: a plain launch, after fit_kernel has completed
        SelectArgs sa{};
        sa.n = st.n / st.hyp.S; sa.S = st.hyp.S; sa.rows = st.fit_rows; sa.poses = st.poses_out; sa.trans = st.out_trans; sa.rot = st.out_rot;
        sa.poses_out = st.hyp.poses_out; sa.trans_out = st.hyp.trans_out; sa.rot_out = st.hyp.rot_out; sa.choice = st.hyp.choice;
        sa.fit_out = st.hyp.fit_out;
        CU_TRY(c, launch_select(sa, s));
        ++c->launches;
    }
    return SE3TN_OK;
}

// One step through the context's CUDA graphs (not with SE3TN_GRAPH=0, profiling or SE3TN_PREC_FP32): a step whose key was seen
// before is one graph launch; a new one is captured from step_launches on the private capture stream, then launched.  Otherwise,
// or when capture turns out not to be possible (plain launches from then on), step_launches runs on s.
int run_step(se3tn_ctx* c, const Step& st, cudaStream_t s) {
    int rc;
    if (st.fill && (rc = reserve_fill(c, st.H, st.W, true, s))) return rc;   // before the lookup: a new block drops every graph
    c->last_was_graph = false;
    const StepKey& key = st;
    bool capture = c->use_graphs && !c->profiling && st.precision != SE3TN_PREC_FP32;
    if (capture)
        for (auto& g : c->graphs)
            if (memcmp(&g.key, &key, sizeof key) == 0) {
                CU_TRY(c, cudaGraphLaunch(g.exec.get(), s));
                g.last_use = ++c->graph_clock; c->launches = g.launches; c->last_was_graph = true;
                return SE3TN_OK;
            }
    // host-side refreshes: synchronous copies, which must not happen inside a capture
    if (st.kind != kStepPairs && (rc = sync_stats(c, s))) return rc;     // a pair step runs no network
    if (st.mixed && (rc = sync_tables(c, s))) return rc;
    if (st.render_mode >= 0 && (rc = sync_meshes(c, s))) return rc;
    if (capture) {
        if (c->sched_dirty) { CU_TRY(c, cudaMemsetAsync(c->sched.get(), 0, trunk_sched_words(c->max_batch) * sizeof(unsigned), s)); c->sched_dirty = false; }
        cudaStream_t cs = nullptr;
        if (!c->cap_stream && cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) == cudaSuccess) c->cap_stream.reset(cs);
        capture = c->cap_stream && cudaStreamBeginCapture(c->cap_stream.get(), cudaStreamCaptureModeRelaxed) == cudaSuccess;
        if (!capture) { cudaGetLastError(); c->use_graphs = 0; }
    }
    if (capture) {
        // turn what was recorded into an executable graph and run it; any failure falls back to plain stream launches for good
        rc = step_launches(c, st, c->cap_stream.get());
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        const bool ok = cudaStreamEndCapture(c->cap_stream.get(), &graph) == cudaSuccess && rc == SE3TN_OK && graph &&
                        cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
        if (graph) cudaGraphDestroy(graph);
        if (ok) {
            if (c->graphs.size() >= 64)                        // evict the least recently used step
                c->graphs.erase(std::min_element(c->graphs.begin(), c->graphs.end(), [](const auto& a, const auto& b) { return a.last_use < b.last_use; }));
            c->graphs.push_back({key, Handle<cudaGraphExec_t>(exec), c->launches, ++c->graph_clock});
            CU_TRY(c, cudaGraphLaunch(exec, s));
            c->last_was_graph = true;
            return SE3TN_OK;
        }
        cudaGetLastError(); c->use_graphs = 0; c->sched_dirty = true;
        if (rc) return rc;                                     // a real launch error
    }
    return step_launches(c, st, s);
}

// se3tn_eval_pairs and se3tn_eval_pairs_augmented: `aug` carries the augmentation fields of the step (NULL: none).
int eval_pairs_step(se3tn_ctx* c, const char* fn, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                    const double* A_in_cam, const double* B_in_cam, const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                    double tn, double rn, int precision, float* out_trans, float* out_rot, float* out_sq, double* out_labels,
                    float* out_sums, const Step* aug, void* stream) {
    const std::string f(fn);
    if (!c) return SE3TN_ERR_INVALID;
    if (!rgbA || !depthA || !rgbB || !depthB || !A_in_cam || !B_in_cam) return fail(c, SE3TN_ERR_INVALID, f + ": null input");
    if (!out_trans || !out_rot || !out_sums) return fail(c, SE3TN_ERR_INVALID, f + ": null output");
    if (precision < SE3TN_PREC_TF32 || precision > SE3TN_PREC_FP16) return fail(c, SE3TN_ERR_INVALID, f + ": unknown precision");
    bool multi = false;
    int rc = check_step(c, fn, weight_ids_host, weight_ids_dev, n, false, &multi, precision);
    if (rc) return rc;
    if (n == 0) return fail(c, SE3TN_ERR_INVALID, f + ": n == 0 (the loss of no pairs is undefined)");
    DeviceGuard guard(c->device);
    const bool tensor = precision != SE3TN_PREC_FP32;
    // allocated once, at max_batch pairs: nothing queued uses it before, and captured steps keep its address after
    if (tensor && !out_sq) CU_TRY(c, grow(c->loss_sq, c->loss_sq_floats, static_cast<size_t>(c->max_batch) * 6));
    Step st{};
    if (aug) {
        if ((rc = reserve_aug(c))) return rc;
        st.aug = aug->aug; st.aug_seg = aug->aug_seg; st.pair_index = aug->pair_index;
        st.aug_rgb = aug->aug_rgb ? aug->aug_rgb : aug_rgb(c);
        st.aug_depth = aug->aug_depth ? aug->aug_depth : aug_depth(c);
    }
    st.kind = kStepEval; st.n = n; st.precision = precision; st.tn = tn; st.rn = rn; st.render_mode = -1;
    st.wid_host = weight_ids_host; st.first_wid = weight_ids_host ? weight_ids_host[0] : 0; st.mixed = multi;
    st.rgbA = rgbA; st.depthA = depthA; st.rgbB = rgbB; st.depthB = depthB; st.poses_in = A_in_cam; st.B_in_cam = B_in_cam;
    st.wid_dev = weight_ids_dev; st.out_trans = out_trans; st.out_rot = out_rot;
    st.sq = out_sq ? out_sq : (tensor ? c->loss_sq.get() : nullptr); st.labels = out_labels; st.sums = out_sums;
    return run_step(c, st, static_cast<cudaStream_t>(stream));
}

// A render step's se3tn_track_arrays checked against its options (st, from track_opts), before anything is queued: each field is
// taken only where the options use it (host: the host route, which keeps no per-round, per-hypothesis or per-iteration poses).
// On the device route the step's outputs must not overlap what it reads later or each other: round_poses the poses a later
// round reads, icp_poses and out_icp those and each other, and a hypothesis step's outputs its inputs.
int track_arrays(se3tn_ctx* c, const char* fn, const se3tn_track_arrays& a, const Step& st, bool host, int n,
                 const double* poses_in, const double* poses_out, const float* out_trans, const float* out_rot) {
    const bool hyp = st.hyp.S != 0, icp = st.icp.iterations != 0, fit_rows = host ? st.fit_tau != 0 : hyp;
    const struct { const void* p; bool taken, required; const char* name; } fields[] = {
        {a.out_fit, fit_rows, fit_rows, "out_fit"}, {a.out_choice, hyp, hyp, "out_choice"},
        {a.draw_keys, hyp, hyp && st.hyp.S > 1, "draw_keys"}, {a.round_poses, !host, false, "round_poses"},
        {a.hyp_poses, hyp && !host, false, "hyp_poses"}, {a.icp_poses, icp && !host, false, "icp_poses"},
        {a.out_icp, icp, false, "out_icp"}};
    for (const auto& x : fields) {
        if (x.p && !x.taken)
            return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": arrays->" + x.name + " is set, but this step does not take it");
        if (!x.p && x.required)
            return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": arrays->" + x.name + " is NULL, but this step's options need it");
    }
    if (host || n <= 0) return SE3TN_OK;
    const size_t nn = static_cast<size_t>(n), rows = nn * (hyp ? st.hyp.S : 1);
    const std::pair<const void*, size_t> in = {poses_in, nn * 128}, out = {poses_out, nn * 128}, rounds = {a.round_poses, st.iterations * rows * 128};
    if (hyp)
        return check_disjoint(c, fn, {out, {out_trans, nn * 12}, {out_rot, nn * 12}, {a.out_choice, nn * 4}, {a.out_fit, nn * 4 * kFitCols},
                                      {a.hyp_poses, rows * 128}, rounds},
                              {{poses_out == poses_in ? nullptr : poses_in, nn * 128}, {a.draw_keys, nn * 8}},
                              "the starts are drawn from poses_in and draw_keys; poses_out may be poses_in itself");
    int rc = check_disjoint(c, fn, {rounds}, {in, out}, "round_poses must not overlap poses_in or poses_out: a later round reads them");
    if (rc || !icp) return rc;
    const char* why = "icp_poses and out_icp must not overlap poses_in, poses_out, round_poses or each other";
    rc = check_disjoint(c, fn, {{a.icp_poses, st.icp.iterations * nn * 128}}, {in, out, rounds, {a.out_icp, nn * kIcpCols * sizeof(double)}}, why);
    if (!rc) rc = check_disjoint(c, fn, {{a.out_icp, nn * kIcpCols * sizeof(double)}}, {in, out, rounds}, why);
    return rc;
}

}  // namespace

extern "C" {

int se3tn_track_batch(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                      const double* K, const double* poses_in, const double* object_width,
                      const uint8_t* rgbA, const uint16_t* depthA,
                      const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                      double tn, double rn, int precision,
                      float* out_trans, float* out_rot, double* poses_out, const se3tn_track_opts* opts, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!out_trans || !out_rot || !poses_out) return fail(c, SE3TN_ERR_INVALID, "se3tn_track_batch: null output");
    bool multi = false;
    Step st{};
    int rc = track_opts(c, "se3tn_track_batch", opts, false, n, st);
    if (rc) return rc;
    rc = check_step(c, "se3tn_track_batch", weight_ids_host, weight_ids_dev, n, false, &multi, precision);
    if (rc) return rc;
    if (n == 0) return SE3TN_OK;
    if (!frame_rgb || !frame_depth || !K || !poses_in || !object_width || !rgbA || !depthA || H <= 0 || W <= 0)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_track_batch: null argument or empty frame");
    if (precision < SE3TN_PREC_TF32 || precision > SE3TN_PREC_FP16) return fail(c, SE3TN_ERR_INVALID, "se3tn_track_batch: unknown precision");
    DeviceGuard guard(c->device);
    track_step(st, H, W, K, weight_ids_host, multi, n, tn, rn, precision);
    st.frame_rgb = frame_rgb; st.frame_depth = frame_depth; st.poses_in = poses_in; st.object_width = object_width;
    st.rgbA = rgbA; st.depthA = depthA; st.wid_dev = weight_ids_dev;
    st.out_trans = out_trans; st.out_rot = out_rot; st.poses_out = poses_out;
    return run_step(c, st, static_cast<cudaStream_t>(stream));
}

int se3tn_track_render(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W,
                       const double* K, const double* poses_in, const double* object_width,
                       int render_mode, int render_H, int render_W,
                       const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                       double tn, double rn, int precision,
                       float* out_trans, float* out_rot, double* poses_out, const se3tn_track_opts* opts,
                       const se3tn_track_arrays* arrays, void* stream) {
    const char* fn = "se3tn_track_render";
    const std::string f(fn);
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !K || !poses_in || !object_width || H <= 0 || W <= 0)
        return fail(c, SE3TN_ERR_INVALID, f + ": null argument or empty frame");
    if (!out_trans || !out_rot || !poses_out) return fail(c, SE3TN_ERR_INVALID, f + ": null output");
    RenderSpec r;
    int rc = render_spec(c, fn, render_mode, render_H, render_W, r);
    if (rc) return rc;
    Step st{};
    if ((rc = track_opts(c, fn, opts, true, n, st))) return rc;
    bool multi = false;
    if ((rc = check_step(c, fn, weight_ids_host, weight_ids_dev, n, true, &multi, precision))) return rc;
    // The struct is read on the host.  A device pointer in its place (a caller built against a header whose se3tn_track_render
    // took a device round_poses there) is refused rather than dereferenced.
    if (arrays) {
        cudaPointerAttributes where{};
        if (cudaPointerGetAttributes(&where, arrays) != cudaSuccess) cudaGetLastError();   // unknown to the runtime: host memory
        else if (where.type == cudaMemoryTypeDevice)
            return fail(c, SE3TN_ERR_INVALID, f + ": arrays points to device memory; se3tn_track_arrays is HOST memory whose fields "
                        "(round_poses and the other outputs) point to the device");
    }
    const se3tn_track_arrays a = arrays ? *arrays : se3tn_track_arrays{};
    if ((rc = track_arrays(c, fn, a, st, false, n, poses_in, poses_out, out_trans, out_rot))) return rc;
    if (n == 0) return SE3TN_OK;
    if (precision < SE3TN_PREC_TF32 || precision > SE3TN_PREC_FP16) return fail(c, SE3TN_ERR_INVALID, f + ": unknown precision");
    DeviceGuard guard(c->device);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (st.hyp.S) {
        st.hyp.poses_in = poses_in; st.hyp.keys = a.draw_keys; st.hyp.wid_in = weight_ids_dev; st.hyp.width_in = object_width;
        st.hyp.poses_out = poses_out; st.hyp.trans_out = out_trans; st.hyp.rot_out = out_rot; st.hyp.choice = a.out_choice;
        st.hyp.fit_out = a.out_fit;
        return run_hypotheses(c, st, r, frame_rgb, frame_depth, H, W, K, weight_ids_host, multi, n, tn, rn, precision, a.hyp_poses,
                              a.round_poses, s);
    }
    st.icp.poses = a.icp_poses; st.icp.stats = a.out_icp;
    track_step(st, H, W, K, weight_ids_host, multi, n, tn, rn, precision);
    st.frame_rgb = frame_rgb; st.frame_depth = frame_depth; st.poses_in = poses_in; st.object_width = object_width;
    st.wid_dev = weight_ids_dev; st.out_trans = out_trans; st.out_rot = out_rot; st.poses_out = poses_out;
    st.round_poses = a.round_poses;
    if ((rc = render_into_scratch(c, r, st))) return rc;
    return run_step(c, st, s);
}

int se3tn_draw_hypotheses(se3tn_ctx* c, const double* poses_in, const int64_t* draw_keys, int n, const se3tn_hypothesis_opts* hyp,
                          double* out_poses, double* out_draws, void* stream) {
    const char* fn = "se3tn_draw_hypotheses";
    if (!c) return SE3TN_ERR_INVALID;
    if (!poses_in || !out_poses) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": null argument");
    Step st{};
    int rc = hypothesis_opts(c, fn, "hyp", hyp, n, st);
    if (rc) return rc;
    if (st.hyp.S > 1 && !draw_keys) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": draw_keys is NULL with hyp->hypotheses > 1");
    if (n == 0) return SE3TN_OK;
    const size_t nn = static_cast<size_t>(n), rows = nn * st.hyp.S;
    rc = check_disjoint(c, fn, {{out_poses, rows * 128}, {out_draws, rows * 8 * kHypDraws}}, {{poses_in, nn * 128}, {draw_keys, nn * 8}},
                        "the starts are drawn from poses_in and draw_keys");
    if (rc) return rc;
    DeviceGuard guard(c->device);
    HypArgs h{};
    h.poses_in = poses_in; h.keys = draw_keys; h.n = n; h.S = st.hyp.S; h.seed = st.hyp.seed; h.max_t = st.hyp.max_t;
    h.max_r_deg = st.hyp.max_r; h.poses = out_poses; h.draws = out_draws;
    CU_TRY(c, launch_hypotheses(h, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

int se3tn_eval_pairs(se3tn_ctx* c, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                     const double* A_in_cam, const double* B_in_cam,
                     const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                     double tn, double rn, int precision,
                     float* out_trans, float* out_rot, float* out_sq, double* out_labels, float* out_sums, void* stream) {
    return eval_pairs_step(c, "se3tn_eval_pairs", rgbA, depthA, rgbB, depthB, A_in_cam, B_in_cam, weight_ids_host, weight_ids_dev, n, tn,
                           rn, precision, out_trans, out_rot, out_sq, out_labels, out_sums, nullptr, stream);
}

int se3tn_eval_pairs_augmented(se3tn_ctx* c, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                               const double* A_in_cam, const double* B_in_cam,
                               const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n,
                               double tn, double rn, int precision,
                               float* out_trans, float* out_rot, float* out_sq, double* out_labels, float* out_sums,
                               const uint8_t* segB, const int64_t* pair_index, const se3tn_augment* aug,
                               uint8_t* out_rgbB, uint16_t* out_depthB, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!pair_index) return fail(c, SE3TN_ERR_INVALID, "se3tn_eval_pairs_augmented: NULL pair_index");
    Step st{};
    int rc = check_augment(c, "se3tn_eval_pairs_augmented", aug, n, &st.aug);
    if (rc) return rc;
    const size_t px = static_cast<size_t>(n) * kImg * kImg;
    if ((rc = check_disjoint(c, "se3tn_eval_pairs_augmented", {{out_rgbB, px * 3}, {out_depthB, px * 2}},
                             {{rgbB, px * 3}, {depthB, px * 2}, {segB, px}, {pair_index, n * sizeof(int64_t)}})))
        return rc;
    st.aug_seg = segB; st.pair_index = pair_index; st.aug_rgb = out_rgbB; st.aug_depth = out_depthB;
    return eval_pairs_step(c, "se3tn_eval_pairs_augmented", rgbA, depthA, rgbB, depthB, A_in_cam, B_in_cam, weight_ids_host, weight_ids_dev,
                           n, tn, rn, precision, out_trans, out_rot, out_sq, out_labels, out_sums, &st, stream);
}

int se3tn_augment_draws(se3tn_ctx* c, const se3tn_augment* aug, const uint16_t* depthB, const uint8_t* segB, const int64_t* pair_index,
                        int n, double* out_params, double* out_noise_rgb, double* out_noise_depth, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    AugKey k;
    int rc = check_augment(c, "se3tn_augment_draws", aug, n, &k);
    if (rc) return rc;
    if (!depthB || !pair_index || !out_params) return fail(c, SE3TN_ERR_INVALID, "se3tn_augment_draws: null argument");
    const size_t px = static_cast<size_t>(n) * kImg * kImg;
    if ((rc = check_disjoint(c, "se3tn_augment_draws", {{out_params, n * SE3TN_AUG_PARAMS * sizeof(double)}, {out_noise_rgb, px * 3 * sizeof(double)},
                                                        {out_noise_depth, px * sizeof(double)}},
                             {{depthB, px * 2}, {segB, px}, {pair_index, n * sizeof(int64_t)}})))
        return rc;
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const aug::Config cfg = k.config();
    c->launches = 0;
    CU_TRY(c, launch_augment_draws(cfg, depthB, segB, pair_index, n, out_params, s));
    CU_TRY(c, launch_augment_noise(cfg, pair_index, out_params, n, out_noise_rgb, out_noise_depth, s));
    c->launches = out_noise_rgb || out_noise_depth ? 2 : 1;
    return SE3TN_OK;
}

int se3tn_augment_crops(se3tn_ctx* c, const se3tn_augment* aug, const uint8_t* rgbB, const uint16_t* depthB, const uint8_t* segB,
                        const int64_t* pair_index, int n, uint8_t* out_rgbB, uint16_t* out_depthB, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    AugKey k;
    int rc = check_augment(c, "se3tn_augment_crops", aug, n, &k);
    if (rc) return rc;
    if (!rgbB || !depthB || !pair_index || !out_rgbB || !out_depthB) return fail(c, SE3TN_ERR_INVALID, "se3tn_augment_crops: null argument");
    const size_t px = static_cast<size_t>(n) * kImg * kImg;
    if ((rc = check_disjoint(c, "se3tn_augment_crops", {{out_rgbB, px * 3}, {out_depthB, px * 2}},
                             {{rgbB, px * 3}, {depthB, px * 2}, {segB, px}, {pair_index, n * sizeof(int64_t)}})))
        return rc;
    DeviceGuard guard(c->device);
    if ((rc = reserve_aug(c))) return rc;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const aug::Config cfg = k.config();
    c->launches = 0;
    CU_TRY(c, launch_augment_draws(cfg, depthB, segB, pair_index, n, aug_params(c), s));
    CU_TRY(c, launch_augment_pixels(cfg, rgbB, depthB, pair_index, aug_params(c), n, out_rgbB, out_depthB, s));
    c->launches = 2;
    return SE3TN_OK;
}

int se3tn_pair_loss(se3tn_ctx* c, const float* trans, const float* rot, const double* trans_label, const double* rot_label, int n,
                    float* out_sums, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!trans || !rot || !trans_label || !rot_label || !out_sums || n <= 0) return fail(c, SE3TN_ERR_INVALID, "se3tn_pair_loss: null/invalid argument");
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    c->launches = 0;
    { ProfScope ps(c, 21, s); CU_TRY(c, launch_pair_loss(trans, rot, trans_label, rot_label, LossArgs{}, n, out_sums, s)); }
    ++c->launches;
    return SE3TN_OK;
}

int se3tn_crop_bbox_seg(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, const uint8_t* seg, int H, int W,
                        const int32_t* bbox, const int32_t* class_ids, int n, int out_h, int out_w,
                        uint8_t* crop_rgb, uint16_t* crop_depth, uint8_t* crop_seg, int32_t* seg_count, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !seg || !bbox || !crop_rgb || !crop_depth || !crop_seg || H <= 0 || W <= 0 || out_h <= 0 ||
        out_w <= 0 || n < 0 || (seg_count && !class_ids))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_crop_bbox_seg: null/invalid argument");
    DeviceGuard guard(c->device);
    CU_TRY(c, launch_crop_seg(frame_rgb, frame_depth, seg, H, W, bbox, class_ids, n, out_h, out_w, crop_rgb, crop_depth, crop_seg,
                              seg_count, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

}  // extern "C"

namespace {
// The mesh ids of a visibility, pair, init or fit_poses call, checked on the host before anything is queued: both or neither of
// the host and device copies (ids_name: the arguments' stem, mesh_ids or weight_ids), n within max_batch, a model for every id.
int check_meshes(se3tn_ctx* c, const char* fn, const char* ids_name, const int32_t* ids_host, const int32_t* ids_dev, int n) {
    if ((ids_host == nullptr) != (ids_dev == nullptr))
        return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": " + ids_name + "_host and " + ids_name + "_dev must both be given or both NULL");
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": n is " + std::to_string(n) + ", not in [0, max_batch]");
    for (int i = 0; i < n; ++i) {
        const int id = ids_host ? ids_host[i] : 0;
        if (!c->meshes.count(id))
            return fail(c, SE3TN_ERR_STATE, std::string(fn) + ": mesh id " + std::to_string(id) + " (row " + std::to_string(i) + ") has no mesh (se3tn_set_mesh)");
        if (!ids_host) break;
    }
    return SE3TN_OK;
}
}  // namespace

extern "C" {

int se3tn_visibility(se3tn_ctx* c, const uint8_t* seg, int H, int W, const double* K, const double* poses,
                     const int32_t* mesh_ids_host, const int32_t* mesh_ids_dev, const int32_t* class_ids, int m,
                     int32_t* out_visible, int32_t* out_covered, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!seg || !K || !poses || !class_ids || !out_visible || !out_covered || H <= 0 || W <= 0 || H > 65536 || W > 65536)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_visibility: null argument or frame size out of range");
    int rc = check_meshes(c, "se3tn_visibility", "mesh_ids", mesh_ids_host, mesh_ids_dev, m);
    if (rc) return rc;
    if (m == 0) return SE3TN_OK;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    if ((rc = sync_meshes(c, s))) return rc;
    const size_t words = static_cast<size_t>(m) * H * W;
    if (words > c->cover_z_words) {                 // the old planes may still be read by a queued call
        CU_TRY(c, cudaStreamSynchronize(s));
        CU_TRY(c, grow(c->cover_z, c->cover_z_words, words));
    }
    int max_nf = 0;
    for (auto& kv : c->meshes) max_nf = std::max(max_nf, kv.second.nf);
    RenderArgs a;
    a.poses = poses; a.object_width = nullptr; a.mesh_ids = mesh_ids_dev; a.meshes = c->d_meshes.get(); a.n_meshes = c->mesh_rows;
    a.fx = K[0]; a.fy = K[1]; a.cx = K[2]; a.cy = K[3];
    a.rgb = nullptr; a.depth = nullptr; a.mode = 2; a.vw = W; a.vh = H;
    a.projected = c->render_proj.get(); a.uniforms = c->render_unif.get(); a.max_nv = c->render_max_nv;
    c->launches = 0;
    { ProfScope ps(c, 20, s); CU_TRY(c, launch_coverage(a, m, max_nf, seg, class_ids, c->cover_z.get(), out_visible, out_covered, s)); }
    c->launches = 3;
    return SE3TN_OK;
}

int se3tn_perturb_pairs(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, const uint8_t* seg, int H, int W,
                        const double* K, const double* A_in_cam, const double* object_width,
                        const int32_t* mesh_ids_host, const int32_t* mesh_ids_dev, const int32_t* class_ids, int n,
                        uint8_t* rgbA, uint16_t* depthA, uint8_t* rgbB, uint16_t* depthB, uint8_t* segB, int32_t* seg_count,
                        void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !seg || !K || !A_in_cam || !object_width || !class_ids || H <= 0 || W <= 0 || H > 65536 || W > 65536)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_perturb_pairs: null argument or frame size out of range");
    if (!rgbA || !depthA || !rgbB || !depthB || !segB || !seg_count) return fail(c, SE3TN_ERR_INVALID, "se3tn_perturb_pairs: null output");
    int rc = check_meshes(c, "se3tn_perturb_pairs", "mesh_ids", mesh_ids_host, mesh_ids_dev, n);
    if (rc) return rc;
    if (n == 0) return SE3TN_OK;
    DeviceGuard guard(c->device);
    // allocated once, at max_batch rows: captured steps keep its address after
    CU_TRY(c, grow(c->pair_bbox, c->pair_bbox_ints, c->max_batch * 8));
    Step st{};
    st.kind = kStepPairs; st.n = n; st.H = H; st.W = W;
    for (int i = 0; i < 4; ++i) st.K[i] = K[i];
    st.render_mode = SE3TN_RENDER_PYRENDER; st.render_H = H; st.render_W = W;
    st.frame_rgb = frame_rgb; st.frame_depth = frame_depth; st.seg = seg; st.poses_in = A_in_cam; st.object_width = object_width;
    st.wid_dev = mesh_ids_dev; st.class_ids = class_ids;
    st.rgbA = rgbA; st.depthA = depthA; st.rgbB = rgbB; st.depthB = depthB; st.segB = segB; st.seg_count = seg_count;
    return run_step(c, st, static_cast<cudaStream_t>(stream));
}

// se3tn_append_pairs (with_seg false: segB / q_segB are ignored and the kernel copies four planes) and se3tn_append_pairs_seg
static int append_pairs(se3tn_ctx* c, const char* fn, bool with_seg, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB,
                        const uint16_t* depthB, const uint8_t* segB, const int32_t* seg_count, const double* A_in_cam,
                        const double* B_in_cam, const int32_t* queue_ids_host, const int32_t* queue_ids_dev, int n,
                        int num_queues, int cap, const int32_t* tails_host, int32_t* tails_dev,
                        uint8_t* q_rgbA, uint16_t* q_depthA, uint8_t* q_rgbB, uint16_t* q_depthB, uint8_t* q_segB,
                        double* q_A_in_cam, double* q_B_in_cam, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    const std::string name(fn);
    const void* words[] = {rgbA, depthA, rgbB, depthB, A_in_cam, B_in_cam, q_rgbA, q_depthA, q_rgbB, q_depthB, q_A_in_cam, q_B_in_cam,
                           with_seg ? segB : rgbA, with_seg ? q_segB : rgbA};
    for (const void* p : words)
        if (!p || reinterpret_cast<uintptr_t>(p) % 16)
            return fail(c, SE3TN_ERR_INVALID, name + ": a pair or queue array is null or not 16-byte aligned");
    if (!seg_count || !queue_ids_host || !queue_ids_dev || !tails_host || !tails_dev || n < 0 || num_queues <= 0 || cap <= 0)
        return fail(c, SE3TN_ERR_INVALID, name + ": null/invalid argument");
    if (n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, name + ": n exceeds max_batch");
    std::vector<int> rows(num_queues, 0);
    for (int i = 0; i < n; ++i) {
        const int q = queue_ids_host[i];
        if (q < 0 || q >= num_queues)
            return fail(c, SE3TN_ERR_INVALID, name + ": row " + std::to_string(i) + " has queue id " + std::to_string(q) +
                                              ", outside [0, " + std::to_string(num_queues) + ")");
        ++rows[q];
    }
    for (int q = 0; q < num_queues; ++q)
        if (tails_host[q] < 0 || static_cast<long long>(tails_host[q]) + rows[q] > cap)
            return fail(c, SE3TN_ERR_INVALID, name + ": queue " + std::to_string(q) + " holds " + std::to_string(tails_host[q]) +
                                              " of " + std::to_string(cap) + " rows and cannot take " + std::to_string(rows[q]) + " more");
    if (n == 0) return SE3TN_OK;
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (!c->append_done_words) {
        CU_TRY(c, grow(c->append_done, c->append_done_words, 1));
        CU_TRY(c, cudaMemsetAsync(c->append_done.get(), 0, sizeof(unsigned), s));
    }
    AppendArgs a{};
    a.rgbA = rgbA; a.depthA = depthA; a.rgbB = rgbB; a.depthB = depthB;
    a.count = seg_count; a.A_in_cam = A_in_cam; a.B_in_cam = B_in_cam; a.queue_ids = queue_ids_dev;
    a.n = n; a.num_queues = num_queues; a.cap = cap; a.min_count = SE3TN_PAIR_MIN_SEG;
    a.tails = tails_dev; a.done = c->append_done.get();
    a.q_rgbA = q_rgbA; a.q_depthA = q_depthA; a.q_rgbB = q_rgbB; a.q_depthB = q_depthB; a.q_A = q_A_in_cam; a.q_B = q_B_in_cam;
    if (with_seg) a.segB = segB, a.q_segB = q_segB;
    c->launches = 0;
    CU_TRY(c, launch_append_pairs(a, s));
    c->launches = 1;
    return SE3TN_OK;
}

int se3tn_append_pairs(se3tn_ctx* c, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                       const int32_t* seg_count, const double* A_in_cam, const double* B_in_cam,
                       const int32_t* queue_ids_host, const int32_t* queue_ids_dev, int n,
                       int num_queues, int cap, const int32_t* tails_host, int32_t* tails_dev,
                       uint8_t* q_rgbA, uint16_t* q_depthA, uint8_t* q_rgbB, uint16_t* q_depthB, double* q_A_in_cam, double* q_B_in_cam,
                       void* stream) {
    return append_pairs(c, "se3tn_append_pairs", false, rgbA, depthA, rgbB, depthB, nullptr, seg_count, A_in_cam, B_in_cam, queue_ids_host,
                        queue_ids_dev, n, num_queues, cap, tails_host, tails_dev, q_rgbA, q_depthA, q_rgbB, q_depthB, nullptr,
                        q_A_in_cam, q_B_in_cam, stream);
}

int se3tn_append_pairs_seg(se3tn_ctx* c, const uint8_t* rgbA, const uint16_t* depthA, const uint8_t* rgbB, const uint16_t* depthB,
                           const int32_t* seg_count, const double* A_in_cam, const double* B_in_cam,
                           const int32_t* queue_ids_host, const int32_t* queue_ids_dev, int n,
                           int num_queues, int cap, const int32_t* tails_host, int32_t* tails_dev,
                           uint8_t* q_rgbA, uint16_t* q_depthA, uint8_t* q_rgbB, uint16_t* q_depthB, double* q_A_in_cam, double* q_B_in_cam,
                           const uint8_t* segB, uint8_t* q_segB, void* stream) {
    return append_pairs(c, "se3tn_append_pairs_seg", true, rgbA, depthA, rgbB, depthB, segB, seg_count, A_in_cam, B_in_cam, queue_ids_host,
                        queue_ids_dev, n, num_queues, cap, tails_host, tails_dev, q_rgbA, q_depthA, q_rgbB, q_depthB, q_segB,
                        q_A_in_cam, q_B_in_cam, stream);
}

int se3tn_add_adi(se3tn_ctx* c, const double* model_pts, int m, const double* pred, const double* gt, int n,
                  double* out_add, double* out_adi, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!model_pts || !pred || !gt || m <= 0 || n < 0 || (!out_add && !out_adi)) return fail(c, SE3TN_ERR_INVALID, "se3tn_add_adi: null/invalid argument");
    DeviceGuard guard(c->device);
    CU_TRY(c, launch_add_adi(model_pts, m, pred, gt, n, out_add, out_adi, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

int se3tn_vocap(se3tn_ctx* c, const double* errs, int n, double* out_ap, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!out_ap || n < 0 || (n > 0 && !errs)) return fail(c, SE3TN_ERR_INVALID, "se3tn_vocap: null/invalid argument");
    DeviceGuard guard(c->device);
    CU_TRY(c, vocap(errs, n, out_ap, static_cast<cudaStream_t>(stream)));
    return SE3TN_OK;
}

namespace {
// A point table's set offsets (host, n_sets + 1) and the set id (host) of each of n items: SE3TN_ERR_INVALID unless the offsets
// start at 0, increase strictly and end at M, and every id is in [0, n_sets).
int check_sets(se3tn_ctx* c, const char* fn, int M, const int32_t* set_offsets, int n_sets, const int32_t* ids, int n, const char* item) {
    const std::string f(fn);
    if (set_offsets[0] != 0 || set_offsets[n_sets] != M)
        return fail(c, SE3TN_ERR_INVALID, f + ": set_offsets must start at 0 and end at M = " + std::to_string(M));
    for (int s = 0; s < n_sets; ++s)
        if (set_offsets[s + 1] <= set_offsets[s])
            return fail(c, SE3TN_ERR_INVALID, f + ": set " + std::to_string(s) + " is empty or its offsets decrease");
    for (int i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= n_sets)
            return fail(c, SE3TN_ERR_INVALID, f + ": " + item + " " + std::to_string(i) + " has set id " + std::to_string(ids[i]) +
                                              " outside [0, " + std::to_string(n_sets) + ")");
    return SE3TN_OK;
}

// Grows the metrics scratch to hold the checked offsets and ids and `extra` more bytes after them, and queues the upload of the
// offsets and ids on s.  -> their device copies and the extra bytes (256-byte aligned).
int stage_sets(se3tn_ctx* c, const int32_t* set_offsets, int n_sets, const int32_t* ids, int n, size_t extra, cudaStream_t s,
               int32_t** d_off, int32_t** d_ids, uint8_t** d_extra) {
    const size_t off_bytes = align256(sizeof(int32_t) * (static_cast<size_t>(n_sets) + 1));
    const size_t id_bytes = align256(sizeof(int32_t) * static_cast<size_t>(n));
    CU_TRY(c, grow(c->metrics, c->metrics_bytes, off_bytes + id_bytes + extra));
    *d_off = reinterpret_cast<int32_t*>(c->metrics.get());
    *d_ids = reinterpret_cast<int32_t*>(c->metrics.get() + off_bytes);
    *d_extra = c->metrics.get() + off_bytes + id_bytes;
    CU_TRY(c, cudaMemcpyAsync(*d_off, set_offsets, sizeof(int32_t) * (n_sets + 1), cudaMemcpyHostToDevice, s));
    CU_TRY(c, cudaMemcpyAsync(*d_ids, ids, sizeof(int32_t) * n, cudaMemcpyHostToDevice, s));
    return SE3TN_OK;
}
}  // namespace

int se3tn_add_adi_sets(se3tn_ctx* c, const double* pts, int M, const int32_t* set_offsets, int n_sets, const int32_t* pose_set,
                       const double* pred, const double* gt, int n, double* out_add, double* out_adi, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!pts || !set_offsets || M <= 0 || n_sets <= 0 || n < 0 || (n > 0 && (!pose_set || !pred || !gt || (!out_add && !out_adi))))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_add_adi_sets: null/invalid argument");
    int rc = check_sets(c, "se3tn_add_adi_sets", M, set_offsets, n_sets, pose_set, n, "pose");
    if (rc || n == 0) return rc;
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int32_t *d_off, *d_set; uint8_t* unused;
    if ((rc = stage_sets(c, set_offsets, n_sets, pose_set, n, 0, s, &d_off, &d_set, &unused))) return rc;
    CU_TRY(c, launch_add_adi_sets(pts, d_off, d_set, pred, gt, n, out_add, out_adi, s));
    return SE3TN_OK;
}

int se3tn_pose_errors_sets(se3tn_ctx* c, const double* pts, int M, const int32_t* set_offsets, int n_sets, const int32_t* pose_set,
                           const double* pred, const double* gt, const uint8_t* keep, int n, double* out_errors, int32_t* out_set,
                           void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!pts || !set_offsets || M <= 0 || n_sets <= 0 || n < 0 || (n > 0 && (!pose_set || !pred || !gt || !out_errors)))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_pose_errors_sets: null/invalid argument");
    int rc = check_sets(c, "se3tn_pose_errors_sets", M, set_offsets, n_sets, pose_set, n, "pose");
    if (rc || n == 0) return rc;
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int32_t *d_off, *d_set; uint8_t* unused;
    if ((rc = stage_sets(c, set_offsets, n_sets, pose_set, n, 0, s, &d_off, &d_set, &unused))) return rc;
    CU_TRY(c, launch_pose_errors_sets(pts, d_off, d_set, pred, gt, keep, n, out_errors, out_set, s));
    return SE3TN_OK;
}

int se3tn_draw_tracks(se3tn_ctx* c, const uint8_t* frame_rgb, int H, int W, const double* K, const double* poses, int n,
                      const double* pts, int M, const int32_t* set_offsets, int n_sets, const int32_t* track_set,
                      const uint8_t* label_mask, int label_y0, int label_h, int label_order, uint8_t* out_bgr, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !K || !pts || !set_offsets || M <= 0 || n_sets <= 0 || n < 0 || (n > 0 && (!poses || !track_set || !out_bgr)))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_draw_tracks: null/invalid argument");
    if (H <= 0 || W <= 0 || H % 2 || W % 2 || H > (1 << 15) || W > (1 << 15))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_draw_tracks: the frame must have an even height and width in [2, 32768], not " +
                                          std::to_string(H) + " x " + std::to_string(W));
    if (label_order != SE3TN_LABEL_UNDER_POINTS && label_order != SE3TN_LABEL_OVER_POINTS)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_draw_tracks: unknown label_order");
    if (label_mask && (label_y0 < 0 || label_h <= 0 || label_y0 > H - label_h))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_draw_tracks: label rows [" + std::to_string(label_y0) + ", " +
                                          std::to_string(static_cast<long long>(label_y0) + label_h) + ") outside the frame");
    int rc = check_sets(c, "se3tn_draw_tracks", M, set_offsets, n_sets, track_set, n, "track");
    if (rc || n == 0) return rc;
    int max_m = 0;
    for (int i = 0; i < n; ++i) max_m = std::max(max_m, set_offsets[track_set[i] + 1] - set_offsets[track_set[i]]);
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int32_t *d_off, *d_set; uint8_t* masks;
    if ((rc = stage_sets(c, set_offsets, n_sets, track_set, n, sizeof(uint32_t) * overlay_mask_words(H, W) * n, s, &d_off, &d_set, &masks)))
        return rc;
    CU_TRY(c, launch_draw_tracks(frame_rgb, H, W, K, poses, n, pts, d_off, d_set, max_m, label_mask, label_y0, label_h,
                                 label_order == SE3TN_LABEL_OVER_POINTS, reinterpret_cast<uint32_t*>(masks), out_bgr, s));
    return SE3TN_OK;
}

int se3tn_vocap_sets(se3tn_ctx* c, const double* errs, const int32_t* err_set, int n, int n_sets, double* out_ap, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!out_ap || n < 0 || n_sets <= 0 || (n > 0 && (!errs || !err_set))) return fail(c, SE3TN_ERR_INVALID, "se3tn_vocap_sets: null/invalid argument");
    if (n == 0) { std::fill(out_ap, out_ap + n_sets + 1, 0.0); return SE3TN_OK; }
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    size_t bytes = 0;
    CU_TRY(c, vocap_sets_scratch_bytes(n, n_sets, &bytes));
    CU_TRY(c, grow(c->metrics, c->metrics_bytes, bytes));
    int bad = 0;
    CU_TRY(c, vocap_sets(errs, err_set, n, n_sets, c->metrics.get(), out_ap, &bad, s));
    if (bad) return fail(c, SE3TN_ERR_INVALID, "se3tn_vocap_sets: a set id is outside [0, " + std::to_string(n_sets) + ")");
    return SE3TN_OK;
}

size_t se3tn_metrics_scratch_bytes(se3tn_ctx* c) { return c ? c->metrics_bytes : 0; }

namespace {
// crop window of one track in frame pixels: compute_bbox + crop_bbox's window (reference Utils.py:302-316, 324-327), the same
// arithmetic as bbox.cuh on the device
inline void host_crop_window(const double* pose, const double* K, double width, int& top, int& left, int& ch, int& cw) {
    const double ox = pose[3] * 1000.0, oy = pose[7] * 1000.0, oz = pose[11] * 1000.0, half = width / 2;
    const double u0 = std::nearbyint((ox - half) * K[0] / oz + K[2]), u1 = std::nearbyint((ox + half) * K[0] / oz + K[2]);
    const double v0 = std::nearbyint((oy - half) * K[1] / oz + K[3]), v1 = std::nearbyint((oy + half) * K[1] / oz + K[3]);
    const double umin = std::fmin(u0, u1), umax = std::fmax(u0, u1), vmin = std::fmin(v0, v1), vmax = std::fmax(v0, v1);
    const double lim = 1.0e9;
    if (!(umin == umin && umax == umax && vmin == vmin && vmax == vmax)) { top = left = ch = cw = 0; return; }
    left = static_cast<int>(std::fmax(-lim, std::fmin(lim, umin))); top = static_cast<int>(std::fmax(-lim, std::fmin(lim, vmin)));
    cw = static_cast<int>(std::fmax(-lim, std::fmin(lim, umax))) - left; ch = static_cast<int>(std::fmax(-lim, std::fmin(lim, vmax))) - top;
}

// se3tn_track_host and se3tn_track_render_host: every pointer is HOST memory.  The crop-window rectangle of the frame and the
// per-track inputs are staged through the context's pinned block into its device buffers (one copy for the per-track
// inputs), one step runs on them -- with input A from the caller (render == NULL) or rendered inside the step, in which case
// nothing of input A crosses the bus -- and one copy brings the outputs back before the stream is synchronised.
int track_host_step(se3tn_ctx* c, const char* fn, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const double* K,
                    const double* poses, const double* object_width, const uint8_t* rgbA, const uint16_t* depthA, const RenderSpec* render,
                    const int32_t* weight_ids, int n, double tn, double rn, int precision,
                    double* poses_out, float* out_trans, float* out_rot, const se3tn_track_opts* opts, const se3tn_track_arrays* arrays,
                    void* stream) {
    bool multi = false;
    Step st{};                                     // options, arrays and ids are checked before anything is staged or copied
    int rc = track_opts(c, fn, opts, render != nullptr, n, st);
    if (rc) return rc;
    const se3tn_track_arrays a = arrays ? *arrays : se3tn_track_arrays{};
    if ((rc = track_arrays(c, fn, a, st, true, n, nullptr, nullptr, nullptr, nullptr))) return rc;
    rc = check_step(c, fn, weight_ids, weight_ids, n, render != nullptr, &multi, precision);
    if (rc) return rc;
    if (n == 0) return SE3TN_OK;
    if (precision < SE3TN_PREC_TF32 || precision > SE3TN_PREC_FP16) return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": unknown precision");
    DeviceGuard guard(c->device);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    auto& io = c->hio;
    const size_t px = static_cast<size_t>(H) * W, img = static_cast<size_t>(kImg) * kImg;
    // ---- (re)size the context-owned buffers: stable addresses from then on, so the captured step is replayed ----
    if (io.H != H || io.W != W || io.n_cap < n) {
        CU_TRY(c, cudaStreamSynchronize(s));
        const int cap = std::max(n, io.n_cap);
        const size_t per = 128 + 8 + img * 3 + img * 2 + 8 + 4 + 128 + 12 + 12 + 4 * kFitCols + 4 + 8 * kIcpCols;
        c->graphs.clear();                                       // before the buffers are replaced: captured steps hold their addresses
        CU_TRY(c, grow(io.dev, io.dev_bytes, align256(px * 3) + align256(px * 2) + align256(per * cap) + 12 * 256));
        CU_TRY(c, grow(io.pin, io.pin_bytes, px * 5 + per * cap + 4096));
        CU_TRY(c, cudaMemsetAsync(io.dev.get(), 0, io.dev_bytes, s));   // on the caller's stream, ahead of the copies below; frame pixels outside the uploaded windows are never read, keep them defined
        io.H = H; io.W = W; io.n_cap = cap;
    }
    uint8_t* d = io.dev.get();
    uint8_t* d_rgb = d; d += align256(px * 3);
    uint16_t* d_depth = reinterpret_cast<uint16_t*>(d); d += align256(px * 2);
    // the per-track arrays are packed by THIS call's n (a step's graph is keyed by n anyway), inputs first, outputs behind them:
    // one host -> device copy carries all inputs, one device -> host copy all outputs; input A takes no room when it is rendered
    const size_t nn = static_cast<size_t>(n), a_img = render ? 0 : img;
    // a hypothesis step's draw keys go up with the poses, its choices come back behind the fit rows
    const size_t o_ow = align256(nn * 128), o_rgbA = o_ow + align256(nn * 8), o_depthA = o_rgbA + align256(nn * a_img * 3),
                 o_key = o_depthA + align256(nn * a_img * 2), o_wid = o_key + (st.hyp.S ? align256(nn * 8) : 0), in_bytes = o_wid + align256(nn * 4);
    const size_t o_tr = align256(nn * 128), o_ro = o_tr + align256(nn * 12), o_fit = o_ro + align256(nn * 12);
    const size_t o_choice = st.fit_tau ? o_fit + align256(nn * 4 * kFitCols) : o_fit;   // the fit check's rows come back too
    const size_t o_icp = st.hyp.S ? o_choice + align256(nn * 4) : o_choice;      // ICP's stats rows come back last
    const size_t out_bytes = st.icp.iterations ? o_icp + nn * 8 * kIcpCols : o_icp;
    uint8_t* d_in = d;
    double* d_poses = reinterpret_cast<double*>(d_in);
    double* d_ow = reinterpret_cast<double*>(d_in + o_ow);
    uint8_t* d_rgbA = d_in + o_rgbA;
    uint16_t* d_depthA = reinterpret_cast<uint16_t*>(d_in + o_depthA);
    int32_t* d_wid = reinterpret_cast<int32_t*>(d_in + o_wid);
    uint8_t* d_res = d_in + in_bytes;
    double* d_out = reinterpret_cast<double*>(d_res);
    float* d_tr = reinterpret_cast<float*>(d_res + o_tr);
    float* d_ro = reinterpret_cast<float*>(d_res + o_ro);
    int32_t* d_fit = reinterpret_cast<int32_t*>(d_res + o_fit);
    int32_t* d_choice = reinterpret_cast<int32_t*>(d_res + o_choice);
    double* d_icp = reinterpret_cast<double*>(d_res + o_icp);
    // ---- the part of the frame the tracks' crop windows touch (K0 reads nothing else) ----
    int y0 = H, y1 = 0, x0 = W, x1 = 0;
    for (int i = 0; i < n; ++i) {
        int top, left, ch, cw;
        host_crop_window(poses + 16 * i, K, object_width[i], top, left, ch, cw);
        if (ch <= 0 || cw <= 0) continue;
        y0 = std::min(y0, std::max(top - 1, 0)); y1 = std::max(y1, std::min(top + ch + 1, H));       // one pixel of margin
        x0 = std::min(x0, std::max(left - 1, 0)); x1 = std::max(x1, std::min(left + cw + 1, W));
    }
    if (y1 <= y0 || x1 <= x0) { y0 = y1 = x0 = x1 = 0; }         // every window misses the frame: nothing of it is read
    // refinement rounds after the first crop at poses only the step computes, and hypotheses' starts: their windows are not known here
    const bool whole_frame = st.iterations > 1 || st.hyp.S > 1;
    if (whole_frame || static_cast<size_t>(y1 - y0) * (x1 - x0) * 2 >= px) { y0 = 0; y1 = H; x0 = 0; x1 = W; }
    // ---- stage through pinned memory, one asynchronous copy per array ----
    // A step that fills the depth reads all of it: OpenCV's bilateral range table is scaled by the min and max of the whole
    // median-filtered image, and extrapolate scans whole columns.  The fit check crops the depth at the windows of the poses the
    // step computes, and ICP associates pixels in the windows of the poses it refines.  Then the whole depth frame goes up; rgb
    // stays windowed.
    const bool whole_depth = st.fill || st.fit_tau || st.icp.iterations;
    uint8_t* hp = io.pin.get();
    const int wh = y1 - y0, ww = x1 - x0;
    if (wh > 0 && ww > 0) {
        uint8_t* st_rgb = hp; hp += static_cast<size_t>(wh) * ww * 3;
        uint8_t* st_dep = hp; if (!whole_depth) hp += align256(static_cast<size_t>(wh) * ww * 2);
        for (int y = 0; y < wh; ++y) {
            memcpy(st_rgb + static_cast<size_t>(y) * ww * 3, frame_rgb + (static_cast<size_t>(y0 + y) * W + x0) * 3, static_cast<size_t>(ww) * 3);
            if (!whole_depth) memcpy(st_dep + static_cast<size_t>(y) * ww * 2, frame_depth + static_cast<size_t>(y0 + y) * W + x0, static_cast<size_t>(ww) * 2);
        }
        const size_t off = static_cast<size_t>(y0) * W + x0;
        CU_TRY(c, cudaMemcpy2DAsync(d_rgb + off * 3, static_cast<size_t>(W) * 3, st_rgb, static_cast<size_t>(ww) * 3, static_cast<size_t>(ww) * 3, wh, cudaMemcpyHostToDevice, s));
        if (!whole_depth)
            CU_TRY(c, cudaMemcpy2DAsync(d_depth + off, static_cast<size_t>(W) * 2, st_dep, static_cast<size_t>(ww) * 2, static_cast<size_t>(ww) * 2, wh, cudaMemcpyHostToDevice, s));
    }
    if (whole_depth) {
        memcpy(hp, frame_depth, px * 2);
        CU_TRY(c, cudaMemcpyAsync(d_depth, hp, px * 2, cudaMemcpyHostToDevice, s));
        hp += px * 2;
    }
    hp = io.pin.get() + align256(static_cast<size_t>(hp - io.pin.get()));
    memcpy(hp, poses, nn * 128);
    memcpy(hp + o_ow, object_width, nn * 8);
    if (!render) {
        memcpy(hp + o_rgbA, rgbA, nn * img * 3);
        memcpy(hp + o_depthA, depthA, nn * img * 2);
    }
    if (a.draw_keys) memcpy(hp + o_key, a.draw_keys, nn * 8);
    if (weight_ids) memcpy(hp + o_wid, weight_ids, nn * 4);
    CU_TRY(c, cudaMemcpyAsync(d_in, hp, weight_ids ? in_bytes : o_wid, cudaMemcpyHostToDevice, s));
    hp += in_bytes;
    if (st.hyp.S) {                              // the n x S rows' fit rows stay in the context's block; the chosen ones come back
        st.hyp.poses_in = d_poses; st.hyp.keys = a.draw_keys ? reinterpret_cast<const int64_t*>(d_in + o_key) : nullptr;
        st.hyp.wid_in = weight_ids ? d_wid : nullptr; st.hyp.width_in = d_ow;
        st.hyp.poses_out = d_out; st.hyp.trans_out = d_tr; st.hyp.rot_out = d_ro; st.hyp.choice = d_choice; st.hyp.fit_out = d_fit;
        rc = run_hypotheses(c, st, *render, d_rgb, d_depth, H, W, K, weight_ids, multi, n, tn, rn, precision, nullptr, nullptr, s);
    } else {
        track_step(st, H, W, K, weight_ids, multi, n, tn, rn, precision);
        st.frame_rgb = d_rgb; st.frame_depth = d_depth; st.poses_in = d_poses; st.object_width = d_ow;
        st.rgbA = d_rgbA; st.depthA = d_depthA; st.wid_dev = weight_ids ? d_wid : nullptr;
        st.out_trans = d_tr; st.out_rot = d_ro; st.poses_out = d_out;
        if (render && (rc = render_into_scratch(c, *render, st))) return rc;
        if (st.fit_tau) st.fit_rows = d_fit;
        if (st.icp.iterations) st.icp.stats = d_icp;
        rc = run_step(c, st, s);
    }
    if (rc) return rc;
    uint8_t* ho = hp;                                            // outputs come back through the same pinned block
    CU_TRY(c, cudaMemcpyAsync(ho, d_res, (out_trans || out_rot || st.fit_tau || a.out_icp) ? out_bytes : nn * 128, cudaMemcpyDeviceToHost, s));
    CU_TRY(c, cudaStreamSynchronize(s));
    memcpy(poses_out, ho, nn * 128);
    if (out_trans) memcpy(out_trans, ho + o_tr, nn * 12);
    if (out_rot) memcpy(out_rot, ho + o_ro, nn * 12);
    if (a.out_fit) memcpy(a.out_fit, ho + o_fit, nn * 4 * kFitCols);
    if (a.out_choice) memcpy(a.out_choice, ho + o_choice, nn * 4);
    if (a.out_icp) memcpy(a.out_icp, ho + o_icp, nn * 8 * kIcpCols);
    return SE3TN_OK;
}
}  // namespace

int se3tn_track_host(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const double* K,
                     const double* poses, const double* object_width, const uint8_t* rgbA, const uint16_t* depthA,
                     const int32_t* weight_ids, int n, double tn, double rn, int precision,
                     double* poses_out, float* out_trans, float* out_rot, const se3tn_track_opts* opts, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !K || !poses || !object_width || !rgbA || !depthA || !poses_out || H <= 0 || W <= 0)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_track_host: null argument or empty frame");
    return track_host_step(c, "se3tn_track_host", frame_rgb, frame_depth, H, W, K, poses, object_width, rgbA, depthA, nullptr,
                           weight_ids, n, tn, rn, precision, poses_out, out_trans, out_rot, opts, nullptr, stream);
}

int se3tn_track_render_host(se3tn_ctx* c, const uint8_t* frame_rgb, const uint16_t* frame_depth, int H, int W, const double* K,
                            const double* poses, const double* object_width, int render_mode, int render_H, int render_W,
                            const int32_t* weight_ids, int n, double tn, double rn, int precision,
                            double* poses_out, float* out_trans, float* out_rot, const se3tn_track_opts* opts,
                            const se3tn_track_arrays* arrays, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_rgb || !frame_depth || !K || !poses || !object_width || !poses_out || H <= 0 || W <= 0)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_track_render_host: null argument or empty frame");
    RenderSpec r;
    const int rc = render_spec(c, "se3tn_track_render_host", render_mode, render_H, render_W, r);
    if (rc) return rc;
    return track_host_step(c, "se3tn_track_render_host", frame_rgb, frame_depth, H, W, K, poses, object_width, nullptr, nullptr, &r,
                           weight_ids, n, tn, rn, precision, poses_out, out_trans, out_rot, opts, arrays, stream);
}

int se3tn_allgather_poses(se3tn_ctx* c, void* nccl_comm, const double* local_poses, double* all_poses, int n_local, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!nccl_comm || n_local < 0 || (n_local > 0 && (!local_poses || !all_poses))) return fail(c, SE3TN_ERR_INVALID, "se3tn_allgather_poses: bad arguments");
    if (n_local == 0) return SE3TN_OK;
    // ncclResult_t ncclAllGather(const void* send, void* recv, size_t sendcount, ncclDataType_t, ncclComm_t, cudaStream_t)
    typedef int (*AllGatherFn)(const void*, void*, size_t, int, void*, cudaStream_t);
    static AllGatherFn fn = nullptr;
    if (!fn) {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);        // the copy torch (or the host) already loaded
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (h) fn = reinterpret_cast<AllGatherFn>(dlsym(h, "ncclAllGather"));
        if (!fn) return fail(c, SE3TN_ERR_UNSUPPORTED, "se3tn_allgather_poses: libnccl.so.2 / ncclAllGather not found");
    }
    DeviceGuard guard(c->device);
    const int kNcclFloat64 = 8;
    const int rc = fn(local_poses, all_poses, static_cast<size_t>(n_local) * 16, kNcclFloat64, nccl_comm, static_cast<cudaStream_t>(stream));
    if (rc != 0) return fail(c, SE3TN_ERR_CUDA, "se3tn_allgather_poses: ncclAllGather returned " + std::to_string(rc));
    return SE3TN_OK;
}

int se3tn_fill_depth_ex(se3tn_ctx* c, const uint16_t* depth_mm, int H, int W, double max_depth, int extrapolate, int blur_type,
                        uint16_t* out_mm, float* out_m, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!depth_mm || H <= 0 || W <= 0 || (!out_mm && !out_m) || (blur_type != SE3TN_BLUR_BILATERAL && blur_type != SE3TN_BLUR_GAUSSIAN))
        return fail(c, SE3TN_ERR_INVALID, "se3tn_fill_depth: bad arguments");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    const int rc = reserve_fill(c, H, W, false, s);   // a larger frame replaces the block, and drops the steps that captured it
    if (rc) return rc;
    CU_TRY(c, launch_fill_depth(depth_mm, H, W, static_cast<float>(max_depth), extrapolate != 0, blur_type == SE3TN_BLUR_GAUSSIAN, fill_scratch(c, H, W), out_mm, out_m, s));
    c->launches += fill_depth_launches(extrapolate != 0, blur_type == SE3TN_BLUR_GAUSSIAN);
    return SE3TN_OK;
}

int se3tn_fill_depth(se3tn_ctx* c, const uint16_t* depth_mm, int H, int W, double max_depth,
                     uint16_t* out_mm, float* out_m, void* stream) {
    return se3tn_fill_depth_ex(c, depth_mm, H, W, max_depth, 0, SE3TN_BLUR_BILATERAL, out_mm, out_m, stream);
}

int se3tn_fit_rows(se3tn_ctx* c, const int32_t** rows) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!rows) return fail(c, SE3TN_ERR_INVALID, "se3tn_fit_rows: null argument");
    if (!c->fit) return fail(c, SE3TN_ERR_STATE, "se3tn_fit_rows: no step has run the fit check yet");
    *rows = fit_rows(c);
    return SE3TN_OK;
}

int se3tn_set_mesh(se3tn_ctx* c, int mesh_id, const float* pos, const float* nrm, const uint8_t* col,
                   const int32_t* faces, int nv, int nf) {
    if (!c) return SE3TN_ERR_INVALID;
    if (mesh_id < 0 || mesh_id > 4095 || !pos || !nrm || !col || !faces || nv <= 0 || nf <= 0)
        return fail(c, SE3TN_ERR_INVALID, "se3tn_set_mesh: bad arguments");
    for (int i = 0; i < 3 * nf; ++i)
        if (faces[i] < 0 || faces[i] >= nv) return fail(c, SE3TN_ERR_INVALID, "se3tn_set_mesh: face index out of range");
    DeviceGuard guard(c->device);
    CU_TRY(c, cudaDeviceSynchronize());
    Mesh m; m.nv = nv; m.nf = nf;                  // the id's previous model stays in place until this one is complete
    CU_TRY(c, dev_alloc(m.pos, 3 * static_cast<size_t>(nv)));
    CU_TRY(c, dev_alloc(m.nrm, 3 * static_cast<size_t>(nv)));
    CU_TRY(c, dev_alloc(m.col, 3 * static_cast<size_t>(nv)));
    CU_TRY(c, dev_alloc(m.faces, 3 * static_cast<size_t>(nf)));
    CU_TRY(c, cudaMemcpy(m.pos.get(), pos, sizeof(float) * 3 * nv, cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(m.nrm.get(), nrm, sizeof(float) * 3 * nv, cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(m.col.get(), col, 3 * static_cast<size_t>(nv), cudaMemcpyHostToDevice));
    CU_TRY(c, cudaMemcpy(m.faces.get(), faces, sizeof(int) * 3 * nf, cudaMemcpyHostToDevice));
    c->meshes[mesh_id] = std::move(m);             // frees the previous model: the device table is rebuilt before the next render
    c->meshes_dirty = true;
    c->graphs.clear();                             // captured track_render steps hold the old table, workspace and largest vertex count
    return SE3TN_OK;
}

int se3tn_render(se3tn_ctx* c, const double* K, const double* poses, const double* object_width,
                 const int32_t* mesh_ids, int n, uint8_t* rgbA, uint16_t* depthA, void* stream) {
    return se3tn_render_ex(c, K, poses, object_width, mesh_ids, n, SE3TN_RENDER_VISPY, 0, 0, rgbA, depthA, stream);
}

int se3tn_render_ex(se3tn_ctx* c, const double* K, const double* poses, const double* object_width,
                    const int32_t* mesh_ids, int n, int mode, int H, int W, uint8_t* rgbA, uint16_t* depthA, void* stream) {
    if (!c) return SE3TN_ERR_INVALID;
    if (n < 0 || !K || (n > 0 && (!poses || !object_width || !rgbA || !depthA))) return fail(c, SE3TN_ERR_INVALID, "se3tn_render: bad arguments");
    if (mode != SE3TN_RENDER_VISPY && mode != SE3TN_RENDER_PYRENDER) return fail(c, SE3TN_ERR_INVALID, "se3tn_render_ex: unknown mode");
    // the camera image of the pyrender-style mode: sample positions are kept in 1/256 pixel as int32
    if (mode == SE3TN_RENDER_PYRENDER && (H <= 0 || W <= 0 || H > 65536 || W > 65536)) return fail(c, SE3TN_ERR_INVALID, "se3tn_render_ex: camera image size out of range");
    if (n == 0) return SE3TN_OK;
    if (n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, "se3tn_render: n exceeds the context's max_batch");
    if (c->meshes.empty()) return fail(c, SE3TN_ERR_STATE, "se3tn_render: no mesh loaded (se3tn_set_mesh)");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    DeviceGuard guard(c->device);
    const int rc = sync_meshes(c, s); if (rc) return rc;
    return queue_render(c, K, poses, object_width, mesh_ids, n, mode, H, W, rgbA, depthA, s);
}

int se3tn_debug_buffer(se3tn_ctx* c, int id, float** ptr, size_t* floats_per_image) {
    if (!c) return SE3TN_ERR_INVALID;
    if (id < 0 || id >= B_COUNT || !ptr || !floats_per_image) return fail(c, SE3TN_ERR_INVALID, "se3tn_debug_buffer: bad id");
    *ptr = c->buf[id]; *floats_per_image = kBufFloats[id];
    return SE3TN_OK;
}

int se3tn_last_launch_count(se3tn_ctx* c) { return c ? c->launches : 0; }
int se3tn_last_step_was_graph(se3tn_ctx* c) { return (c && c->last_was_graph) ? 1 : 0; }

int se3tn_get_trace(se3tn_ctx* c, unsigned long long* out) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!out) return fail(c, SE3TN_ERR_INVALID, "se3tn_get_trace: null argument");
    if (!c->trace) return fail(c, SE3TN_ERR_STATE, "se3tn_get_trace: the context was created without SE3TN_TRACE=1");
    DeviceGuard guard(c->device);
    CU_TRY(c, cudaDeviceSynchronize());
    CU_TRY(c, cudaMemcpy(out, c->trace.get(), SE3TN_TRACE_WORDS * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return SE3TN_OK;
}

int se3tn_set_profiling(se3tn_ctx* c, int enable) {
    if (!c) return SE3TN_ERR_INVALID;
    DeviceGuard guard(c->device);
    if (enable && !c->ev[0][0]) {
        Handle<cudaEvent_t> ev[2][SE3TN_PROFILE_SLOTS];   // installed only once every event exists
        for (auto& row : ev) for (auto& h : row) { cudaEvent_t e = nullptr; CU_TRY(c, cudaEventCreate(&e)); h.reset(e); }
        std::swap(c->ev, ev);
    }
    c->profiling = enable != 0;
    for (int i = 0; i < SE3TN_PROFILE_SLOTS; ++i) c->ev_used[i] = false;
    return SE3TN_OK;
}

int se3tn_get_profile(se3tn_ctx* c, float* ms) {
    if (!c) return SE3TN_ERR_INVALID;
    if (!ms) return fail(c, SE3TN_ERR_INVALID, "se3tn_get_profile: null argument");
    if (!c->ev[0][0]) return fail(c, SE3TN_ERR_STATE, "se3tn_get_profile: profiling was never enabled");
    for (int i = 0; i < SE3TN_PROFILE_SLOTS; ++i) {
        ms[i] = 0.f;
        if (!c->ev_used[i]) continue;
        CU_TRY(c, cudaEventSynchronize(c->ev[1][i].get()));
        CU_TRY(c, cudaEventElapsedTime(&ms[i], c->ev[0][i].get(), c->ev[1][i].get()));
        c->ev_used[i] = false;
    }
    return SE3TN_OK;
}

}  // extern "C"

namespace {
// se3tn_init_poses' and se3tn_init_boxes' scratch for n objects, D depths, D V R candidates each and K kept: offsets into the
// context's init block.  `labels` holds the n labels or the n boxes.
struct InitLayout {
    size_t labels, acc, hist, stats, t0, grid, width, ids, rows, depth, kept_rows, kept_poses, kept_width, kept_ids, icp_poses,
           icp_rows, icp_stats, bytes;
    InitLayout(size_t n, size_t D, size_t VR, size_t K, size_t max_batch) {
        size_t o = 0;
        auto take = [&o](size_t b) { const size_t at = o; o += align256(b); return at; };
        labels = take(n * 4 * sizeof(int32_t)); acc = take(n * kInitAcc * sizeof(unsigned long long));
        hist = take(n * kInitBins * sizeof(unsigned)); stats = take(n * kInitStats * sizeof(long long)); t0 = take(n * D * 3 * sizeof(double));
        const size_t cand = D * VR;
        grid = take(n * cand * 16 * sizeof(double)); width = take(n * cand * sizeof(double)); ids = take(n * cand * sizeof(int32_t));
        rows = take(n * cand * kInitCols * sizeof(int32_t)); depth = take(max_batch * kImg * kImg * sizeof(uint16_t));
        kept_rows = take(n * K * kInitCols * sizeof(int32_t)); kept_poses = take(n * K * 16 * sizeof(double));
        kept_width = take(n * K * sizeof(double)); kept_ids = take(n * K * sizeof(int32_t));
        icp_poses = take(n * K * 16 * sizeof(double)); icp_rows = take(n * K * kInitCols * sizeof(int32_t));
        icp_stats = take(n * K * kIcpCols * sizeof(double));
        bytes = o;
    }
};

static_assert(sizeof(se3tn_init_opts) == 32, "se3tn_init_opts is 32 bytes without padding: _lib.InitOpts mirrors it");
static_assert(kInitCols == SE3TN_INIT_COLS && kInitStats == SE3TN_INIT_STATS && kInitMaxKeep == SE3TN_MAX_INIT_KEEP, "include/se3tn.h");

// opts checked for n objects and D depths (the ICP options and block by icp_opts).  Refused before anything is queued.
int init_opts(se3tn_ctx* c, const char* fn, const se3tn_init_opts* o, int n, int D, Step& st) {
    const std::string f(fn);
    if (!o) return fail(c, SE3TN_ERR_INVALID, f + ": opts is NULL");
    auto range = [&](int v, int lo, int hi, const char* name) {
        return v >= lo && v <= hi ? SE3TN_OK
                                  : fail(c, SE3TN_ERR_INVALID, f + ": opts->" + name + " is " + std::to_string(v) + ", not in [" +
                                                                   std::to_string(lo) + ", " + std::to_string(hi) + "]");
    };
    int rc;
    if ((rc = range(o->viewpoints, 1, 4096, "viewpoints")) || (rc = range(o->inplane, 1, 360, "inplane")) ||
        (rc = range(o->keep, 1, kInitMaxKeep, "keep")) || (rc = range(o->tau_mm, 1, 1000, "tau_mm")) ||
        (rc = range(o->min_pixels, 1, kImg * kImg, "min_pixels")))
        return rc;
    if (o->reserved) return fail(c, SE3TN_ERR_INVALID, f + ": opts->reserved must be 0");
    const long long VR = static_cast<long long>(o->viewpoints) * o->inplane;
    if (VR > 65536) return fail(c, SE3TN_ERR_INVALID, f + ": opts->viewpoints x opts->inplane = " + std::to_string(VR) + " exceeds 65536");
    if (o->keep > D * VR) return fail(c, SE3TN_ERR_INVALID, f + ": opts->keep exceeds the " + std::to_string(D * VR) + " candidates");
    if (static_cast<long long>(n) * o->keep > c->max_batch)
        return fail(c, SE3TN_ERR_INVALID, f + ": n x opts->keep = " + std::to_string(static_cast<long long>(n) * o->keep) +
                    " exceeds max_batch " + std::to_string(c->max_batch));
    if (!o->icp) return SE3TN_OK;
    DeviceGuard guard(c->device);
    return icp_opts(c, fn, o->icp, st);
}

// Where the pixels of the n objects come from: seg == labels[i] (se3tn_init_poses) or boxes[i] (se3tn_init_boxes, D depths).
struct InitSource {
    const uint8_t* seg; const int32_t* labels;          // HOST labels
    const int32_t* boxes; int D;                        // HOST (n, 4); null with a mask, and D = 1
};

// The stages shared by se3tn_init_poses and se3tn_init_boxes: every check first (nothing queued on a refusal), then the
// launches.  check_object(i) checks object i's label or box.
template <class CheckObject>
int init_run(se3tn_ctx* c, const char* fn, const uint16_t* frame_depth, int H, int W, const double* K, const InitSource& src,
             const double* object_width, int render_mode, int render_H, int render_W, const int32_t* weight_ids_host,
             const int32_t* weight_ids_dev, int n, const se3tn_init_opts* opts, double* poses_out, int32_t* out_rows,
             const se3tn_init_arrays* arrays, void* stream, CheckObject check_object) {
    const std::string f(fn);
    if (!c) return SE3TN_ERR_INVALID;
    // the mask pass counts pixels in 32 bits (mask_finish_kernel's scan): H x W stays below 2^31
    if (!frame_depth || !(src.boxes || (src.seg && src.labels)) || !K || !object_width || H <= 0 || W <= 0 ||
        static_cast<long long>(H) * W >= (1LL << 31))
        return fail(c, SE3TN_ERR_INVALID, f + ": null argument or frame size out of range (H x W must be below 2^31)");
    if (!poses_out || !out_rows) return fail(c, SE3TN_ERR_INVALID, f + ": null output");
    int rc = check_meshes(c, fn, "weight_ids", weight_ids_host, weight_ids_dev, n);
    if (rc) return rc;
    if (src.D < 1 || src.D > kInitMaxDepths)
        return fail(c, SE3TN_ERR_INVALID, f + ": depths is " + std::to_string(src.D) + ", not in [1, " + std::to_string(kInitMaxDepths) + "]");
    RenderSpec r;
    if ((rc = render_spec(c, fn, render_mode, render_H, render_W, r))) return rc;
    Step st{};
    if ((rc = init_opts(c, fn, opts, n, src.D, st))) return rc;
    const se3tn_init_arrays a = arrays ? *arrays : se3tn_init_arrays{};
    const bool icp = opts->icp != nullptr;
    const struct { const void* p; const char* name; } icp_only[] = {{a.icp_poses, "icp_poses"}, {a.icp_rows, "icp_rows"}, {a.icp_stats, "icp_stats"}};
    for (const auto& x : icp_only)
        if (x.p && !icp) return fail(c, SE3TN_ERR_INVALID, f + ": arrays->" + x.name + " is set, but opts->icp is NULL");
    for (int i = 0; i < n; ++i)
        if ((rc = check_object(i))) return rc;
    const size_t nn = static_cast<size_t>(n), D = static_cast<size_t>(src.D), VR = static_cast<size_t>(opts->viewpoints) * opts->inplane;
    const size_t DVR = D * VR, Kk = opts->keep, nK = nn * Kk, px = static_cast<size_t>(H) * W;
    rc = check_disjoint(c, fn, {{poses_out, nn * 128}, {out_rows, nn * 4 * kInitCols}, {a.stats, nn * 8 * kInitStats}, {a.t0, nn * D * 24},
                                {a.cand_rows, nn * DVR * 4 * kInitCols}, {a.kept_rows, nK * 4 * kInitCols}, {a.kept_poses, nK * 128},
                                {a.icp_poses, nK * 128}, {a.icp_rows, nK * 4 * kInitCols}, {a.icp_stats, nK * 8 * kIcpCols}},
                        {{frame_depth, px * 2}, {src.seg, src.seg ? px : 0}, {object_width, nn * 8}, {weight_ids_dev, nn * 4}},
                        src.boxes ? "the outputs must not overlap frame_depth, object_width or weight_ids_dev"
                                  : "the outputs must not overlap frame_depth, seg, object_width or weight_ids_dev");
    if (rc || n == 0) return rc;

    DeviceGuard guard(c->device);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if ((rc = sync_meshes(c, s))) return rc;
    const InitLayout L(nn, D, VR, Kk, static_cast<size_t>(c->max_batch));
    if (L.bytes > c->init_bytes) {                       // the old block may still be read by a queued call
        CU_TRY(c, cudaStreamSynchronize(s));
        CU_TRY(c, grow(c->init, c->init_bytes, L.bytes));
    }
    uint8_t* b = c->init.get();
    auto at = [b](size_t off) { return static_cast<void*>(b + off); };
    int32_t* d_src = static_cast<int32_t*>(at(L.labels));   // the labels or the boxes
    long long* stats = a.stats ? reinterpret_cast<long long*>(a.stats) : static_cast<long long*>(at(L.stats));
    double* t0 = a.t0 ? a.t0 : static_cast<double*>(at(L.t0));
    double* grid = static_cast<double*>(at(L.grid));
    double* gwidth = static_cast<double*>(at(L.width));
    int32_t* gids = weight_ids_dev ? static_cast<int32_t*>(at(L.ids)) : nullptr;
    int32_t* rows = a.cand_rows ? a.cand_rows : static_cast<int32_t*>(at(L.rows));
    uint16_t* depth = static_cast<uint16_t*>(at(L.depth));
    int32_t* kept_rows = a.kept_rows ? a.kept_rows : static_cast<int32_t*>(at(L.kept_rows));
    double* kept_poses = a.kept_poses ? a.kept_poses : static_cast<double*>(at(L.kept_poses));
    double* kept_width = static_cast<double*>(at(L.kept_width));
    int32_t* kept_ids = weight_ids_dev ? static_cast<int32_t*>(at(L.kept_ids)) : nullptr;
    double* icp_poses = a.icp_poses ? a.icp_poses : static_cast<double*>(at(L.icp_poses));
    int32_t* icp_rows = a.icp_rows ? a.icp_rows : static_cast<int32_t*>(at(L.icp_rows));
    double* icp_stats = a.icp_stats ? a.icp_stats : static_cast<double*>(at(L.icp_stats));
    c->launches = 0;

    // 1. mask or box statistics and t0
    const int32_t* d_labels = src.boxes ? nullptr : d_src;
    const int32_t* d_boxes = src.boxes ? d_src : nullptr;
    CU_TRY(c, cudaMemcpyAsync(d_src, src.boxes ? src.boxes : src.labels, nn * (src.boxes ? 4 : 1) * sizeof(int32_t), cudaMemcpyHostToDevice, s));
    MaskArgs ma{};
    ma.depth = frame_depth; ma.seg = src.seg; ma.H = H; ma.W = W; ma.labels = d_labels; ma.boxes = d_boxes; ma.D = src.D; ma.n = n;
    for (int i = 0; src.boxes && i < n; ++i) {
        const int32_t* bx = src.boxes + 4 * i;
        ma.box_px_max = std::max(ma.box_px_max, static_cast<long long>(bx[2] - bx[0]) * (bx[3] - bx[1]));
    }
    ma.acc = static_cast<unsigned long long*>(at(L.acc)); ma.hist = static_cast<unsigned*>(at(L.hist)); ma.min_pixels = opts->min_pixels;
    ma.fx = K[0]; ma.fy = K[1]; ma.cx = K[2]; ma.cy = K[3]; ma.stats = stats; ma.t0 = t0;
    CU_TRY(c, launch_mask_stats(ma, s));
    c->launches += 2;
    // 2. the rotation grid at each t0_d
    GridArgs ga{};
    ga.n = n; ga.V = opts->viewpoints; ga.R = opts->inplane; ga.D = src.D; ga.t0 = t0; ga.width_in = object_width; ga.ids_in = weight_ids_dev;
    ga.poses = grid; ga.width = gwidth; ga.ids = gids;
    CU_TRY(c, launch_grid(ga, s));
    ++c->launches;
    // 3. render and score in chunks of max_batch rows: each render waits (PDL) for the score before it, which read the chunk
    // depth it overwrites
    ScoreArgs sa{};
    sa.object_width = gwidth; sa.fx = K[0]; sa.fy = K[1]; sa.cx = K[2]; sa.cy = K[3];
    sa.frame_depth = frame_depth; sa.seg = src.seg; sa.H = H; sa.W = W; sa.rendered = depth; sa.labels = d_labels; sa.boxes = d_boxes;
    sa.stats = stats; sa.tau = opts->tau_mm;
    const size_t total = nn * DVR;
    for (size_t g0 = 0; g0 < total; g0 += c->max_batch) {
        const int m = static_cast<int>(std::min(total - g0, static_cast<size_t>(c->max_batch)));
        const RenderArgs ra = render_args(c, K, grid + 16 * g0, gwidth + g0, gids ? gids + g0 : nullptr, r.mode, r.H, r.W, nullptr, depth);
        CU_TRY(c, launch_render(ra, m, s));
        sa.poses = grid; sa.row0 = static_cast<int>(g0); sa.per_object = static_cast<int>(DVR); sa.rows = rows;
        CU_TRY(c, launch_score(sa, m, s));
        c->launches += 3;
    }
    // 4. keep the K best of each object
    KeepArgs ka{};
    ka.n = n; ka.per_object = static_cast<int>(DVR); ka.K = opts->keep; ka.rows = rows; ka.poses = grid; ka.width_in = object_width;
    ka.ids_in = weight_ids_dev; ka.kept_rows = kept_rows; ka.kept_poses = kept_poses; ka.kept_width = kept_width; ka.kept_ids = kept_ids;
    CU_TRY(c, launch_keep(ka, s));
    ++c->launches;
    // 5. ICP on the n K kept poses as n K tracks, then each rescored where it landed
    ChooseArgs ca{};
    ca.n = n; ca.K = opts->keep; ca.rows = kept_rows; ca.poses = kept_poses; ca.stats = stats; ca.poses_out = poses_out; ca.rows_out = out_rows;
    if (icp) {
        const int nk = static_cast<int>(nK);
        CU_TRY(c, cudaMemcpyAsync(icp_poses, kept_poses, nK * 16 * sizeof(double), cudaMemcpyDeviceToDevice, s));
        RenderArgs ra = render_args(c, K, icp_poses, kept_width, kept_ids, r.mode, r.H, r.W, nullptr, icp_depth(c));
        ra.tri = icp_tri(c);
        IcpArgs ia{};
        ia.poses = icp_poses; ia.object_width = kept_width; ia.mesh_ids = kept_ids; ia.meshes = c->d_meshes.get(); ia.n_meshes = c->mesh_rows;
        ia.fx = K[0]; ia.fy = K[1]; ia.cx = K[2]; ia.cy = K[3]; ia.frame_depth = frame_depth; ia.H = H; ia.W = W; ia.tri = icp_tri(c);
        ia.tau = st.icp.tau; ia.min_inliers = st.icp.min_inliers; ia.sums = icp_sums(c); ia.stats = icp_stats;
        for (int it = 0; it < st.icp.iterations; ++it) {
            CU_TRY(c, launch_render(ra, nk, s));
            CU_TRY(c, launch_icp(ia, nk, s));
            c->launches += 4;
        }
        const RenderArgs rs = render_args(c, K, icp_poses, kept_width, kept_ids, r.mode, r.H, r.W, nullptr, depth);
        CU_TRY(c, launch_render(rs, nk, s));
        ScoreArgs sr = sa;
        sr.poses = icp_poses; sr.object_width = kept_width; sr.row0 = 0; sr.per_object = opts->keep; sr.cand_rows = kept_rows;
        sr.fixed_delta = 1; sr.rows = icp_rows;
        CU_TRY(c, launch_score(sr, nk, s));
        c->launches += 3;
        ca.rows = icp_rows; ca.poses = icp_poses;
    }
    // 6. the best of each object's K
    CU_TRY(c, launch_choose(ca, s));
    ++c->launches;
    return SE3TN_OK;
}
}  // namespace

extern "C" {

int se3tn_init_poses(se3tn_ctx* c, const uint16_t* frame_depth, const uint8_t* seg, int H, int W, const double* K,
                     const int32_t* labels, const double* object_width, int render_mode, int render_H, int render_W,
                     const int32_t* weight_ids_host, const int32_t* weight_ids_dev, int n, const se3tn_init_opts* opts,
                     double* poses_out, int32_t* out_rows, const se3tn_init_arrays* arrays, void* stream) {
    const char* fn = "se3tn_init_poses";
    const InitSource src{seg, labels, nullptr, 1};
    return init_run(c, fn, frame_depth, H, W, K, src, object_width, render_mode, render_H, render_W, weight_ids_host, weight_ids_dev,
                    n, opts, poses_out, out_rows, arrays, stream, [&](int i) -> int {
                        if (labels[i] >= 1 && labels[i] <= 255) return SE3TN_OK;
                        return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": labels[" + std::to_string(i) + "] is " +
                                                              std::to_string(labels[i]) + ", not in [1, 255]");
                    });
}

int se3tn_init_boxes(se3tn_ctx* c, const uint16_t* frame_depth, int H, int W, const double* K, const int32_t* boxes, int depths,
                     const double* object_width, int render_mode, int render_H, int render_W, const int32_t* weight_ids_host,
                     const int32_t* weight_ids_dev, int n, const se3tn_init_opts* opts, double* poses_out, int32_t* out_rows,
                     const se3tn_init_arrays* arrays, void* stream) {
    const char* fn = "se3tn_init_boxes";
    const InitSource src{nullptr, nullptr, boxes, depths};
    return init_run(c, fn, frame_depth, H, W, K, src, object_width, render_mode, render_H, render_W, weight_ids_host, weight_ids_dev,
                    n, opts, poses_out, out_rows, arrays, stream, [&](int i) -> int {
                        const int32_t* b = boxes + 4 * i;
                        if (b[0] >= 0 && b[1] >= 0 && b[2] <= W && b[3] <= H && b[2] >= b[0] && b[3] >= b[1]) return SE3TN_OK;
                        return fail(c, SE3TN_ERR_INVALID, std::string(fn) + ": boxes[" + std::to_string(i) + "] = (" +
                                    std::to_string(b[0]) + ", " + std::to_string(b[1]) + ", " + std::to_string(b[2]) + ", " +
                                    std::to_string(b[3]) + ") is not a box inside the frame (0 <= x0 <= x1 <= W = " + std::to_string(W) +
                                    ", 0 <= y0 <= y1 <= H = " + std::to_string(H) + ")");
                    });
}

}  // extern "C"

namespace {
static_assert(sizeof(se3tn_reinit_opts) == 16, "se3tn_reinit_opts is 16 bytes without padding: _lib.ReinitOpts mirrors it");
static_assert(kReinitNone == SE3TN_REINIT_NONE && kReinitBelow == SE3TN_REINIT_BELOW && kReinitRestarted == SE3TN_REINIT_RESTARTED &&
              kReinitNoStart == SE3TN_REINIT_NO_START && kReinitRejected == SE3TN_REINIT_REJECTED, "include/se3tn.h");
}  // namespace

extern "C" {

int se3tn_lost_tracks(se3tn_ctx* c, const int32_t* fit_rows, int n, const se3tn_reinit_opts* opts, int32_t* streak,
                      int32_t* out_event, int32_t* out_lost, void* stream) {
    const std::string f("se3tn_lost_tracks");
    if (!c) return SE3TN_ERR_INVALID;
    if (!fit_rows || !opts || !streak || !out_event || !out_lost) return fail(c, SE3TN_ERR_INVALID, f + ": null argument");
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, f + ": n is " + std::to_string(n) + ", not in [0, max_batch]");
    const struct { int v; const char* name; } fields[] = {{opts->below_permille, "below_permille"}, {opts->after, "after"}};
    for (const auto& x : fields)
        if (x.v < 1 || x.v > 1000)
            return fail(c, SE3TN_ERR_INVALID, f + ": opts->" + x.name + " is " + std::to_string(x.v) + ", not in [1, 1000]");
    if (opts->reserved[0] || opts->reserved[1]) return fail(c, SE3TN_ERR_INVALID, f + ": opts->reserved must be 0");
    const size_t nn = static_cast<size_t>(n);
    const int rc = check_disjoint(c, f.c_str(), {{streak, nn * 4}, {out_event, nn * 4}, {out_lost, (nn + 1) * 4}},
                                  {{fit_rows, nn * 4 * kFitCols}}, "the outputs must not overlap fit_rows");
    if (rc) return rc;
    DeviceGuard guard(c->device);
    LostArgs a{};
    a.fit_rows = fit_rows; a.n = n; a.below_permille = opts->below_permille; a.after = opts->after;
    a.streak = streak; a.event = out_event; a.lost = out_lost;
    CU_TRY(c, launch_lost(a, static_cast<cudaStream_t>(stream)));
    c->launches = 1;
    return SE3TN_OK;
}

int se3tn_fit_poses(se3tn_ctx* c, const uint16_t* frame_depth, int H, int W, const double* K, const double* poses,
                    const double* object_width, int render_mode, int render_H, int render_W, const int32_t* weight_ids_host,
                    const int32_t* weight_ids_dev, int n, int fit_tau_mm, int32_t* out_rows, void* stream) {
    const char* fn = "se3tn_fit_poses";
    const std::string f(fn);
    if (!c) return SE3TN_ERR_INVALID;
    if (!frame_depth || !K || !poses || !object_width || !out_rows || H <= 0 || W <= 0)
        return fail(c, SE3TN_ERR_INVALID, f + ": null argument or empty frame");
    int rc = check_meshes(c, fn, "weight_ids", weight_ids_host, weight_ids_dev, n);
    if (rc) return rc;
    if (fit_tau_mm < 1 || fit_tau_mm > 1000)
        return fail(c, SE3TN_ERR_INVALID, f + ": fit_tau_mm is " + std::to_string(fit_tau_mm) + ", not in [1, 1000]");
    RenderSpec r;
    if ((rc = render_spec(c, fn, render_mode, render_H, render_W, r))) return rc;
    const size_t nn = static_cast<size_t>(n);
    rc = check_disjoint(c, fn, {{out_rows, nn * 4 * kFitCols}},
                        {{frame_depth, static_cast<size_t>(H) * W * 2}, {poses, nn * 128}, {object_width, nn * 8}, {weight_ids_dev, nn * 4}},
                        "out_rows must not overlap an input");
    if (rc || n == 0) return rc;
    DeviceGuard guard(c->device);
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if ((rc = sync_meshes(c, s))) return rc;
    const size_t bytes = nn * kImg * kImg * sizeof(uint16_t);
    if (bytes > c->fit_poses_bytes) {                    // the old block may still be read by a queued call
        CU_TRY(c, cudaStreamSynchronize(s));
        CU_TRY(c, grow(c->fit_poses, c->fit_poses_bytes, bytes));
    }
    uint16_t* depth = reinterpret_cast<uint16_t*>(c->fit_poses.get());
    // the step's fit check (step_launches), as plain launches at the given poses
    const RenderArgs ra = render_args(c, K, poses, object_width, weight_ids_dev, r.mode, r.H, r.W, nullptr, depth);
    CU_TRY(c, launch_render(ra, n, s, false));
    FitArgs fa;
    fa.poses = poses; fa.object_width = object_width; fa.fx = K[0]; fa.fy = K[1]; fa.cx = K[2]; fa.cy = K[3];
    fa.frame_depth = frame_depth; fa.H = H; fa.W = W; fa.rendered = depth; fa.tau = fit_tau_mm; fa.rows = out_rows;
    CU_TRY(c, launch_fit(fa, n, s));
    c->launches = 3;
    return SE3TN_OK;
}

int se3tn_accept_starts(se3tn_ctx* c, const int32_t* lost_idx_host, const int32_t* lost_idx_dev, int m, const double* starts,
                        const int32_t* init_rows, const int32_t* start_fit, int n, double* poses, int32_t* fit_rows, int32_t* streak,
                        int32_t* out_event, void* stream) {
    const std::string f("se3tn_accept_starts");
    if (!c) return SE3TN_ERR_INVALID;
    if (n < 0 || n > c->max_batch) return fail(c, SE3TN_ERR_INVALID, f + ": n is " + std::to_string(n) + ", not in [0, max_batch]");
    if (m < 0 || m > n) return fail(c, SE3TN_ERR_INVALID, f + ": m is " + std::to_string(m) + ", not in [0, n]");
    if (m > 0 && (!lost_idx_host || !lost_idx_dev || !starts || !init_rows || !start_fit || !poses || !fit_rows || !streak || !out_event))
        return fail(c, SE3TN_ERR_INVALID, f + ": null argument");
    std::vector<char> seen(static_cast<size_t>(n), 0);
    for (int k = 0; k < m; ++k) {
        const int i = lost_idx_host[k];
        if (i < 0 || i >= n)
            return fail(c, SE3TN_ERR_INVALID, f + ": lost_idx[" + std::to_string(k) + "] is " + std::to_string(i) + ", not in [0, n)");
        if (seen[i]) return fail(c, SE3TN_ERR_INVALID, f + ": lost_idx[" + std::to_string(k) + "] repeats track " + std::to_string(i));
        seen[i] = 1;
    }
    const size_t nn = static_cast<size_t>(n), mm = static_cast<size_t>(m);
    const int rc = check_disjoint(c, f.c_str(), {{poses, nn * 128}, {fit_rows, nn * 4 * kFitCols}, {streak, nn * 4}, {out_event, nn * 4}},
                                  {{lost_idx_dev, mm * 4}, {starts, mm * 128}, {init_rows, mm * 4 * kInitCols}, {start_fit, mm * 4 * kFitCols}},
                                  "the in-place outputs must not overlap an input");
    if (rc) return rc;
    c->launches = 0;
    if (m == 0) return SE3TN_OK;
    DeviceGuard guard(c->device);
    AcceptArgs a{};
    a.lost_idx = lost_idx_dev; a.m = m; a.starts = starts; a.init_rows = init_rows; a.start_fit = start_fit;
    a.poses = poses; a.fit_rows = fit_rows; a.streak = streak; a.event = out_event;
    CU_TRY(c, launch_accept(a, static_cast<cudaStream_t>(stream)));
    c->launches = 1;
    return SE3TN_OK;
}

}  // extern "C"
