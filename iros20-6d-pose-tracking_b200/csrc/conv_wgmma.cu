// wgmma implicit-GEMM convolutions of the se(3)-TrackNet conv stack (reference se3_tracknet.py:57-78,
// network_modules.py:59-66,86-120), im2col-free: D[pixels, Cout] = sum_tap sum_c A_tap[pixel, c] * W[Cout, tap*Cin + c].
//
// Common to both kernels
//   * M tile = an 11x11 pixel box of one image (121 of 128 rows; 44, 22 and 11 are multiples of 11), as two wgmma M = 64
//     halves.  Accumulators stay in registers.
//   * A operand by TMA "units" (load_a_units): one cp.async.bulk.tensor.4d per (128-byte channel chunk, filter COLUMN) whose
//     box is two rows taller than the tile.  It lands as 143 rows x 128 B in the SWIZZLE_128B K-major layout wgmma reads, and
//     the three vertical taps of that column are the SAME tile read through descriptors whose start address is advanced
//     by whole pixel rows (11 * 128 B; the swizzle is a function of absolute address bits) -- no data moves.
//     Out-of-image coordinates are zero-filled by TMA = the conv padding.  Stride-2 convs: six units per chunk over four
//     parity views of the input.  Stem (7x7 s2, Cin = 4): two units (even / odd input rows) of an overlapping 8-pixel-window
//     view; the 7 filter rows are row shifts 0/11/22/33.
//   * warp roles (384 threads = 3 warpgroups): warp 0 activation TMA producer (+ work scheduler in the trunk kernel),
//     warp 1 weight TMA producer, warps 2-3 idle; warpgroups 1 and 2 issue the MMAs and run the epilogue from registers.
//     Operands pass through mbarrier rings (Ring).  A consumer warpgroup keeps one MMA group in flight and hands an operand
//     stage back once the group after it has been issued (wgmma.wait_group 1).
//   * ping-pong (the trunk always, the resident kernel in launches with more tiles than SMs): consumer warpgroup g owns the
//     CTA's tiles / work units it % 2 == g, both 64-row halves, and issues each MMA step once per half, in the same K order
//     as with one warpgroup per half: bit-identical results.  The two take turns issuing MMAs (Turn): a warpgroup starts its
//     tile's MMAs once the other has ISSUED all of its previous tile's, so one warpgroup's epilogue runs under the other's
//     MMAs.  Both walk every operand ring; the one that does not own a tile steps its positions past the tile's stages.
//   * registers: a whole-tile accumulator takes up to 128 registers per consumer thread; setmaxnreg moves them from the
//     producer warpgroup (168 at launch -> 40) to the consumers (-> 232).
//   * PREC (an SE3TN_PREC_* value) selects arithmetic and storage (storage.cuh): TF32 (4 x k8 tf32 MMAs per chunk-tap),
//     BF16X3 (x = hi + lo as two bf16, 3 products per MAC: fp32-faithful), BF16 (2-byte activations, 1 product), FP8 (the
//     trunk on e4m3 codes, 4 x k32 MMAs per chunk-tap; epilogue acc * mul[co] + bias (+ residual code * s_res), then the
//     code of y / s_out; in the resident kernel FP8 means the bf16 layer that writes CAT as e4m3), FP16 (2-byte fp16
//     activations and weights, 1 product, f16 k16 MMAs; its stems run the bf16x3 arithmetic and store fp16).
//   * programmatic dependent launch: every CTA signals launch_dependents at entry; only the threads that touch
//     activations execute griddepcontrol.wait, so barrier init and the weight TMA run under the previous kernel's tail.
//   * per-object weights (reference README.md:132: one checkpoint per object class): with img_wid every work unit takes
//     its weight tensor map and bias from per-set device tables, so all tracks of a frame share the launches.
//
// conv_resident_kernel<KIND, PREC, PP>  (Cout = 64: stems, 64-channel 3x3 convs)
//   * the whole K-major weight matrix (<= 147 KB) is TMA-loaded into shared memory once per CTA (again only when the
//     weight-set id changes between consecutive tiles of the CTA's contiguous range), one mbarrier per filter-column
//     unit so the first MMAs start when the first third has landed.
//   * in the bf16 hi/lo modes the weight halves are STACKED along N: rows [w_hi ; w_lo] -> one N = 128 MMA forms
//     a_hi*w_hi and a_hi*w_lo, one N = 64 MMA adds a_lo*w_hi into the first half, the epilogue sums the two column halves
//     (4 instead of 6 MMAs per chunk-tap; the stem's [w_hi|w_hi ; w_lo|0] rows give all three products in one N = 128 MMA
//     per K step).  The accumulator is then 128 registers, otherwise 64.
//   * 64-channel layers keep their weight ROWS permuted (column 8j + 2m + e of a 32-column block carries channel
//     8m + 2j + e, se3tn.cu) so that in the wgmma accumulator fragment each thread owns 8 consecutive channels of a pixel:
//     16-byte pieces, no staging.
//   * stem: fused MaxPool2d(3,2,1): the M tile is the 11x11 block of conv outputs that feeds a 5x5 block of pooled
//     outputs; max -> +bias -> SELU (monotone, so they commute) on 1/4.84 of the values; the 88x88x64 conv output never
//     reaches HBM.  The fp32 sums are staged in shared memory for the 3x3 max.
//   * PP = false: the halves schedule (each consumer warpgroup one half of every tile) for launches where no CTA has a
//     second tile.  PP = true: ping-pong; an A stage then has one reader (a_empty: one arrival).  Both warpgroups track the
//     weight generation, and at a weight-set switch each arrives on b_empty once its own MMAs on the old weights have
//     retired.  The stem's epilogue runs on the owning 128 threads (warpgroup-local named barriers); in bf16 / bf16x3 its
//     one staging buffer (a second does not fit next to the resident weights) passes between the warpgroups as a second
//     Turn, in tf32 warpgroup g keeps buffer g.  The stem's bias is loaded before the MMAs.  In the 64-channel bf16x3
//     layers the second half's residual loads wait until the first half's epilogue has freed its accumulator registers.
//
// conv_trunk_kernel<PREC>  (Cout >= 256: convAB1, convAB2.{conv1,conv2}, {trans,rot}_conv1, {trans,rot}_conv2.{conv1,conv2})
//   * ONE launch for all six layers.  A work unit = (layer, image, 11x11 tile, 128 output channels).  A persistent CTA per
//     SM pulls the next unit from a global counter (layer-major, image-major order) when its producer has issued the last
//     loads of the current one, and a unit of layer l first waits until done[l-1][image] says that image's previous-layer
//     output is complete (release/acquire at gpu scope; the waits point backwards in the pull order and all CTAs are
//     co-resident, so the schedule cannot deadlock).  Every role walks the same ring of pulled units.
//   * the 128 x 128 fp32 accumulator is 128 registers per consumer thread.
//   * weights stream through a 6-stage ring of {32 words, 128 rows} tiles fed by their own producer warp.
//   * epilogue: each warp post-processes 32 rows (a 16-row slice of each half, one after the other); every 16-row x 32-column
//     accumulator block is transposed through a per-warp shared-memory tile so every global load / store instruction covers
//     whole lines; the last layer reduces its 121 rows to per-slice column sums instead (AdaptiveAvgPool2d(1) fused; eight
//     16-row slices, fixed order -> deterministic).
#include "conv_common.h"
#include "launch.h"
#include "ptx.cuh"
#include "storage.cuh"
#include <algorithm>

namespace se3tn {
namespace {

constexpr int kThreads2 = 384;                 // warpgroup 0: warp 0 A-TMA, warp 1 B-TMA; warpgroups 1, 2: MMA + epilogue
constexpr int kPoolPitch = 68;                 // floats per staged conv position (64 + 4: bank spread)
constexpr int kPoolStageBytes = 121 * kPoolPitch * 4;
constexpr int kPoolStageAlloc = (kPoolStageBytes + 1023) & ~1023;
constexpr int kWgRowBytes = 64 * kChunkBytes;  // the second 64-row half of a tile starts 64 rows into an A unit

// Compile-time unit / tap structure per conv kind, so the MMA issue loop is straight-line code with immediate row
// shifts / weight-tile indices, and the TMA producer's box coordinates are immediates too.  kAUnit: bytes of an A ring stage.
template <int KIND> struct KTab;
template <> struct KTab<KIND_S1> {            // 3x3 stride 1: unit = filter column s, taps = filter rows r
    static constexpr int NU = 3;
    static constexpr int kAUnit = 19 * 1024;   // (22 + 128) rows * 128 B = 19,200
    __host__ __device__ static constexpr int ntaps(int) { return 3; }
    __host__ __device__ static constexpr int wtap(int u, int k) { return k * 3 + u; }
    __host__ __device__ static constexpr int amap(int) { return 0; }
    __host__ __device__ static constexpr int c1(int u) { return u - 1; }
    __host__ __device__ static constexpr int c2(int) { return -1; }
    __host__ __device__ static constexpr int rows(int) { return 11 * 13; }
};
template <> struct KTab<KIND_S2> {            // 3x3 stride 2: per column s an even-row unit (r=1) and an odd-row unit (r=0,2)
    static constexpr int NU = 6;
    static constexpr int kAUnit = 19 * 1024;   // as stride 1: the trunk's A ring serves both
    __host__ __device__ static constexpr int ntaps(int u) { return (u & 1) ? 2 : 1; }
    __host__ __device__ static constexpr int wtap(int u, int k) { return (u & 1) ? (k == 0 ? (u >> 1) : 6 + (u >> 1)) : 3 + (u >> 1); }
    // iy = 2*oy + dy: dy = -1 -> odd row oy-1; dy = 0 -> even row oy; dy = +1 -> odd row oy; columns likewise
    __host__ __device__ static constexpr int amap(int u) { return (u & 1) * 2 + ((u >> 1) == 1 ? 0 : 1); }
    __host__ __device__ static constexpr int c1(int u) { return (u >> 1) == 0 ? -1 : 0; }
    __host__ __device__ static constexpr int c2(int u) { return (u & 1) ? -1 : 0; }
    __host__ __device__ static constexpr int rows(int u) { return (u & 1) ? 11 * 12 : 11 * 11; }
};
template <> struct KTab<KIND_STEM> {          // 7x7 stride 2 stem: even input rows (r=0,2,4,6), odd input rows (r=1,3,5)
    static constexpr int NU = 2;
    static constexpr int kAUnit = 21 * 1024;   // (33 + 128) rows * 128 B = 20,608
    __host__ __device__ static constexpr int ntaps(int u) { return u == 0 ? 4 : 3; }
    __host__ __device__ static constexpr int wtap(int u, int k) { return 2 * k + u; }
    __host__ __device__ static constexpr int amap(int u) { return u; }
    __host__ __device__ static constexpr int c1(int) { return 0; }
    __host__ __device__ static constexpr int c2(int) { return 0; }
    __host__ __device__ static constexpr int rows(int u) { return u == 0 ? 11 * 14 : 11 * 13; }
};
constexpr int kRowShift = 11;                  // rows a descriptor advances per vertical tap (tile width)

__device__ __forceinline__ float selu_fast(float x) {
    constexpr float kAlpha = 1.6732632423543772f, kScale = 1.0507009873554805f;
    return x > 0.f ? kScale * x : (kScale * kAlpha) * (__expf(x) - 1.f);
}
__device__ __forceinline__ float act_apply(float x, int act) {
    return act == ACT_RELU ? fmaxf(x, 0.f) : (act == ACT_SELU ? selu_fast(x) : x);
}

// timeline stamps (debug): slot 0 kernel entry, 1 setup done, 2 first consumer has its first weights, 3 first consumer has its
// first A unit, 4 first consumer issued its last MMA, 5 first consumer's first accumulator is complete, 6 first consumer finished
// its last tile, 7 CTA exit (low 8 bits: SM id)
__device__ __forceinline__ unsigned long long gtimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ void trace_stamp(unsigned long long* tr, int slot) { if (tr) tr[blockIdx.x * 8 + slot] = gtimer(); }
__device__ __forceinline__ void trace_exit(unsigned long long* tr) {
    if (!tr) return;
    unsigned smid; asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    tr[blockIdx.x * 8 + 7] = (gtimer() & ~0xffull) | (smid & 0xff);
}
// per-tile timeline of a resident launch (SE3TN_TRACE, tiles < SE3TN_TRACE_TILES): 4 stamps per tile, written by the first thread
// of the warpgroup that owns the tile (of warpgroup 0 in the halves schedule): 0 first A unit landed (after the MMA turn came),
// 1 last MMA completed, 2 accumulator handed to the epilogue, 3 that thread finished its epilogue (low 8 bits: CTA index)
__device__ __forceinline__ void tile_stamp(unsigned long long* tt, int tile, int k) {
    if (tt && tile < SE3TN_TRACE_TILES) tt[tile * 4 + k] = k == 3 ? (gtimer() & ~0xffull) | (blockIdx.x & 0xff) : gtimer();
}

using ptx::desc_lo;
using ptx::mk_desc;

// The first 32 accumulator registers (columns 0..63) of a 64-register (N = 128) accumulator
__device__ __forceinline__ float (&acc_lo32(float (&d)[64]))[32] { return *reinterpret_cast<float (*)[32]>(&d[0]); }

// Consumer thread coordinates: warpgroup cg owns tile rows [64 cg, 64 cg + 64); warp cw of it rows 16 cw + [0, 16);
// lane (R = lane / 4, m = lane % 4) holds rows 16 cw + R + 8h (h < 2) of the wgmma fragment.
struct Consumer {
    int ct, cg, cw, ew, lane, R, m;
    __device__ __forceinline__ Consumer() {
        ct = static_cast<int>(threadIdx.x) - 128; cg = ct >> 7; ew = ct >> 5; cw = ew & 3; lane = ct & 31; R = lane >> 2; m = lane & 3;
    }
    __device__ __forceinline__ bool leader() const { return (ct & 127) == 0; }   // arrives on the operand-release barriers
    __device__ __forceinline__ int row(int half, int h) const { return 64 * half + 16 * cw + R + 8 * h; }   // in 64-row half `half`
};

// registers per thread after setmaxnreg: the producer warpgroup gives up what the consumers' 128 accumulators need
// (launch: 168 x 384 threads; after: 40 x 128 + 232 x 256 = the same 64,512)
constexpr int kProducerRegs = 40;
constexpr int kConsumerRegs = 232;
// named barriers (0 is __syncthreads): ping-pong MMA turn, the resident stem's staging-buffer hand-over, warpgroup-local epilogue
constexpr int kTurnBar = 1;                    // kTurnBar + g: consumer warpgroup g may issue its tile's / unit's MMAs
constexpr int kStageBar = 3;                   // kStageBar + g: consumer warpgroup g may write the stem's single staging buffer
constexpr int kEpiBar = 5;                     // kEpiBar + g: the 128 threads of warpgroup g (halves schedule: kEpiBar, all 256)

// Position in a ring of N stages, each with a full and an empty mbarrier; phase flips at every wrap.  The producer waits on
// empty[stage] with producer_parity() (its first pass goes straight through), a consumer on full[stage] with consumer_parity().
// A consumer that leaves some stages to another consumer still moves its position past them (skip).
template <int N> struct Ring {
    uint32_t phase = 0;
    int stage = 0;
    __device__ __forceinline__ void next() { if (++stage == N) { stage = 0; phase ^= 1; } }
    __device__ __forceinline__ void skip(int n) {
        stage += n;
        phase ^= static_cast<uint32_t>(stage / N) & 1u;
        stage %= N;
    }
    __device__ __forceinline__ uint32_t producer_parity() const { return phase ^ 1; }
    __device__ __forceinline__ uint32_t consumer_parity() const { return phase; }
};

// Turn-taking of the two consumer warpgroups on the named-barrier pair base + {0, 1}: barrier base + g gives warpgroup g the
// turn.  A turn is one bar.arrive by the warpgroup that passes it and one bar.sync by the one that takes it.  Warpgroup 0 has
// the first turn (begin).  After the last turn has been passed the warpgroup it went to takes it (end), so that neither
// barrier is left with a pending arrival when the CTA exits.
struct Turn {
    int base, g;                               // barrier pair, this consumer warpgroup (0 or 1)
    __device__ __forceinline__ void begin() const { if (g == 1) ptx::bar_arrive(base, 256); }
    __device__ __forceinline__ void wait() const { ptx::bar_sync(base + g, 256); }
    __device__ __forceinline__ void pass() const { ptx::bar_arrive(base + (g ^ 1), 256); }
    __device__ __forceinline__ bool mine(int t) const { return (t & 1) == g; }           // turns alternate, from warpgroup 0
    __device__ __forceinline__ void end(int turns) const { if (mine(turns)) wait(); }      // turns: number of turns passed so far
};

// TMA loads of a tile's A units (producer thread): chunks [c0, c1) x KT::NU filter-column units, one A ring stage each.
// (ox, oy): the tile's box origin in A-map coordinates; cbase: first channel word of the conv group; img: the image.
template <int KIND, int N>
__device__ __forceinline__ void load_a_units(const LayerDesc& L, int ox, int oy, int cbase, int img, int c0, int c1,
                                             uint8_t* sA, uint64_t* a_full, uint64_t* a_empty, Ring<N>& ring)
{
    using KT = KTab<KIND>;
    for (int ch = c0; ch < c1; ++ch) {
#pragma unroll
        for (int u = 0; u < KT::NU; ++u) {
            ptx::mbar_wait(&a_empty[ring.stage], ring.producer_parity());
            ptx::mbar_arrive_expect_tx(&a_full[ring.stage], static_cast<uint32_t>(KT::rows(u)) * kChunkBytes);
            ptx::tma_load_4d(sA + ring.stage * KT::kAUnit, &L.amap[KT::amap(u)], &a_full[ring.stage],
                             cbase + ch * 32, ox + KT::c1(u), oy + KT::c2(u), img);
            ring.next();
        }
    }
}

// The MMAs of one 128-byte K chunk: four K steps of 32 bytes (tf32 k8 with PREC == SE3TN_PREC_TF32, bf16 k16 in the bf16
// modes, f16 k16 in SE3TN_PREC_FP16, e4m3 k32 in SE3TN_PREC_FP8 (trunk only, N = 128)) at N = 64 or 128.  a_lo / b_lo: low
// descriptor words (+2 per K step).  fresh == 0: the first step overwrites acc.
template <int PREC, int N>
__device__ __forceinline__ void mma_chunk(float (&acc)[N / 2], uint32_t a_lo, uint32_t b_lo, uint32_t fresh) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const uint64_t a = mk_desc(a_lo + 2 * kk), b = mk_desc(b_lo + 2 * kk);
        const uint32_t f = fresh | (kk ? 1u : 0u);
        if constexpr (PREC == SE3TN_PREC_TF32) {
            if constexpr (N == 64) ptx::wgmma_tf32_n64(acc, a, b, f); else ptx::wgmma_tf32_n128(acc, a, b, f);
        } else if constexpr (PREC == SE3TN_PREC_FP8) {
            static_assert(N == 128, "e4m3 MMAs only in the trunk");
            ptx::wgmma_e4m3_n128(acc, a, b, f);
        } else if constexpr (PREC == SE3TN_PREC_FP16) {
            if constexpr (N == 64) ptx::wgmma_f16_n64(acc, a, b, f); else ptx::wgmma_f16_n128(acc, a, b, f);
        } else {
            if constexpr (N == 64) ptx::wgmma_bf16_n64(acc, a, b, f); else ptx::wgmma_bf16_n128(acc, a, b, f);
        }
    }
}

// ================================================================================================================
// conv_resident_kernel
// ================================================================================================================
template <int KIND, int PREC> struct RCfg {
    static constexpr bool POOL = (KIND == KIND_STEM);
    static constexpr int BN = 64;
    // STACK: hi / lo weight rows stacked along N (header comment) for layers whose input is in the bf16x3 format
    static constexpr int kStack = ((POOL ? stem_input_prec(PREC) : PREC) == SE3TN_PREC_BF16X3) ? 2 : 1;
    static constexpr int kBTile = BN * kStack * kChunkBytes;
    static constexpr int kAStages = POOL ? (PREC == SE3TN_PREC_TF32 ? 4 : 3) : (prec_2byte(PREC) ? 6 : 4);
    static constexpr int kPoolBufs = POOL ? (PREC == SE3TN_PREC_TF32 ? 2 : 1) : 0;
    static constexpr int kAcc = BN * kStack / 2;                    // accumulator registers per thread (N / 2)
    static constexpr int kMaxWTiles = POOL ? 7 : ((PREC == SE3TN_PREC_TF32) ? 18 : 9);
    static constexpr int kSmem = kAStages * KTab<KIND>::kAUnit + kMaxWTiles * kBTile + kPoolBufs * kPoolStageAlloc + 1024 + 512;
    static_assert(kSmem <= 232448, "shared memory budget");
};

// the MMAs of one (chunk, filter-column unit) of a resident layer: ntaps(u) vertical taps, row shifts of the same A unit
template <int KIND, int PREC>
__device__ __forceinline__ void resident_mma_unit(float (&acc)[RCfg<KIND, PREC>::kAcc], uint32_t a_unit_lo, const uint8_t* sB,
                                                  int u, int ch, int tiles_per_tap, uint32_t& fresh)
{
    using C = RCfg<KIND, PREC>;
    using KT = KTab<KIND>;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (k >= KT::ntaps(u)) break;
        // low descriptor words: +2 per 32-byte K step, +8 per pixel row
        const uint32_t a_lo = a_unit_lo + k * kRowShift * (kChunkBytes >> 4);
        uint32_t b_lo;
        if (C::kStack == 2) b_lo = desc_lo(sB + KT::wtap(u, k) * C::kBTile) + ch * 4;   // chunk ch sits 64 bytes (4 x 16 B) further along K
        else                b_lo = desc_lo(sB + (KT::wtap(u, k) * tiles_per_tap + ch) * C::kBTile);
        if constexpr (C::kStack == 2 && !C::POOL) {
            // chunk = [32 hi | 32 lo] (A); weight rows [w_hi ; w_lo]: a_hi x both (N = 128), then a_lo x w_hi (N = 64, columns 0-63)
#pragma unroll
            for (int sl = 0; sl < 2; ++sl) {
                ptx::wgmma_bf16_n128(acc, mk_desc(a_lo + 2 * sl), mk_desc(b_lo + 2 * sl), fresh | (sl ? 1u : 0u));
                ptx::wgmma_bf16_n64(acc_lo32(acc), mk_desc(a_lo + 4 + 2 * sl), mk_desc(b_lo + 2 * sl), 1u);
            }
        } else {
            // tf32, bf16, fp16, and the stems of the modes with a bf16x3 input: window = 8 pixels x [hi4|lo4] against rows
            // [w_hi|w_hi ; w_lo|0], all three products in one bf16 N = 128 MMA per K step
            mma_chunk<C::POOL ? stem_input_prec(PREC) : PREC, C::BN * C::kStack>(acc, a_lo, b_lo, fresh);
        }
        fresh = 1u;
    }
}

// PP: ping-pong schedule (consumer warpgroup g owns the CTA's tiles it % 2 == g, both 64-row halves); otherwise the halves
// schedule (each consumer warpgroup owns one half of every tile), for launches where no CTA has a second tile to overlap with.
// PREC == SE3TN_PREC_FP8: a 64-channel layer that writes CAT: bf16 operands and arithmetic (AP), the output encoded to e4m3
// with CAT's scale in the epilogue.
template <int KIND, int PREC, bool PP>
__global__ void __launch_bounds__(kThreads2, 1)
conv_resident_kernel(const __grid_constant__ ResidentParams p)
{
    constexpr int AP = resident_prec(PREC);                             // operand format and arithmetic
    static_assert(PREC != SE3TN_PREC_FP8 || KIND == KIND_S1, "e4m3 output: the 64-channel layers only");
    using C = RCfg<KIND, AP>;
    using KT = KTab<KIND>;
    constexpr bool POOL = C::POOL;
    constexpr int NH = PP ? 2 : 1;                                      // 64-row halves of a tile one consumer warpgroup computes
    constexpr bool kShareStage = PP && C::kPoolBufs == 1;               // both warpgroups' stem epilogues use the one staging buffer
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const LayerDesc& L = p.L;
    const int chunks = L.chunks;
    // K tiles of the resident weight matrix: STACK keeps all chunks of a tap in one 128-row tile, otherwise one tile per (tap, chunk)
    const int tiles_per_tap = (C::kStack == 2) ? 1 : chunks;
    uint8_t* sA = smem;                                                 // [kAStages][unit]
    uint8_t* sB = sA + C::kAStages * KT::kAUnit;                        // [num_taps * tiles_per_tap][BN*kStack rows x 128 B]
    uint8_t* sP = sB + C::kMaxWTiles * C::kBTile;                       // pool staging (stem only)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sP + C::kPoolBufs * kPoolStageAlloc);
    uint64_t* a_full = bars;                       // [kAStages]
    uint64_t* a_empty = a_full + C::kAStages;      // [kAStages]: one arrival per consumer warpgroup that reads the stage
    uint64_t* b_full = a_empty + C::kAStages;      // [NU]: weights of filter-column unit u have landed
    uint64_t* b_empty = b_full + KT::NU;           // [1]: MMAs that read the current weights have retired (multi-set reload):
                                                   // one arrival per consumer warpgroup at each weight switch

    ptx::grid_dep_launch();
    if (threadIdx.x == 0) trace_stamp(p.trace, 0);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int tiles_img = L.tiles_x * L.tiles_y;
    // each CTA owns a contiguous range of tiles (consecutive tiles of the same image / weight set)
    const int w_begin = static_cast<int>(static_cast<long long>(blockIdx.x) * p.m_tiles / gridDim.x);
    const int w_end = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * p.m_tiles / gridDim.x);
    auto img_of = [&](int tile) -> int { return p.img_first + tile / tiles_img; };
    auto wid_of = [&](int tile) -> int { return p.img_wid ? p.img_wid[img_of(tile)] : -1; };   // -1: single-set launch

    if (threadIdx.x == 0) {
        for (int s = 0; s < C::kAStages; ++s) { ptx::mbar_init(&a_full[s], 1); ptx::mbar_init(&a_empty[s], PP ? 1 : 2); }
        for (int u = 0; u < KT::NU; ++u) ptx::mbar_init(&b_full[u], 1);
        ptx::mbar_init(&b_empty[0], 2);
        ptx::fence_barrier_init();
        ptx::fence_proxy_async();
    }
    __syncthreads();
    if (threadIdx.x == 0) trace_stamp(p.trace, 1);

    if (warp < 4) {
        ptx::setmaxnreg_dec<kProducerRegs>();       // the whole producer warpgroup, idle warps 2-3 included
        if (warp == 0) {
            // ============================== A producer ================================
            if (lane == 0) {
                ptx::grid_dep_wait();                   // activations come from the previous kernel
                Ring<C::kAStages> ring;
                for (int tile = w_begin; tile < w_end; ++tile) {
                    const int n0 = img_of(tile), r = tile % tiles_img;
                    const int ty = r / L.tiles_x, tx = r - ty * L.tiles_x;
                    load_a_units<KIND>(L, tx * p.step_x + p.off_x, ty * p.step_y + p.off_y, 0, n0, 0, chunks, sA, a_full, a_empty, ring);
                }
            }
        } else if (warp == 1) {
            // ============================== weight loader ================================
            if (lane == 0) {
                int cur = -2; uint32_t gen = 0;
                for (int tile = w_begin; tile < w_end; ++tile) {
                    const int wid = wid_of(tile);
                    if (wid == cur) continue;
                    if (gen) ptx::mbar_wait(&b_empty[0], (gen - 1) & 1);       // MMAs that read the previous weights have retired
                    const CUtensorMap* bm = wid < 0 ? &L.bmap : p.gbmaps + wid * kLayersPerSet + L.li;
#pragma unroll
                    for (int u = 0; u < KT::NU; ++u) {                          // in the order the MMAs need them: unit by unit
                        ptx::mbar_arrive_expect_tx(&b_full[u], static_cast<uint32_t>(KT::ntaps(u) * tiles_per_tap) * C::kBTile);
#pragma unroll
                        for (int k = 0; k < KT::ntaps(u); ++k)
                            for (int c = 0; c < tiles_per_tap; ++c) {
                                const int wt = KT::wtap(u, k) * tiles_per_tap + c;   // tile wt covers K words [wt*32, wt*32 + 32)
                                ptx::tma_load_2d(sB + wt * C::kBTile, bm, &b_full[u], wt * 32, 0);
                            }
                    }
                    cur = wid; ++gen;
                }
            }
        }
    } else {
        // ============================== MMA + epilogue (two warpgroups) ==========================
        ptx::setmaxnreg_inc<kConsumerRegs>();
        ptx::grid_dep_wait();                       // residual reads / output writes must follow the previous kernel
        using S = Storage<AP>;
        const Consumer cs;
        const bool stamp = threadIdx.x == 128;
        const bool tstamp = cs.leader() && (PP || cs.cg == 0);     // per-tile stamps (tile_stamp)
        constexpr int kEpiThreads = PP ? 128 : 256;                 // threads that run one tile's epilogue
        const int et = PP ? (cs.ct & 127) : cs.ct;                  // this thread's index among them
        auto half_of = [&](int hf) { return PP ? hf : cs.cg; };     // 64-row half of the tile in accumulator acc[hf]
        Ring<C::kAStages> a_ring;
        int w_cur = -2; uint32_t w_gen = 0;        // weight set currently in shared memory
        const Turn turn{kTurnBar, cs.cg}, stage_turn{kStageBar, cs.cg};   // one turn per tile of the CTA (PP)
        if constexpr (PP) {
            turn.begin();
            if constexpr (kShareStage) stage_turn.begin();
        }
        int it = 0;
        for (int tile = w_begin; tile < w_end; ++tile, ++it) {
            const int wid = wid_of(tile);
            const bool new_w = (wid != w_cur);     // wait for each unit's weights at its first use below
            const bool w_last = tile + 1 < w_end && wid_of(tile + 1) != wid;   // the loader replaces these weights after this tile
            if (PP && !turn.mine(it)) {
                // the other warpgroup's tile: step this warpgroup's A ring position past its stages.  Keep the weight generation
                // in step, and take part in the hand-back of the weights as below: this warpgroup's MMAs on them retired with its
                // previous tile.  Waiting for a new generation first keeps this warpgroup's arrival for the next switch after
                // the loader has seen both arrivals for this one.
                a_ring.skip(chunks * KT::NU);
                if (new_w) {
#pragma unroll
                    for (int u = 0; u < KT::NU; ++u) ptx::mbar_wait(&b_full[u], w_gen & 1);
                    w_cur = wid; ++w_gen;
                }
                if (w_last && cs.leader()) ptx::mbar_arrive(&b_empty[0]);
                continue;
            }
            const int n0 = img_of(tile), r = tile % tiles_img;
            const int ty = r / L.tiles_x, tx = r - ty * L.tiles_x;

            // 64-channel layers: this thread's pixels and their residual pieces are known before the accumulator is: issue the
            // residual loads now so their latency hides behind the MMAs.  Piece (hf, h, b): row cs.row(half_of(hf), h),
            // channels 32b + 8m .. + 7.  Ping-pong with the 128-register bf16x3 accumulator: only the first half's pieces here,
            // the second half's once the first half's accumulator registers are free (0 spills; their latency then overlaps
            // the first half's epilogue and the other warpgroup's MMAs).
            constexpr int kPreRes = (PP && C::kStack == 2) ? 1 : NH;
            size_t rpix[NH][2]; bool rvalid[NH][2]; Raw<AP, 8> rres[NH][2][2];
            auto load_res = [&](int hf) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int rw = cs.row(half_of(hf), h);
                    const int py = rw / 11, px = rw - py * 11;
                    const int y = ty * 11 + py, x = tx * 11 + px;
                    rvalid[hf][h] = (rw < 121) && (y < L.Ho) && (x < L.Wo);
                    rpix[hf][h] = (static_cast<size_t>(n0) * L.Ho + y) * L.Wo + x;
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        rres[hf][h][b] = Raw<AP, 8>{};
                        if (L.res && rvalid[hf][h]) {
                            const uint8_t* rp = L.res + S::addr(rpix[hf][h], L.res_c, 32 * b + 8 * cs.m);
#pragma unroll
                            for (int q = 0; q < Raw<AP, 8>::kPieces; ++q) rres[hf][h][b].set(q, __ldg(Raw<AP, 8>::at(rp, q)));
                        }
                    }
                }
            };
            if constexpr (!POOL) {
#pragma unroll
                for (int hf = 0; hf < kPreRes; ++hf) load_res(hf);
            }
            // stem: every pooled vector this thread finishes has channels c4 = (et % 16) * 4 (the thread stride is a multiple
            // of 16): its bias is loaded under the MMAs too
            float4 pb4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if constexpr (POOL) pb4 = __ldg(reinterpret_cast<const float4*>((p.img_wid ? p.gbias[p.img_wid[n0] * kLayersPerSet + L.li] : L.bias) + (et & 15) * 4));

            float acc[NH][C::kAcc];
#pragma unroll
            for (int hf = 0; hf < NH; ++hf)
#pragma unroll
                for (int i = 0; i < C::kAcc; ++i) acc[hf][i] = 0.f;
            if constexpr (PP) turn.wait();          // the other warpgroup has issued all MMAs of its previous tile
            uint32_t fresh = 0;                     // 0 until the first MMA of this tile has been issued
            int pend = -1;                          // A stage of the previous MMA group, released once that group has completed
            for (int ch = 0; ch < chunks; ++ch) {
#pragma unroll
                for (int u = 0; u < KT::NU; ++u) {
                    if (new_w && ch == 0) {
                        ptx::mbar_wait(&b_full[u], w_gen & 1);
                        if (it == 0 && u == 0 && stamp) trace_stamp(p.trace, 2);
                    }
                    ptx::mbar_wait(&a_full[a_ring.stage], a_ring.consumer_parity());
                    if (ch == 0 && u == 0) {
                        if (it == 0 && stamp) trace_stamp(p.trace, 3);
                        if (tstamp) tile_stamp(p.tile_trace, tile, 0);
                    }
                    ptx::wgmma_fence();
                    // each MMA step once per 64-row half, every half's accumulator in the same K order
                    const uint32_t a_unit_lo = desc_lo(sA + a_ring.stage * KT::kAUnit);
#pragma unroll
                    for (int hf = 0; hf < NH; ++hf) {
                        uint32_t f = fresh;
                        resident_mma_unit<KIND, AP>(acc[hf], a_unit_lo + half_of(hf) * (kWgRowBytes >> 4), sB, u, ch, tiles_per_tap, f);
                    }
                    fresh = 1u;
                    ptx::wgmma_commit();
                    ptx::wgmma_wait<1>();
                    if (pend >= 0 && cs.leader()) ptx::mbar_arrive(&a_empty[pend]);
                    pend = a_ring.stage;
                    a_ring.next();
                }
            }
            if constexpr (PP) turn.pass();          // all of this tile's MMAs are issued
            ptx::wgmma_wait<0>();
#pragma unroll
            for (int hf = 0; hf < NH; ++hf) ptx::wgmma_reg_fence(acc[hf]);
            if (tstamp) tile_stamp(p.tile_trace, tile, 1);
            if (cs.leader()) {
                ptx::mbar_arrive(&a_empty[pend]);
                // the next tile uses other weights -> tell the loader that these MMAs have retired
                if (w_last) ptx::mbar_arrive(&b_empty[0]);
            }
            if (new_w) { w_cur = wid; ++w_gen; }
            if (it == 0 && stamp) trace_stamp(p.trace, 5);
            if (tstamp) tile_stamp(p.tile_trace, tile, 2);

            if constexpr (!POOL) {
                // ---------------- 64-channel layers ----------------
                // Fragment register 16b + 4jj + 2h + e = row cs.row(half, h), column 32b + 8jj + 2m + e, which carries channel
                // 32b + 8m + 2jj + e (permuted weight rows): the thread owns 8 CONSECUTIVE channels of each of its pixels per
                // 32-column block.
                float inv_out = 1.f;                // SE3TN_PREC_FP8: 1 / CAT's scale (a power of two: exact)
                if constexpr (PREC == SE3TN_PREC_FP8) inv_out = 1.f / __ldg((p.img_wid ? p.gfp8[p.img_wid[n0]] : p.fp8) + L.q_out);
#pragma unroll
                for (int hf = 0; hf < NH; ++hf) {
                    if (hf >= kPreRes) load_res(hf);
#pragma unroll
                    for (int b = 0; b < 2; ++b) {
                        const int ch0 = 32 * b + 8 * cs.m;
                        const float* bias_base = (p.img_wid ? p.gbias[p.img_wid[n0] * kLayersPerSet + L.li] : L.bias) + ch0;
                        const float4 bA = __ldg(reinterpret_cast<const float4*>(bias_base)), bB = __ldg(reinterpret_cast<const float4*>(bias_base + 4));
                        const float bias8[8] = {bA.x, bA.y, bA.z, bA.w, bB.x, bB.y, bB.z, bB.w};
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            if (!rvalid[hf][h]) continue;
                            float v[8];
#pragma unroll
                            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const int ri = 16 * b + 4 * jj + 2 * h + e;
                                    float a = acc[hf][ri];
                                    if constexpr (C::kStack == 2) a += acc[hf][32 + ri];
                                    v[2 * jj + e] = a + bias8[2 * jj + e];
                                }
                            if (L.res) {
                                float r[8];
                                S::decode(rres[hf][h][b], r);
#pragma unroll
                                for (int e = 0; e < 8; ++e) v[e] += r[e];
                            }
#pragma unroll
                            for (int e = 0; e < 8; ++e) v[e] = act_apply(v[e], L.act);
                            if constexpr (PREC == SE3TN_PREC_FP8) {
                                using S8 = Storage<SE3TN_PREC_FP8>;
#pragma unroll
                                for (int e = 0; e < 8; ++e) v[e] *= inv_out;
                                S8::encode(v).store(L.out + S8::addr(rpix[hf][h], L.out_c, L.out_coff + ch0));
                            } else {
                                S::encode(v).store(L.out + S::addr(rpix[hf][h], L.out_c, L.out_coff + ch0));
                            }
                        }
                    }
                }
            } else {
                // ---- stem: conv tile 11x11 -> 5x5 max-pooled outputs (MaxPool2d(3,2,1), -inf padding) ----
                // Ping-pong: with one staging buffer the two warpgroups' epilogues take turns on it (stage_turn); with two, tile
                // it % 2 == g always uses buffer g, and this warpgroup's readers of two tiles ago must be done before it writes.
                float* stage = reinterpret_cast<float*>(sP + (C::kPoolBufs == 2 ? (it & 1) : 0) * kPoolStageAlloc);
                if constexpr (kShareStage) stage_turn.wait();
                else if constexpr (PP) ptx::bar_sync(kEpiBar + cs.cg, 128);
#pragma unroll
                for (int hf = 0; hf < NH; ++hf)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int rw = cs.row(half_of(hf), h);
                        if (rw >= 121) continue;
                        const int cy_l = rw / 11, cx_l = rw - cy_l * 11;            // conv position inside the tile
                        const int cy = ty * p.step_y + p.off_y + cy_l, cx = tx * p.step_x + p.off_x + cx_l;   // conv output coordinates
                        const bool cvalid = cy >= 0 && cy < 88 && cx >= 0 && cx < 88;
                        float* srow = stage + rw * kPoolPitch + 2 * cs.m;
                        const float ninf = -3.0e38f;
#pragma unroll
                        for (int j = 0; j < 8; ++j) {                               // columns 8j + 2m + {0, 1}
                            float a0 = acc[hf][4 * j + 2 * h], a1 = acc[hf][4 * j + 2 * h + 1];
                            if constexpr (C::kStack == 2) { a0 += acc[hf][32 + 4 * j + 2 * h]; a1 += acc[hf][32 + 4 * j + 2 * h + 1]; }
                            *reinterpret_cast<float2*>(srow + 8 * j) = cvalid ? make_float2(a0, a1) : make_float2(ninf, ninf);
                        }
                    }
                ptx::bar_sync(PP ? kEpiBar + cs.cg : kEpiBar, kEpiThreads);    // staging tile complete

                // 25 pooled pixels x 16 float4 channel groups = 400 vectors over the epilogue's threads
                for (int v = et; v < 400; v += kEpiThreads) {
                    const int pp = v >> 4, c4 = (v & 15) * 4;
                    const int ppy = pp / 5, ppx = pp - ppy * 5;
                    const int oy = ty * 5 + ppy, ox = tx * 5 + ppx;     // pooled output coordinates
                    if (oy >= L.Ho || ox >= L.Wo) continue;
                    float4 mx = make_float4(-3.0e38f, -3.0e38f, -3.0e38f, -3.0e38f);
#pragma unroll
                    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                        for (int dx = 0; dx < 3; ++dx) {
                            const float4 s4 = *reinterpret_cast<const float4*>(stage + ((2 * ppy + dy) * 11 + 2 * ppx + dx) * kPoolPitch + c4);
                            mx.x = fmaxf(mx.x, s4.x); mx.y = fmaxf(mx.y, s4.y); mx.z = fmaxf(mx.z, s4.z); mx.w = fmaxf(mx.w, s4.w);
                        }
                    const float v4[4] = {selu_fast(mx.x + pb4.x), selu_fast(mx.y + pb4.y), selu_fast(mx.z + pb4.z), selu_fast(mx.w + pb4.w)};
                    S::encode(v4).store(L.out + S::addr((static_cast<size_t>(n0) * L.Ho + oy) * L.Wo + ox, L.out_c, L.out_coff + c4));
                }
                if constexpr (kShareStage) stage_turn.pass();   // this warpgroup's readers are done
                else if constexpr (!PP) { if (C::kPoolBufs == 1) ptx::bar_sync(kEpiBar, 256); }   // readers done before the next tile writes
            }
            if (tstamp) tile_stamp(p.tile_trace, tile, 3);
        }
        if constexpr (PP) {
            turn.end(it);
            if constexpr (kShareStage) stage_turn.end(it);
        }
        if (stamp) { trace_stamp(p.trace, 4); trace_stamp(p.trace, 6); }
    }

    __syncthreads();
    if (threadIdx.x == 0) trace_exit(p.trace);
}

// ================================================================================================================
// conv_trunk_kernel
// ================================================================================================================
template <int PREC> struct TCfg {
    static constexpr int BN = 128;                                      // output channels per work unit
    static constexpr int kAcc = BN / 2;                                 // accumulator registers per thread and 64-row half of the tile
    static constexpr int kAStages = 3;
    static constexpr int kBStages = 6;
    static constexpr int kBTile = BN * kChunkBytes;                     // 16 KB
    static constexpr int kEpiPitch = 36;                                // words per staged row (32 + 4: conflict-free 16 B accesses)
    static constexpr int kEpiWarpBytes = 16 * kEpiPitch * 4 + 128;      // 16 rows + 32-entry pixel-index table
    static constexpr int kEpiBytes = 8 * kEpiWarpBytes;
    static constexpr int kSched = 4;                                    // work-unit ring between the scheduler (A producer) and the other roles
    static constexpr int kAUnit = KTab<KIND_S1>::kAUnit;               // one A ring for both 3x3 kinds
    static_assert(kAUnit == KTab<KIND_S2>::kAUnit, "A ring stage size");
    static constexpr int kSmem = kAStages * kAUnit + kBStages * kBTile + ((kEpiBytes + 1023) & ~1023) + 1024 + 512;
    static_assert(kSmem <= 232448, "shared memory budget");
};
constexpr int kTaps3 = 9;                      // weight tiles per K chunk of a 3x3 conv (one per filter tap, both strides)

struct UnitCoord { int l, img, tx, ty, n_tile, grp, c0, c1, piece, gidx; };
// per-unit timeline (SE3TN_TRACE, small launches only): 5 stamps per work unit behind the trunk's per-CTA stamps:
// 0 dependency satisfied (producer), 1 first A unit landed (owning consumer warpgroup, after its MMA turn came), 2 last MMA
// completed, 3 accumulator handed to the epilogue, 4 the owning warpgroup's first warp finished (stores + completion signal; low
// 8 bits: CTA index).  Stamps 1-4 are written by the first thread of the owning warpgroup.
__device__ __forceinline__ void unit_stamp(const TrunkParams& p, int u, int k) {
    if (p.trace && u < 2048) p.trace[256 * 8 + u * 5 + k] = k == 4 ? (gtimer() & ~0xffull) | (blockIdx.x & 0xff) : gtimer();
}   // [c0, c1): K chunks of this piece; gidx: unsplit unit index in the launch

__device__ __forceinline__ int unit_layer(const TrunkParams& p, int u) {
    int l = 0;
#pragma unroll
    for (int i = 1; i < kTrunkMaxLayers; ++i) if (i < p.n_layers && u >= p.layer[i].unit_base) l = i;
    return l;
}

__device__ __forceinline__ UnitCoord decode_unit(const TrunkParams& p, int u) {
    UnitCoord c;
    c.l = unit_layer(p, u);
    const LayerDesc& L = p.layer[c.l];
    int local = u - L.unit_base;
    c.piece = 0; c.c0 = 0; c.c1 = L.chunks;
    if (p.ksplit > 1) {                            // consecutive indices = the pieces of one unit (pulled by different CTAs at about the same time)
        c.piece = local % p.ksplit; local /= p.ksplit;
        c.c0 = c.piece * L.chunks / p.ksplit; c.c1 = (c.piece + 1) * L.chunks / p.ksplit;
    }
    c.gidx = L.base_unit0 + local;
    const int im = local / L.units_per_image;
    int r = local - im * L.units_per_image;
    c.img = p.img_first + im;
    c.n_tile = r % L.n_tiles; r /= L.n_tiles;
    c.grp = r % L.groups; r /= L.groups;
    c.ty = r / L.tiles_x; c.tx = r - c.ty * L.tiles_x;
    return c;
}

// weight-tile loads of one work unit (B producer thread)
template <int KIND, int PREC>
__device__ __forceinline__ void trunk_load_weights(const LayerDesc& L, const CUtensorMap* bm, const UnitCoord& c, uint8_t* sB,
                                                   uint64_t* b_full, uint64_t* b_empty, Ring<TCfg<PREC>::kBStages>& ring)
{
    using KT = KTab<KIND>;
    using C = TCfg<PREC>;
    const int wrow = c.grp * L.cout + c.n_tile * C::BN;
    for (int ch = c.c0; ch < c.c1; ++ch) {
#pragma unroll
        for (int u = 0; u < KT::NU; ++u) {
#pragma unroll
            for (int k = 0; k < KT::ntaps(u); ++k) {
                ptx::mbar_wait(&b_empty[ring.stage], ring.producer_parity());
                ptx::mbar_arrive_expect_tx(&b_full[ring.stage], C::kBTile);
                ptx::tma_load_2d(sB + ring.stage * C::kBTile, bm, &b_full[ring.stage], KT::wtap(u, k) * L.cin_words + ch * 32, wrow);
                ring.next();
            }
        }
    }
}

// MMAs of one work unit (one consumer warpgroup, all 128 rows: each MMA step is issued once per 64-row half, into that half's
// accumulator), issued in the warpgroup's turn.  One MMA group per weight tile; a group's weight stage (and, after the last tap
// of a filter column, its A stage) is handed back once the next group has been issued and the group has completed.
template <int KIND, int PREC>
__device__ __forceinline__ void trunk_mma_unit(float (&acc)[2][TCfg<PREC>::kAcc], const Consumer& cs, const Turn& turn, int chunks,
                                               uint8_t* sA, uint8_t* sB, uint64_t* a_full, uint64_t* a_empty, uint64_t* b_full,
                                               uint64_t* b_empty, Ring<TCfg<PREC>::kAStages>& a_ring, Ring<TCfg<PREC>::kBStages>& b_ring,
                                               unsigned long long* trace, bool first_unit, unsigned long long* ustamp)
{
    using KT = KTab<KIND>;
    using C = TCfg<PREC>;
    const bool stamp = cs.leader();
    uint32_t fresh = 0;
    int pend_b = -1, pend_a = -1;
    turn.wait();
    for (int ch = 0; ch < chunks; ++ch) {
#pragma unroll
        for (int u = 0; u < KT::NU; ++u) {
            ptx::mbar_wait(&a_full[a_ring.stage], a_ring.consumer_parity());
            if (first_unit && ch == 0 && u == 0 && stamp) trace_stamp(trace, 3);
            if (ustamp && ch == 0 && u == 0 && stamp) *ustamp = gtimer();
            const uint32_t a_unit_lo = desc_lo(sA + a_ring.stage * C::kAUnit);
#pragma unroll
            for (int k = 0; k < KT::ntaps(u); ++k) {
                ptx::mbar_wait(&b_full[b_ring.stage], b_ring.consumer_parity());
                if (first_unit && ch == 0 && u == 0 && k == 0 && stamp) trace_stamp(trace, 2);
                const uint32_t b_lo = desc_lo(sB + b_ring.stage * C::kBTile);
                ptx::wgmma_fence();
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const uint32_t a_lo = a_unit_lo + hf * (kWgRowBytes >> 4) + k * kRowShift * (kChunkBytes >> 4);
                    if constexpr (PREC == SE3TN_PREC_BF16X3) {
                        // chunk = [32 hi | 32 lo] bf16 (A) x [32 w_hi | 32 w_lo] (B); offsets in 16-byte units
                        constexpr int AO[6] = {0, 2, 4, 6, 0, 2};      // hi, hi, lo, lo, hi, hi
                        constexpr int BO[6] = {0, 2, 0, 2, 4, 6};      // w_hi x4,        w_lo x2
#pragma unroll
                        for (int i = 0; i < 6; ++i)
                            ptx::wgmma_bf16_n128(acc[hf], mk_desc(a_lo + AO[i]), mk_desc(b_lo + BO[i]), fresh | (i ? 1u : 0u));
                    } else {
                        mma_chunk<PREC, C::BN>(acc[hf], a_lo, b_lo, fresh);
                    }
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();
                if (cs.leader()) {
                    if (pend_b >= 0) ptx::mbar_arrive(&b_empty[pend_b]);
                    if (pend_a >= 0) ptx::mbar_arrive(&a_empty[pend_a]);
                }
                pend_b = b_ring.stage;
                pend_a = (k + 1 == KT::ntaps(u)) ? a_ring.stage : -1;
                fresh = 1u;
                b_ring.next();
            }
            a_ring.next();
        }
    }
    turn.pass();
    ptx::wgmma_wait<0>();
    ptx::wgmma_reg_fence(acc[0]);
    ptx::wgmma_reg_fence(acc[1]);
    if (cs.leader()) {
        if (pend_b >= 0) ptx::mbar_arrive(&b_empty[pend_b]);
        if (pend_a >= 0) ptx::mbar_arrive(&a_empty[pend_a]);
    }
}

template <int PREC>
__global__ void __launch_bounds__(kThreads2, 1)
conv_trunk_kernel(const __grid_constant__ TrunkParams p)
{
    using C = TCfg<PREC>;
    constexpr int BN = C::BN;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;                                                 // [kAStages][unit]
    uint8_t* sB = sA + C::kAStages * C::kAUnit;                         // [kBStages][128 rows x 128 B]
    uint8_t* sT = sB + C::kBStages * C::kBTile;                         // epilogue transpose tiles
    uint64_t* bars = reinterpret_cast<uint64_t*>(sT + ((C::kEpiBytes + 1023) & ~1023));
    uint64_t* a_full = bars;                       // [kAStages]
    uint64_t* a_empty = a_full + C::kAStages;
    uint64_t* b_full = a_empty + C::kAStages;      // [kBStages]
    uint64_t* b_empty = b_full + C::kBStages;
    uint64_t* sched_full = b_empty + C::kBStages;  // [kSched]
    uint64_t* sched_empty = sched_full + C::kSched;
    int* sched_slot = reinterpret_cast<int*>(sched_empty + C::kSched);   // [kSched] work-unit indices

    ptx::grid_dep_launch();
    if (threadIdx.x == 0) trace_stamp(p.trace, 0);
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    unsigned* done = p.sched + 1;                  // done[layer * max_batch + image]

    if (threadIdx.x == 0) {
        // an operand stage is read by the one consumer warpgroup that owns its unit
        for (int s = 0; s < C::kAStages; ++s) { ptx::mbar_init(&a_full[s], 1); ptx::mbar_init(&a_empty[s], 1); }
        for (int s = 0; s < C::kBStages; ++s) { ptx::mbar_init(&b_full[s], 1); ptx::mbar_init(&b_empty[s], 1); }
        for (int s = 0; s < C::kSched; ++s) { ptx::mbar_init(&sched_full[s], 1); ptx::mbar_init(&sched_empty[s], 9); }   // B producer + 8 consumer warps
        ptx::fence_barrier_init();
        ptx::fence_proxy_async();
    }
    __syncthreads();
    if (threadIdx.x == 0) trace_stamp(p.trace, 1);

    // every consumer role walks the same ring of work units
    Ring<C::kSched> sring;
    auto next_unit = [&](bool whole_warp) -> int {  // a consumer role's next work unit: called by a whole warp, or by lane 0 alone
        ptx::mbar_wait(&sched_full[sring.stage], sring.consumer_parity());
        int u = 0;
        if (lane == 0) u = sched_slot[sring.stage];   // read by the one thread that hands the slot back (a direct mbarrier edge to the writer)
        if (whole_warp) u = __shfl_sync(0xffffffffu, u, 0);
        if (lane == 0) ptx::mbar_arrive(&sched_empty[sring.stage]);
        sring.next();
        return u;
    };

    if (warp < 4) {
        ptx::setmaxnreg_dec<kProducerRegs>();       // the whole producer warpgroup, idle warps 2-3 included
        if (warp == 0) {
            // ============================== scheduler + A producer ================================
            if (lane == 0) {
                for (int l = 0; l < p.n_layers; ++l)    // every layer brings its own tensor maps: fetch the descriptors now, not at each layer's first load
                    for (int m = 0; m < (p.layer[l].kind == KIND_S2 ? 4 : 1); ++m) ptx::prefetch_tmap(&p.layer[l].amap[m]);
                ptx::grid_dep_wait();                   // the first layer's input comes from the previous kernel
                Ring<C::kAStages> a_ring;
                Ring<C::kSched> slot;
                // latency mode: the pieces of a unit (consecutive indices) must sit on DIFFERENT CTAs, because a piece's epilogue waits for
                // the others' partial sums -- units are dealt round robin (index i goes to CTA i mod grid; every wait then points at a
                // smaller index or at a piece whose CTA only has smaller indices left to finish: no cycle).  Throughput mode: first come, first served.
                const bool dealt = p.ksplit > 1;
                int u = dealt ? static_cast<int>(blockIdx.x) : static_cast<int>(atomicAdd(p.sched, 1u));
                for (;;) {
                    ptx::mbar_wait(&sched_empty[slot.stage], slot.producer_parity());
                    sched_slot[slot.stage] = u;
                    ptx::mbar_arrive(&sched_full[slot.stage]);  // release: the slot write is visible to the waiters
                    slot.next();
                    if (u >= p.total_units) break;
                    const UnitCoord c = decode_unit(p, u);
                    const LayerDesc& L = p.layer[c.l];
                    if (L.dep_layer >= 0) {
                        // this image's previous-layer output is complete once all its units' epilogue warps have signalled
                        const int* flag = reinterpret_cast<const int*>(done + L.dep_layer * p.max_batch + c.img);
                        if (static_cast<unsigned>(ptx::ld_acquire_gpu(flag)) < L.dep_target) {
                            const long long t0 = clock64();
                            while (static_cast<unsigned>(ptx::ld_acquire_gpu(flag)) < L.dep_target) {
                                __nanosleep(64);
                                if (clock64() - t0 > (1ll << 34)) ptx::timeout_trap();     // ~10 s: a scheduling bug becomes an error, not a hung GPU
                            }
                        }
                        ptx::fence_proxy_async_all();   // the TMA (async proxy) reads below must observe what the acquire made visible
                    }
                    unit_stamp(p, u, 0);
                    const int cbase = c.grp * L.in_gstride_words;
                    if (L.kind == KIND_S1) load_a_units<KIND_S1>(L, c.tx * 11, c.ty * 11, cbase, c.img, c.c0, c.c1, sA, a_full, a_empty, a_ring);
                    else                   load_a_units<KIND_S2>(L, c.tx * 11, c.ty * 11, cbase, c.img, c.c0, c.c1, sA, a_full, a_empty, a_ring);
                    u = dealt ? u + static_cast<int>(gridDim.x) : static_cast<int>(atomicAdd(p.sched, 1u));   // pull the next unit only now: look-ahead = the A pipeline depth
                }
            }
        } else if (warp == 1) {
            // ============================== B producer ================================
            if (lane == 0) {
                if (!p.img_wid) for (int l = 0; l < p.n_layers; ++l) ptx::prefetch_tmap(&p.layer[l].bmap);
                Ring<C::kBStages> b_ring;
                for (;;) {
                    const int u = next_unit(false);
                    if (u >= p.total_units) break;
                    const UnitCoord c = decode_unit(p, u);
                    const LayerDesc& L = p.layer[c.l];
                    const CUtensorMap* bm = p.img_wid ? p.gbmaps + p.img_wid[c.img] * kLayersPerSet + L.li : &L.bmap;
                    if (L.kind == KIND_S1) trunk_load_weights<KIND_S1, PREC>(L, bm, c, sB, b_full, b_empty, b_ring);
                    else                   trunk_load_weights<KIND_S2, PREC>(L, bm, c, sB, b_full, b_empty, b_ring);
                }
            }
        }
    } else {
        // ============================== MMA + epilogue (two warpgroups, alternate units) ==========================
        ptx::setmaxnreg_inc<kConsumerRegs>();
        using S = Storage<PREC>;
        using R4 = Raw<PREC, 4>;
        ptx::grid_dep_wait();
        const Consumer cs;
        const int cw = cs.cw;                       // warp cw of a warpgroup = tile rows 16 cw + [0, 16) and 64 + 16 cw + [0, 16) of its units
        float (*stg)[C::kEpiPitch] = reinterpret_cast<float (*)[C::kEpiPitch]>(sT + cs.ew * C::kEpiWarpBytes);
        int* rowtab = reinterpret_cast<int*>(sT + cs.ew * C::kEpiWarpBytes + 16 * C::kEpiPitch * 4);
        const int grp = lane & 7, sub = lane >> 3;  // lane = (16-byte column group, pixel within a group of 4)
        Ring<C::kAStages> a_ring;
        Ring<C::kBStages> b_ring;
        // Ping-pong: warpgroup it % 2 owns the CTA's it-th unit and issues its MMAs in turn it.
        const Turn turn{kTurnBar, cs.cg};
        turn.begin();
        for (int it = 0;; ++it) {
            const int u = next_unit(true);
            const bool mine = turn.mine(it);
            if (u >= p.total_units) { turn.end(it); break; }
            const UnitCoord c = decode_unit(p, u);
            const LayerDesc& L = p.layer[c.l];
            const int chunks = L.chunks / p.ksplit;          // K chunks of this piece (the host makes chunks divisible)
            if (!mine) {
                // the other warpgroup's unit: step this warpgroup's operand ring positions past the stages it occupies
                a_ring.skip(chunks * (L.kind == KIND_S1 ? KTab<KIND_S1>::NU : KTab<KIND_S2>::NU));
                b_ring.skip(chunks * kTaps3);
                continue;
            }
            {
                // lane < 16: tile row 16 cw + lane; lane >= 16: tile row 64 + 16 cw + lane - 16
                const int rw = 64 * (lane >> 4) + 16 * cw + (lane & 15);
                const int py = rw / 11, px = rw - py * 11;
                const int y = c.ty * 11 + py, x = c.tx * 11 + px;
                const bool valid = (rw < 121) && (y < L.Ho) && (x < L.Wo);
                __syncwarp();
                rowtab[lane] = valid ? (c.img * L.Ho + y) * L.Wo + x : -1;
                __syncwarp();
            }
            const int ch0 = c.grp * L.cout + c.n_tile * BN;      // first output channel of this unit
            const float* bias_base = p.img_wid ? p.gbias[p.img_wid[c.img] * kLayersPerSet + L.li] : L.bias;
            float4 b4[BN / 32];                                  // bias of the four 32-column blocks: loads in flight during the MMAs
#pragma unroll
            for (int bi = 0; bi < BN / 32; ++bi) b4[bi] = __ldg(reinterpret_cast<const float4*>(bias_base + ch0 + 32 * bi + grp * 4));
            // SE3TN_PREC_FP8: y = acc * mul[co] + bias (+ residual code * its scale), then the output code = y / s_out.  A unit's
            // 128 channels lie in one head group, so the two scales are the unit's.  Powers of two: both multiplies are exact.
            const float* q8 = nullptr;
            float s_res = 1.f, inv_out = 1.f;
            if constexpr (PREC == SE3TN_PREC_FP8) {
                q8 = p.img_wid ? p.gfp8[p.img_wid[c.img]] : p.fp8;
                const int qg = L.q_grp_ch ? ch0 / L.q_grp_ch : 0;
                if (L.q_res >= 0) s_res = __ldg(q8 + L.q_res + qg);
                if (L.q_out >= 0) inv_out = 1.f / __ldg(q8 + L.q_out + qg);
            }

            float acc[2][C::kAcc];                               // tile rows [0, 64) and [64, 128)
#pragma unroll
            for (int i = 0; i < C::kAcc; ++i) { acc[0][i] = 0.f; acc[1][i] = 0.f; }
            unsigned long long* ust = (p.trace && u < 2048) ? p.trace + 256 * 8 + u * 5 + 1 : nullptr;
            if (L.kind == KIND_S1) trunk_mma_unit<KIND_S1, PREC>(acc, cs, turn, chunks, sA, sB, a_full, a_empty, b_full, b_empty, a_ring, b_ring, p.trace, it == 0, ust);
            else                   trunk_mma_unit<KIND_S2, PREC>(acc, cs, turn, chunks, sA, sB, a_full, a_empty, b_full, b_empty, a_ring, b_ring, p.trace, it == 0, ust);
            if (cs.leader()) { unit_stamp(p, u, 2); unit_stamp(p, u, 3); if (it == 0) trace_stamp(p.trace, 5); }
            int pix[2][4];                                       // pixels this lane post-processes: rows 4k + sub of each 16-row slice
#pragma unroll
            for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                for (int k = 0; k < 4; ++k) pix[hf][k] = rowtab[16 * hf + 4 * k + sub];

            if (L.res && L.dep_layer >= 0) {
                // the residual was written earlier in THIS launch by other CTAs (an ancestor layer of this unit): order this
                // warp's loads after the completion counter the producer thread already observed
                if (lane == 0) (void)ptx::ld_acquire_gpu(reinterpret_cast<const int*>(done + L.dep_layer * p.max_batch + c.img));
                __syncwarp();
            }
            const bool split = p.ksplit > 1;
            // this warp's slice (its 32 rows x 128 columns) of piece `pc` of this unit in the split-K scratch: per 64-row half and
            // 32-column block the fragment's 16 registers as 4 float4, [half][block][float4 jj][lane]
            auto slice_of = [&](int pc) -> float* {
                return p.partial + ((static_cast<size_t>(c.gidx) * p.ksplit + pc) * 4 + cw) * (32 * BN);
            };
            unsigned own = 0xFu;                                 // which of the unit's four 32-column blocks this warp post-processes
            if (split) {
                // latency mode: this CTA only summed K chunks [c0, c1).  Dump the fp32 slice; the unit's four 32-column blocks are then
                // finished by its pieces in parallel: block b by piece b * ksplit / 4, which waits until every piece has dumped and adds
                // them in piece order 0..ksplit-1 (the result does not depend on arrival order).
                float4* d4 = reinterpret_cast<float4*>(slice_of(c.piece)) + lane;
#pragma unroll
                for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                    for (int q = 0; q < C::kAcc / 4; ++q)
                        d4[(hf * C::kAcc / 4 + q) * 32] = make_float4(acc[hf][4 * q], acc[hf][4 * q + 1], acc[hf][4 * q + 2], acc[hf][4 * q + 3]);
                __threadfence();
                __syncwarp();
                if (lane == 0) atomicAdd(p.slice_cnt + c.gidx * 4 + cw, 1u);
                own = 0u;
#pragma unroll
                for (int bi = 0; bi < BN / 32; ++bi)
                    if (bi * p.ksplit / (BN / 32) == c.piece) own |= 1u << bi;
                if (lane == 0) {
                    const int* cnt = reinterpret_cast<const int*>(p.slice_cnt + c.gidx * 4 + cw);
                    const long long t0 = clock64();
                    while (ptx::ld_acquire_gpu(cnt) < p.ksplit) {
                        __nanosleep(32);
                        if (clock64() - t0 > (1ll << 34)) ptx::timeout_trap();
                    }
                }
                __syncwarp();
                __threadfence();                                                     // order the reads below after the other pieces' dumps
                // the owned blocks' sums of all pieces, in piece order, back into the fragment registers
#pragma unroll
                for (int hf = 0; hf < 2; ++hf)
#pragma unroll
                    for (int bi = 0; bi < BN / 32; ++bi) {
                        if (!((own >> bi) & 1u)) continue;
#pragma unroll
                        for (int jj = 0; jj < 4; ++jj) {
                            float4 v[kSplitK];                       // all pieces' loads in flight before the first add
#pragma unroll
                            for (int pc = 0; pc < kSplitK; ++pc)
                                if (pc < p.ksplit) v[pc] = __ldcg(reinterpret_cast<const float4*>(slice_of(pc)) + lane + (hf * C::kAcc / 4 + 4 * bi + jj) * 32);
                            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                            for (int pc = 0; pc < kSplitK; ++pc)
                                if (pc < p.ksplit) { a.x += v[pc].x; a.y += v[pc].y; a.z += v[pc].z; a.w += v[pc].w; }
                            acc[hf][16 * bi + 4 * jj] = a.x; acc[hf][16 * bi + 4 * jj + 1] = a.y; acc[hf][16 * bi + 4 * jj + 2] = a.z; acc[hf][16 * bi + 4 * jj + 3] = a.w;
                        }
                    }
            }
            // the two 16-row slices of this warp one after the other through its staging tile: slice 4 hf + cw = tile rows 16 (4 hf + cw) + [0, 16)
#pragma unroll
            for (int hf = 0; hf < 2; ++hf) {
                const int slice = 4 * hf + cw;
#pragma unroll
                for (int bi = 0; bi < BN / 32; ++bi) {
                    if (!((own >> bi) & 1u)) continue;
                    const int chan = ch0 + 32 * bi;                   // first channel of this 32-channel block
                    // residual pieces first: their L2 latency overlaps the staging round trip below
                    R4 rr[4];                                        // residual: this lane's 4 pixels, 4 channels each
                    if (L.res) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            rr[k] = R4{};
                            if (pix[hf][k] >= 0) {
                                const uint8_t* rp = L.res + S::addr(pix[hf][k], L.res_c, chan + grp * 4);
#pragma unroll
                                for (int q = 0; q < R4::kPieces; ++q) rr[k].set(q, __ldcg(R4::at(rp, q)));
                            }
                        }
                    }
                    // fragment -> rows of the staging tile: register 16 bi + 4 jj + 2 h + e = slice row R + 8h, block column 8 jj + 2m + e
                    __syncwarp();                                    // previous block's readers are done with stg
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            *reinterpret_cast<float2*>(&stg[cs.R + 8 * h][8 * jj + 2 * cs.m]) = make_float2(acc[hf][16 * bi + 4 * jj + 2 * h], acc[hf][16 * bi + 4 * jj + 2 * h + 1]);
                    float4 m4 = make_float4(1.f, 1.f, 1.f, 1.f);
                    if constexpr (PREC == SE3TN_PREC_FP8) m4 = __ldg(reinterpret_cast<const float4*>(q8 + L.fp8_mul + chan + grp * 4));
                    __syncwarp();
                    float4 a4[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        a4[k] = *reinterpret_cast<const float4*>(&stg[4 * k + sub][grp * 4]);
                        if constexpr (PREC == SE3TN_PREC_FP8) {
                            a4[k].x = a4[k].x * m4.x + b4[bi].x; a4[k].y = a4[k].y * m4.y + b4[bi].y;
                            a4[k].z = a4[k].z * m4.z + b4[bi].z; a4[k].w = a4[k].w * m4.w + b4[bi].w;
                        } else {
                            a4[k].x += b4[bi].x; a4[k].y += b4[bi].y; a4[k].z += b4[bi].z; a4[k].w += b4[bi].w;
                        }
                    }
                    if (L.res) {
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            float r[4];
                            S::decode(rr[k], r);
                            if constexpr (PREC == SE3TN_PREC_FP8) { r[0] *= s_res; r[1] *= s_res; r[2] *= s_res; r[3] *= s_res; }
                            a4[k].x += r[0]; a4[k].y += r[1]; a4[k].z += r[2]; a4[k].w += r[3];
                        }
                    }
                    float4 psum = make_float4(0.f, 0.f, 0.f, 0.f);   // fused average pool: this lane's rows, 4 channels
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float4 o = a4[k];
                        o.x = act_apply(o.x, L.act); o.y = act_apply(o.y, L.act); o.z = act_apply(o.z, L.act); o.w = act_apply(o.w, L.act);
                        if (pix[hf][k] < 0) continue;
                        if (L.pool_part) { psum.x += o.x; psum.y += o.y; psum.z += o.z; psum.w += o.w; continue; }
                        if constexpr (PREC == SE3TN_PREC_FP8) { o.x *= inv_out; o.y *= inv_out; o.z *= inv_out; o.w *= inv_out; }
                        const float o4[4] = {o.x, o.y, o.z, o.w};
                        S::encode(o4).store(L.out + S::addr(pix[hf][k], L.out_c, L.out_coff + chan + grp * 4));
                    }
                    if (L.pool_part) {                                // rows 4k + sub summed above; fold the four `sub` groups (fixed order: deterministic)
#pragma unroll
                        for (int off = 8; off <= 16; off <<= 1) {
                            psum.x += __shfl_xor_sync(0xffffffffu, psum.x, off); psum.y += __shfl_xor_sync(0xffffffffu, psum.y, off);
                            psum.z += __shfl_xor_sync(0xffffffffu, psum.z, off); psum.w += __shfl_xor_sync(0xffffffffu, psum.w, off);
                        }
                        if (sub == 0)
                            *reinterpret_cast<float4*>(L.pool_part + (static_cast<size_t>(c.img) * kPoolSlices + slice) * L.out_c + L.out_coff + chan + grp * 4) = psum;
                    }
                }
            }
            // this warp's part of the unit is in memory: publish it to the units of the next layer that wait for this image
            if (c.l + 1 < p.n_layers) {
                ptx::fence_proxy_async_all();       // consumers read these bytes through TMA (async proxy)
                __threadfence();
                __syncwarp();
                if (lane == 0) atomicAdd(done + c.l * p.max_batch + c.img, 1u);
            }
            if (cs.leader()) unit_stamp(p, u, 4);
        }
        if (threadIdx.x == 128) { trace_stamp(p.trace, 4); trace_stamp(p.trace, 6); }
    }

    __syncthreads();
    if (threadIdx.x == 0) trace_exit(p.trace);
}

// ---------------------------------------------------------------------------------------------------------------
template <int KIND, int PREC>
cudaError_t launch_resident_t(const ResidentParams& p, int num_sms, bool pdl, cudaStream_t stream) {
    using C = RCfg<KIND, resident_prec(PREC)>;
    if (PREC == SE3TN_PREC_FP8 && ((!p.fp8 && !p.gfp8) || p.L.q_out < 0)) return cudaErrorInvalidValue;
    const int tiles_per_tap = (C::kStack == 2) ? 1 : p.L.chunks;
    if ((KIND == KIND_STEM ? 7 : 9) * tiles_per_tap > C::kMaxWTiles) return cudaErrorInvalidValue;
    if (C::kStack == 2 && KIND == KIND_S1 && p.L.chunks != 2) return cudaErrorInvalidValue;    // a stacked tile row is exactly two 32-channel chunks
    if (p.L.cout != 64 || p.L.groups != 1 || p.L.n_tiles != 1 || p.m_tiles <= 0) return cudaErrorInvalidValue;
    // Ping-pong only where some CTA has a second tile whose MMAs can run under its first tile's epilogue.  Where every CTA has
    // one tile (n = 1: 81 stem tiles, 16 per 64-channel layer), the halves schedule runs that one epilogue on twice the threads.
    const bool pp = p.m_tiles > num_sms;
    const cudaError_t e = pp ? set_max_dynamic_smem<conv_resident_kernel<KIND, PREC, true>>(C::kSmem)
                             : set_max_dynamic_smem<conv_resident_kernel<KIND, PREC, false>>(C::kSmem);
    if (e != cudaSuccess) return e;
    return launch_kernel(pp ? conv_resident_kernel<KIND, PREC, true> : conv_resident_kernel<KIND, PREC, false>,
                         dim3(std::min(p.m_tiles, num_sms)), dim3(kThreads2), C::kSmem, stream, pdl, p);
}

template <int PREC>
cudaError_t launch_trunk_t(const TrunkParams& p, int num_sms, bool pdl, cudaStream_t stream) {
    using C = TCfg<PREC>;
    if (p.n_layers < 1 || p.n_layers > kTrunkMaxLayers || p.total_units <= 0 || !p.sched) return cudaErrorInvalidValue;
    if (p.ksplit < 1 || (p.ksplit > 1 && (!p.partial || !p.slice_cnt || p.ksplit > kSplitK))) return cudaErrorInvalidValue;
    if (PREC == SE3TN_PREC_FP8 && !p.fp8 && !p.gfp8) return cudaErrorInvalidValue;
    for (int l = 0; l < p.n_layers; ++l) {
        const LayerDesc& L = p.layer[l];
        if ((L.kind != KIND_S1 && L.kind != KIND_S2) || L.cout % C::BN || L.n_tiles != L.cout / C::BN) return cudaErrorInvalidValue;
        if (L.pool_part && (L.tiles_x != 1 || L.tiles_y != 1)) return cudaErrorInvalidValue;   // fused avg-pool: tile = whole image
        if (L.dep_layer >= l) return cudaErrorInvalidValue;                                    // dependencies point backwards in the pull order
        if (L.chunks % p.ksplit) return cudaErrorInvalidValue;
    }
    const cudaError_t e = set_max_dynamic_smem<conv_trunk_kernel<PREC>>(C::kSmem);
    if (e != cudaSuccess) return e;
    // all CTAs must be co-resident (one per SM): the dependency waits rely on it
    return launch_kernel(conv_trunk_kernel<PREC>, dim3(std::min(p.total_units, num_sms)), dim3(kThreads2), C::kSmem, stream, pdl, p);
}

}  // namespace

cudaError_t launch_conv_resident(const ResidentParams& p, int kind, int prec, int num_sms, bool pdl, cudaStream_t stream) {
    if (kind == KIND_STEM) {
        switch (prec) {
            case SE3TN_PREC_TF32:   return launch_resident_t<KIND_STEM, SE3TN_PREC_TF32>(p, num_sms, pdl, stream);
            case SE3TN_PREC_BF16X3: return launch_resident_t<KIND_STEM, SE3TN_PREC_BF16X3>(p, num_sms, pdl, stream);
            case SE3TN_PREC_BF16:   return launch_resident_t<KIND_STEM, SE3TN_PREC_BF16>(p, num_sms, pdl, stream);
            case SE3TN_PREC_FP16:   return launch_resident_t<KIND_STEM, SE3TN_PREC_FP16>(p, num_sms, pdl, stream);   // bf16x3, fp16 output
        }
    } else if (kind == KIND_S1) {
        switch (prec) {
            case SE3TN_PREC_TF32:   return launch_resident_t<KIND_S1, SE3TN_PREC_TF32>(p, num_sms, pdl, stream);
            case SE3TN_PREC_BF16X3: return launch_resident_t<KIND_S1, SE3TN_PREC_BF16X3>(p, num_sms, pdl, stream);
            case SE3TN_PREC_BF16:   return launch_resident_t<KIND_S1, SE3TN_PREC_BF16>(p, num_sms, pdl, stream);
            case SE3TN_PREC_FP8:    return launch_resident_t<KIND_S1, SE3TN_PREC_FP8>(p, num_sms, pdl, stream);   // bf16, e4m3 output
            case SE3TN_PREC_FP16:   return launch_resident_t<KIND_S1, SE3TN_PREC_FP16>(p, num_sms, pdl, stream);
        }
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_conv_trunk(const TrunkParams& p, int prec, int num_sms, bool pdl, cudaStream_t stream) {
    switch (prec) {
        case SE3TN_PREC_TF32:   return launch_trunk_t<SE3TN_PREC_TF32>(p, num_sms, pdl, stream);
        case SE3TN_PREC_BF16X3: return launch_trunk_t<SE3TN_PREC_BF16X3>(p, num_sms, pdl, stream);
        case SE3TN_PREC_BF16:   return launch_trunk_t<SE3TN_PREC_BF16>(p, num_sms, pdl, stream);
        case SE3TN_PREC_FP8:    return launch_trunk_t<SE3TN_PREC_FP8>(p, num_sms, pdl, stream);
        case SE3TN_PREC_FP16:   return launch_trunk_t<SE3TN_PREC_FP16>(p, num_sms, pdl, stream);
    }
    return cudaErrorInvalidValue;
}

}  // namespace se3tn
