// Plain fp32 FFMA direct convolution over the same NHWC tensors / packed weights as the
// wgmma path.  Two jobs: (1) the `precision = fp32` mode of se3tn_forward (no operand
// rounding at all, bit-for-bit independent of the tensor-core path), and (2) an on-device
// cross-check for the wgmma kernels at sizes where a CPU oracle run is slow.
// 64 pixels x 64 output channels per CTA, 4x4 outputs per thread, K stepped 16 floats at a time.
#include "conv_common.h"
#include "ptx.cuh"

namespace se3tn {
namespace {

constexpr int TP = 64, TC = 64, TK = 16;

__device__ __forceinline__ float selu_d(float x) {
    constexpr float kAlpha = 1.6732632423543772f, kScale = 1.0507009873554805f;
    return x > 0.f ? kScale * x : (kScale * kAlpha) * expm1f(x);
}

__global__ void __launch_bounds__(256)
conv_direct_kernel(const ConvGeom g, const ConvPtrs p)
{
    __shared__ float sA[TK][TP + 4];
    __shared__ float sW[TK][TC + 4];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int grp = blockIdx.z;
    const int co0 = blockIdx.y * TC;
    const long long P = static_cast<long long>(g.n_img) * g.Ho * g.Wo;
    const long long pix0 = static_cast<long long>(blockIdx.x) * TP;
    const int ktot = g.num_taps * g.cin;

    // this thread's load assignment: pixel lp / weight row lp, k-quad lq
    const int lp = tid >> 2, lq = tid & 3;
    const long long lpix = pix0 + lp;
    const bool lvalid = lpix < P;
    int ln = 0, ly = 0, lx = 0;
    if (lvalid) {
        ln = static_cast<int>(lpix / (g.Ho * g.Wo));
        int r = static_cast<int>(lpix - static_cast<long long>(ln) * g.Ho * g.Wo);
        ly = r / g.Wo; lx = r - ly * g.Wo;
    }
    const float* wrow = p.w + static_cast<size_t>(grp * g.cout + co0 + lp) * ktot;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int tap = 0; tap < g.num_taps; ++tap) {
        const int iy = ly * g.stride + g.taps[tap].dy;
        const int ix = lx * g.stride + g.taps[tap].dx;
        const bool inb = lvalid && iy >= 0 && iy < g.Hin && ix >= 0 && ix < g.Win;
        const float* ap = p.in + ((static_cast<size_t>(ln) * g.Hin + iy) * g.Win + ix) * g.in_cstride + g.in_coff + grp * g.cin;
        for (int c0 = 0; c0 < g.cin; c0 += TK) {
            float4 a4 = make_float4(0.f, 0.f, 0.f, 0.f);
            if (inb) a4 = __ldg(reinterpret_cast<const float4*>(ap + c0 + lq * 4));
            const float4 w4 = __ldg(reinterpret_cast<const float4*>(wrow + tap * g.cin + c0 + lq * 4));
            __syncthreads();
            sA[lq * 4 + 0][lp] = a4.x; sA[lq * 4 + 1][lp] = a4.y; sA[lq * 4 + 2][lp] = a4.z; sA[lq * 4 + 3][lp] = a4.w;
            sW[lq * 4 + 0][lp] = w4.x; sW[lq * 4 + 1][lp] = w4.y; sW[lq * 4 + 2][lp] = w4.z; sW[lq * 4 + 3][lp] = w4.w;
            __syncthreads();
#pragma unroll
            for (int k = 0; k < TK; ++k) {
                const float4 a = *reinterpret_cast<const float4*>(&sA[k][ty * 4]);
                const float4 b = *reinterpret_cast<const float4*>(&sW[k][tx * 4]);
                const float av[4] = {a.x, a.y, a.z, a.w};
                const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
        }
    }

    const int ch = grp * g.cout + co0 + tx * 4;
    const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + ch));
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long pix = pix0 + ty * 4 + i;
        if (pix >= P) continue;
        float v[4] = {acc[i][0] + b4.x, acc[i][1] + b4.y, acc[i][2] + b4.z, acc[i][3] + b4.w};
        if (p.res) {
            const float4 r4 = __ldg(reinterpret_cast<const float4*>(p.res + static_cast<size_t>(pix) * g.res_cstride + g.res_coff + ch));
            v[0] += r4.x; v[1] += r4.y; v[2] += r4.z; v[3] += r4.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float o = v[j];
            if (g.act == ACT_RELU) o = fmaxf(o, 0.f);
            else if (g.act == ACT_SELU) o = selu_d(o);
            v[j] = o;
        }
        *reinterpret_cast<float4*>(p.out + static_cast<size_t>(pix) * g.out_cstride + g.out_coff + ch) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

}  // namespace

cudaError_t launch_conv_direct(const ConvGeom& g, const ConvPtrs& p, cudaStream_t stream) {
    if (g.cout % TC != 0 || g.cin % TK != 0) return cudaErrorInvalidValue;
    const long long P = static_cast<long long>(g.n_img) * g.Ho * g.Wo;
    dim3 grid(static_cast<unsigned>((P + TP - 1) / TP), g.cout / TC, g.groups);
    conv_direct_kernel<<<grid, 256, 0, stream>>>(g, p);
    return cudaGetLastError();
}

}  // namespace se3tn
