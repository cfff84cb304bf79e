// Host-side launch helpers shared by the kernel files.
#pragma once
#include <cuda_runtime.h>
#include <utility>

namespace se3tn {

// Launch `kernel` on `stream`.  pdl: with programmatic stream serialization, so the kernel's CTAs may start once every CTA
// of the previous kernel in the stream has executed griddepcontrol.launch_dependents (or exited); the kernel then orders its
// reads of the previous kernel's output with griddepcontrol.wait.
template <typename... Params, typename... Args>
cudaError_t launch_kernel(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl,
                          Args&&... args) {
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// Allow `Kernel` smem bytes of dynamic shared memory on the current device.  The limit is a per-device function attribute:
// it is set once per device, and again only for a larger size.
template <auto Kernel>
cudaError_t set_max_dynamic_smem(size_t smem) {
    static size_t set[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) dev = 0;
    if (smem <= set[dev]) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e == cudaSuccess) set[dev] = smem;
    return e;
}

}  // namespace se3tn
