// Typed kernel launch helper: kern<<<grid, block, smem, s>>>(args...) through cudaLaunchKernelEx with the arguments
// converted to the kernel's parameter types.
//
// Programmatic dependent launch was tried here (griddepcontrol.wait / launch_dependents in every kernel of a decode
// step, the programmatic-serialization launch attribute, also inside the captured CUDA graph) and gave no gain at
// batch 20: inside a graph the kernel-to-kernel gap is already ~1 us and the ~1 900 kernels are bound by their own
// run time, so the attribute and the device-side waits were removed again.
#pragma once
#include <cuda_runtime.h>

#include <utility>

#include "common.cuh"

namespace sealb200 {

template <typename... KArgs, typename... Args>
inline void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(std::forward<Args>(args))...));
}

}  // namespace sealb200
