// Device helpers shared by the training-loss kernels (anchor_loss.cu, monoflex_loss.cu).
#pragma once
#include <cuda_runtime.h>

namespace vd3d {

// torch.nn.functional.logsigmoid, in its overflow-free form
__device__ __forceinline__ float log_sigmoid(float x) { return fminf(x, 0.f) - log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

}  // namespace vd3d
