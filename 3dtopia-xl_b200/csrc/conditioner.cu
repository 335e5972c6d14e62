// Kernels that only the image-conditioner encoder needs (SURVEY.md §8f-2: DINOv2 ViT-B/14-reg, models/conditioner/image_dinov2.py:44-61
// and dinov2/layers/mlp.py:33-39).  Everything else of that encoder reuses the DiT kernels through their per-kernel entry points
// (tpx_ln_modulate, tpx_linear_heads, tpx_attention, tpx_linear, tpx_linear_gated); see 3dtopia-xl_b200/dinov2.py.
#include "kernels.cuh"

namespace tpx {
namespace {

// nn.GELU() (erf form) applied in place to an fp16 tensor: fp32 math on the fp16 value, one rounding of the result, within one fp16
// ulp of the exact GELU for every finite input.  Evaluated as 0.5 x erfc(-x / sqrt 2): the textbook 1 + erf(x / sqrt 2) cancels for
// x below about -3 (near x = -4.3 the result is off by up to 8 fp16 ulps), erfc keeps its relative precision there.
// 8 elements (16 B) per thread per step, grid-stride.
__global__ void __launch_bounds__(256) gelu_erf_kernel(__half* __restrict__ x, long long n8) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        Pack8 v;
        v.u = *reinterpret_cast<const uint4*>(x + 8 * i);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float a = __half2float(v.h[k]);
            v.h[k] = __float2half_rn(0.5f * a * erfcf(a * -0.70710678118654752440f));
        }
        *reinterpret_cast<uint4*>(x + 8 * i) = v.u;
    }
}

}  // namespace
}  // namespace tpx

extern "C" int tpx_gelu_erf(void* x_f16, int64_t n, void* stream) {
    using namespace tpx;
    TPX_CHECK(x_f16 != nullptr || n == 0, TPX_ERR_ARG, "gelu_erf: null argument");
    TPX_CHECK(n >= 0 && n % 8 == 0 && (reinterpret_cast<uintptr_t>(x_f16) & 15) == 0, TPX_ERR_SHAPE, "gelu_erf: %lld elements (need a multiple of 8, 16-B aligned)",
              static_cast<long long>(n));
    if (n == 0) return TPX_OK;
    TPX_DEVICE_GUARD();
    const long long n8 = n / 8;
    const long long want = (n8 + 255) / 256;
    const unsigned blocks = static_cast<unsigned>(want < gemm_num_sms() * 8LL ? want : gemm_num_sms() * 8LL);
    gelu_erf_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<__half*>(x_f16), n8);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}
