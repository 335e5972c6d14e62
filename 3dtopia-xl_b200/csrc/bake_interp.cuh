// Barycentric attribute interpolation shared by tpx_rast_interpolate (texture_bake.cu) and the fused texel query tpx_primsdf_bake
// (primsdf.cu): attr = u a0 + v a1 + (1 - u - v) a2 with (u, v) the weights of vertices 0 and 1 (the layout of a `rast` texel).
// Every operation is rounded or fused as written, so both kernels produce the same bits from the same `rast` texel.
#pragma once

namespace tpx {

__device__ __forceinline__ float bary_interp(float u, float v, float a0, float a1, float a2) {
    const float w = __fsub_rn(__fsub_rn(1.0f, u), v);
    return __fmaf_rn(w, a2, __fmaf_rn(v, a1, __fmul_rn(u, a0)));
}

// triangle id of a rast texel (channel 3 holds id + 1 as a float, 0 = empty), or -1
__device__ __forceinline__ int rast_triangle(float w) { return static_cast<int>(w) - 1; }

}  // namespace tpx
