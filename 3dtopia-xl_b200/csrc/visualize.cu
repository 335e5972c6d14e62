// Preview payloads of the ray-march renders (dva/visualize.py): the coloured-box template of `generate_colored_boxes`
// (dva/ray_marcher.py:232-279) and the rgb / material primitive templates `visualize_*` build from `recon_param` (visualize.py:
// 217-239), each in one launch.  Both follow the reference's eager fp32 op order one explicitly rounded operation at a time
// (__fmul_rn / __fadd_rn / __fdiv_rn are never contracted into FMA; the one fused multiply-add below is torch's own `linspace`
// arithmetic, and expf is the same accurate libdevice function torch's `exp` calls).
//   * colored boxes: per voxel of the S^3 lattice, the dominant-axis sign normal of meshgrid(linspace(-1,1,S)^3) ('ij': z, y, x),
//     (nx, -ny, -nz) / sqrt(|n|^2), lit by lightdir = -3 * 1 / ||-3 * 1||: mult = clamp(sum(lightdir * n), min = 0.2), and
//     rgb = colour[k] * (1.4f * mult), alpha = alpha.  A voxel whose coordinates are all 0 (the centre of an odd S whose linspace
//     hits 0 exactly) has a zero normal, 0 / 0 = NaN, and NaN rgb, as the reference has; the clamp keeps the NaN (torch's clamp
//     propagates it, fmaxf would not).  The template depends on N, K, S, the colours and alpha only.
//   * payload: rgb = feat_tex * 255, alpha = exp(-(sdf * (1 / 0.005f))^2) * 255 with torch's CUDA `tensor / scalar` (a multiply by
//     the fp32 reciprocal), `** 2` (x * x) and the accurate expf; the material mode colours (0, roughness, metallic) * 255.
#include "kernels.cuh"

namespace tpx {

namespace {

constexpr int VZ_THREADS = 256;

// torch.linspace(-1, 1, S)[i] as the CUDA factory computes it (start + step * i below the halfway index, end - step * (S - 1 - i)
// from it on, each contracted into one FMA by nvcc)
__device__ __forceinline__ float linspace_m1_1(int i, int S) {
    const float step = __fdiv_rn(2.f, static_cast<float>(S - 1));
    return i < S / 2 ? fmaf(step, static_cast<float>(i), -1.f) : fmaf(-step, static_cast<float>(S - 1 - i), 1.f);
}

__device__ __forceinline__ float signf(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// The box shading factor 1.4f * clamp(sum(lightdir * n), 0.2) of voxel (z, y, x)
__device__ __forceinline__ float box_shade(int z, int y, int x, int S) {
    const float zz = linspace_m1_1(z, S), yy = linspace_m1_1(y, S), xx = linspace_m1_1(x, S);
    const float ax = fabsf(xx), ay = fabsf(yy), az = fabsf(zz);
    const float nx0 = (ax >= ay && ax >= az) ? signf(xx) : 0.f;
    const float ny0 = (ay >= ax && ay >= az) ? signf(yy) : 0.f;
    const float nz0 = (az >= ax && az >= ay) ? signf(zz) : 0.f;
    const float n[3] = {nx0, -ny0, -nz0};
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(n[0], n[0]), __fmul_rn(n[1], n[1])), __fmul_rn(n[2], n[2])));
    const float light = __fdiv_rn(-3.f, __fsqrt_rn(27.f));
    // The three products have one magnitude (or are zero), so every summation order gives the same sum.
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 3; ++j) m = __fadd_rn(m, __fmul_rn(light, __fdiv_rn(n[j], len)));
    m = m < 0.2f ? 0.2f : m;                                          // clamp(min=0.2): NaN stays NaN
    return __fmul_rn(1.4f, m);
}

__global__ void __launch_bounds__(VZ_THREADS) colored_boxes_kernel(const float* __restrict__ colors, int N, int K, int S, float alpha, int chlast,
                                                                  float* __restrict__ out) {
    const int S3 = S * S * S;
    const int64_t total = static_cast<int64_t>(N) * K * S3;
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int v = static_cast<int>(i % S3);
        const int64_t nk = i / S3;
        const int k = static_cast<int>(nk % K);
        const int x = v % S, y = (v / S) % S, z = v / (S * S);
        const float f = box_shade(z, y, x, S);
        const float r = __fmul_rn(colors[k * 3], f), g = __fmul_rn(colors[k * 3 + 1], f), b = __fmul_rn(colors[k * 3 + 2], f);
        if (chlast) {
            reinterpret_cast<float4*>(out)[i] = make_float4(r, g, b, alpha);
        } else {
            float* o = out + nk * 4 * S3 + v;
            o[0] = r; o[S3] = g; o[2 * S3] = b; o[3 * S3] = alpha;
        }
    }
}

__global__ void __launch_bounds__(VZ_THREADS) primvolume_payload_kernel(const float* __restrict__ recon, int BP, int S, int mode, float* __restrict__ out) {
    const int S3 = S * S * S;
    const int C = 4 + 6 * S3;
    const int64_t total = static_cast<int64_t>(BP) * S3;
    const float inv_var = __fdiv_rn(1.f, 0.005f);                     // `sdf / 0.005` on CUDA: sdf * (1.0f / 0.005f)
    for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < total; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
        const int v = static_cast<int>(i % S3);
        const float* row = recon + (i / S3) * C;
        const float t = __fmul_rn(row[4 + v], inv_var);
        const float a = __fmul_rn(expf(-__fmul_rn(t, t)), 255.f);
        float4 o;
        if (mode == TPX_PAYLOAD_MAT) {
            const float* mat = row + 4 + 4 * S3;                       // [roughness, metallic] after geo (1) and tex (3)
            o = make_float4(0.f, __fmul_rn(mat[v], 255.f), __fmul_rn(mat[S3 + v], 255.f), a);
        } else {
            const float* tex = row + 4 + S3;
            o = make_float4(__fmul_rn(tex[v], 255.f), __fmul_rn(tex[S3 + v], 255.f), __fmul_rn(tex[2 * S3 + v], 255.f), a);
        }
        reinterpret_cast<float4*>(out)[i] = o;
    }
}

int grid_for(int64_t total) {
    return static_cast<int>(std::min<int64_t>((total + VZ_THREADS - 1) / VZ_THREADS, 132 * 32));
}

}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" int tpx_colored_boxes(const float* colors, int N, int K, int S, float alpha, int layout, float* out, void* stream) {
    TPX_CHECK(colors != nullptr && out != nullptr, TPX_ERR_ARG, "tpx_colored_boxes: null argument");
    TPX_CHECK(N >= 1 && K >= 1 && S >= 2 && S <= 64 && static_cast<int64_t>(N) * K * S * S * S * 4 < (int64_t(1) << 40), TPX_ERR_SHAPE,
              "tpx_colored_boxes: bad shape (N %d K %d S %d)", N, K, S);
    TPX_CHECK(layout == TPX_LAYOUT_NCDHW || layout == TPX_LAYOUT_CHLAST, TPX_ERR_ARG, "tpx_colored_boxes: unknown layout %d", layout);
    TPX_CHECK(layout != TPX_LAYOUT_CHLAST || (reinterpret_cast<uintptr_t>(out) & 15) == 0, TPX_ERR_ARG,
              "tpx_colored_boxes: a channels-last output must be 16-B aligned");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_ELEMWISE, st);
    const int64_t total = static_cast<int64_t>(N) * K * S * S * S;
    colored_boxes_kernel<<<grid_for(total), VZ_THREADS, 0, st>>>(colors, N, K, S, alpha, layout, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

extern "C" int tpx_primvolume_payload(const float* recon_param, int B, int P, int S, int mode, float* out, void* stream) {
    TPX_CHECK(recon_param != nullptr && out != nullptr, TPX_ERR_ARG, "tpx_primvolume_payload: null argument");
    TPX_CHECK(B >= 1 && P >= 1 && S >= 1 && S <= 64 && static_cast<int64_t>(B) * P < (int64_t(1) << 31), TPX_ERR_SHAPE,
              "tpx_primvolume_payload: bad shape (B %d P %d S %d)", B, P, S);
    TPX_CHECK(mode == TPX_PAYLOAD_RGB || mode == TPX_PAYLOAD_MAT, TPX_ERR_ARG, "tpx_primvolume_payload: unknown mode %d", mode);
    TPX_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, TPX_ERR_ARG, "tpx_primvolume_payload: output must be 16-B aligned");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_ELEMWISE, st);
    const int64_t total = static_cast<int64_t>(B) * P * S * S * S;
    primvolume_payload_kernel<<<grid_for(total), VZ_THREADS, 0, st>>>(recon_param, B * P, S, mode, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}
