// Ray-march preview of the primitive volume (SURVEY.md §8f-1, second half): the reference renders every 10th denoising step
// and the final turntable through `RayMarcher.forward` (dva/ray_marcher.py:142-229) = `compute_raydirs` (dva/mvp/extensions/
// utils/utils_kernel.cu:15-55) + `mvpraymarch` with the "fixedorder" hierarchy (dva/mvp/extensions/mvpraymarch/
// mvpraymarch_subset_kernel.h:14-101, utils.h:728-824, primtransf.h:104-131, primsampler.h:44-66, primaccum.h:63-79),
// an sm_70 torch extension.  One kernel here does both:
//   * ray set-up per pixel (origin / volradius, direction through the pinhole, slab range of the unit cube);
//   * per warp (the reference's 8 x 4-pixel warp of an 8 x 16 block — the hit list is a per-warp object in the reference and so
//     part of the result) the ASCENDING list of primitives whose box is hit by ANY ray of the warp, capped at 512 like the
//     reference's shared-memory list.  The reference walks a trivial 4095-node tree whose boxes prune next to nothing for
//     unsorted primitives; here the 32 lanes first cull the primitives' bounding spheres against the warp's ray cone (64
//     sphere tests per lane) and only the survivors get the exact per-ray slab test;
//   * the fixed-step march: start at the last step before the ray's first hit, visit the listed primitives at every step
//     (strictly-inside test in the primitive's frame, trilinear channels-last sample, alpha faded by exp(-fadescale * sum |y|^fadeexp)
//     with the fast-math intrinsics the reference is compiled with), additive alpha with saturation at 1.
// The first 96 listed primitives' transforms live in shared memory (the march re-reads them at every step).
#include "kernels.cuh"

namespace tpx {

namespace {

constexpr int RM_MAXHIT = 512;      // mvpraymarch(..., maxhitboxes=512)
constexpr int RM_CACHE = 96;        // listed primitives whose (pos, rot, scale) are cached in shared memory, per warp
constexpr int RM_BX = 8, RM_BY = 16;

struct RayMarchArgs {
    const float* tpl;        // [N, K, S, S, S, 4]
    const float* primpos;    // [N, K, 3]  (already divided by volradius)
    const float* primrot;    // [N, K, 3, 3]
    const float* primscale;  // [N, K, 3]
    const float* campos;     // [N, 3]
    const float* camrot;     // [N, 3, 3]
    const float* focal;      // [N, 2]
    const float* princpt;    // [N, 2]
    float* out;              // [N, H, W, 4]
    int N, K, S, H, W;
    float volradius, stepsize, fadescale, fadeexp;
};

struct Prim {
    float3 t, r0, r1, r2, s;
};

__device__ __forceinline__ float3 ld3(const float* p) { return make_float3(p[0], p[1], p[2]); }
__device__ __forceinline__ float3 operator*(float3 a, float b) { return make_float3(a.x * b, a.y * b, a.z * b); }
__device__ __forceinline__ float3 operator*(float3 a, float3 b) { return make_float3(a.x * b.x, a.y * b.y, a.z * b.z); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return make_float3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

__device__ __forceinline__ Prim load_prim(const RayMarchArgs& a, int n, int k) {
    Prim p;
    const size_t o = static_cast<size_t>(n) * a.K + k;
    p.t = ld3(a.primpos + o * 3);
    p.r0 = ld3(a.primrot + o * 9);
    p.r1 = ld3(a.primrot + o * 9 + 3);
    p.r2 = ld3(a.primrot + o * 9 + 6);
    p.s = ld3(a.primscale + o * 3);
    return p;
}

__global__ void __launch_bounds__(RM_BX * RM_BY) raymarch_preview_kernel(const RayMarchArgs a) {
    __shared__ int s_list[4][RM_MAXHIT];
    __shared__ float s_prim[4][RM_CACHE][16];
    const int lin = threadIdx.y * RM_BX + threadIdx.x;
    const int warp = lin >> 5, lane = lin & 31;
    int w = blockIdx.x * RM_BX + threadIdx.x, h = blockIdx.y * RM_BY + threadIdx.y;
    const int n = blockIdx.z;
    const bool live = w < a.W && h < a.H;
    w = min(w, a.W - 1);
    h = min(h, a.H - 1);                 // threads outside the image march a duplicate of the border ray (as in the reference)

    // ---- ray (compute_raydirs_forward_kernel) ----
    float3 raypos = ld3(a.campos + n * 3);
    raypos = make_float3(raypos.x / a.volradius, raypos.y / a.volradius, raypos.z / a.volradius);
    const float px = (static_cast<float>(w) - a.princpt[n * 2]) / a.focal[n * 2];
    const float py = (static_cast<float>(h) - a.princpt[n * 2 + 1]) / a.focal[n * 2 + 1];
    float3 raydir = ld3(a.camrot + n * 9) * px + ld3(a.camrot + n * 9 + 3) * py + ld3(a.camrot + n * 9 + 6);
    raydir = raydir * rsqrtf(dot3(raydir, raydir));
    float2 tminmax;
    {
        const float3 t1 = make_float3((-1.f - raypos.x) / raydir.x, (-1.f - raypos.y) / raydir.y, (-1.f - raypos.z) / raydir.z);
        const float3 t2 = make_float3((1.f - raypos.x) / raydir.x, (1.f - raypos.y) / raydir.y, (1.f - raypos.z) / raydir.z);
        const float tmin = fmaxf(fminf(t1.x, t2.x), fmaxf(fminf(t1.y, t2.y), fminf(t1.z, t2.z)));
        const float tmax = fminf(fmaxf(t1.x, t2.x), fminf(fmaxf(t1.y, t2.y), fmaxf(t1.z, t2.z)));
        tminmax = make_float2(fmaxf(tmin, 0.f), tmax);
    }

    // ---- the warp's ray cone (all rays share the origin) ----
    float3 axis = raydir;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        axis.x += __shfl_xor_sync(0xffffffffu, axis.x, o);
        axis.y += __shfl_xor_sync(0xffffffffu, axis.y, o);
        axis.z += __shfl_xor_sync(0xffffffffu, axis.z, o);
    }
    axis = axis * rsqrtf(dot3(axis, axis));
    float cmin = dot3(axis, raydir);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmin = fminf(cmin, __shfl_xor_sync(0xffffffffu, cmin, o));
    const float theta = acosf(fminf(cmin, 1.f)) + 1e-4f;

    // ---- hit list (ray_subset_fixedbvh semantics: any ray of the warp, ascending index, first RM_MAXHIT) ----
    int nhit = 0;
    float rtmin = INFINITY, rtmax = -INFINITY;
    for (int k0 = 0; k0 < a.K; k0 += 32) {
        const int kc = k0 + lane;
        bool cand = false;
        if (kc < a.K) {
            const size_t o = static_cast<size_t>(n) * a.K + kc;
            const float3 v = ld3(a.primpos + o * 3) - raypos;
            const float3 s = ld3(a.primscale + o * 3);
            const float rad = sqrtf(1.f / (s.x * s.x) + 1.f / (s.y * s.y) + 1.f / (s.z * s.z)) * 1.001f + 1e-6f;   // bounding sphere of the rotated box
            const float dist = sqrtf(dot3(v, v));
            if (dist <= rad) {
                cand = true;
            } else {
                const float phi = acosf(fminf(fmaxf(dot3(v, axis) / dist, -1.f), 1.f));
                cand = phi <= theta + asinf(fminf(rad / dist, 1.f)) + 1e-4f;
            }
        }
        unsigned m = __ballot_sync(0xffffffffu, cand);
        while (m != 0) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            const int k = k0 + b;
            const Prim p = load_prim(a, n, k);
            // PrimTransfSRT::forward2 + slab test in the primitive's frame
            const float3 xmt = raypos - p.t;
            const float3 r0 = (p.r0 * xmt.x + p.r1 * xmt.y + p.r2 * xmt.z) * p.s;
            const float3 rd = (p.r0 * raydir.x + p.r1 * raydir.y + p.r2 * raydir.z) * p.s;
            const float3 ird = make_float3(1.f / rd.x, 1.f / rd.y, 1.f / rd.z);
            const float3 t0 = make_float3((-1.f - r0.x) * ird.x, (-1.f - r0.y) * ird.y, (-1.f - r0.z) * ird.z);
            const float3 t1 = make_float3((1.f - r0.x) * ird.x, (1.f - r0.y) * ird.y, (1.f - r0.z) * ird.z);
            const float trmin = fmaxf(fminf(t0.x, t1.x), fmaxf(fminf(t0.y, t1.y), fminf(t0.z, t1.z)));
            const float trmax = fminf(fmaxf(t0.x, t1.x), fminf(fmaxf(t0.y, t1.y), fmaxf(t0.z, t1.z)));
            const bool hit = trmin <= trmax;
            if (hit) { rtmin = fminf(rtmin, trmin); rtmax = fmaxf(rtmax, trmax); }
            if (__any_sync(0xffffffffu, hit) && nhit < RM_MAXHIT) {
                if (lane == 0) s_list[warp][nhit] = k;
                ++nhit;
            }
        }
    }
    __syncwarp();
    for (int j = lane; j < min(nhit, RM_CACHE); j += 32) {
        const Prim p = load_prim(a, n, s_list[warp][j]);
        float* d = s_prim[warp][j];
        d[0] = p.t.x; d[1] = p.t.y; d[2] = p.t.z; d[3] = p.r0.x; d[4] = p.r0.y; d[5] = p.r0.z; d[6] = p.r1.x; d[7] = p.r1.y; d[8] = p.r1.z;
        d[9] = p.r2.x; d[10] = p.r2.y; d[11] = p.r2.z; d[12] = p.s.x; d[13] = p.s.y; d[14] = p.s.z;
    }
    __syncwarp();

    // ---- march (raymarch_subset_forward_kernel) ----
    const bool anyhit = rtmin <= rtmax;          // this ray hits at least one primitive (before clamping to the cube)
    rtmin = fmaxf(rtmin, tminmax.x);
    rtmax = fminf(rtmax, tminmax.y);
    float t = tminmax.x;
    float3 pos = raypos + raydir * tminmax.x;
    bool done = !anyhit;
    if (anyhit) {
        const float incs = floorf((rtmin - t) / a.stepsize);
        t += incs * a.stepsize;
        pos = pos + raydir * incs * a.stepsize;
    }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    const int S = a.S;
    const float hs = static_cast<float>(S - 1);
    while (!__all_sync(0xffffffffu, done || t > rtmax + 1e-5f)) {
        const bool active = !done && t < rtmax + 1e-5f;
        for (int ks = 0; ks < nhit; ++ks) {
            const int k = s_list[warp][ks];
            Prim p;
            if (ks < RM_CACHE) {
                const float* d = s_prim[warp][ks];
                p.t = make_float3(d[0], d[1], d[2]); p.r0 = make_float3(d[3], d[4], d[5]); p.r1 = make_float3(d[6], d[7], d[8]);
                p.r2 = make_float3(d[9], d[10], d[11]); p.s = make_float3(d[12], d[13], d[14]);
            } else {
                p = load_prim(a, n, k);
            }
            const float3 xmt = pos - p.t;
            const float3 y = (p.r0 * xmt.x + p.r1 * xmt.y + p.r2 * xmt.z) * p.s;
            const bool inside = y.x > -1.f && y.x < 1.f && y.y > -1.f && y.y < 1.f && y.z > -1.f && y.z < 1.f;
            if (inside && active && !done) {
                // trilinear channels-last sample (grid_sample_chlast_forward; strictly inside, so all eight corners exist)
                const float ix = (y.x + 1.f) * 0.5f * hs, iy = (y.y + 1.f) * 0.5f * hs, iz = (y.z + 1.f) * 0.5f * hs;
                const int x0 = min(static_cast<int>(floorf(ix)), S - 2), y0 = min(static_cast<int>(floorf(iy)), S - 2), z0 = min(static_cast<int>(floorf(iz)), S - 2);
                const float ax = ix - x0, ay = iy - y0, az = iz - z0;
                const float4* tp = reinterpret_cast<const float4*>(a.tpl) + (static_cast<size_t>(n) * a.K + k) * S * S * S + (z0 * S + y0) * S + x0;
                float4 smp = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int dz = c >> 2, dy = (c >> 1) & 1, dx = c & 1;
                    const float wgt = (dx ? ax : 1.f - ax) * (dy ? ay : 1.f - ay) * (dz ? az : 1.f - az);
                    const float4 v = __ldg(tp + (dz * S + dy) * S + dx);
                    smp.x = fmaf(v.x, wgt, smp.x); smp.y = fmaf(v.y, wgt, smp.y); smp.z = fmaf(v.z, wgt, smp.z); smp.w = fmaf(v.w, wgt, smp.w);
                }
                const float fade = __expf(-a.fadescale * (__powf(fabsf(y.x), a.fadeexp) + __powf(fabsf(y.y), a.fadeexp) + __powf(fabsf(y.z), a.fadeexp)));
                const float alpha = smp.w * fade;
                // PrimAccumAdditive::forward_prim
                const float newalpha = acc.w + alpha * a.stepsize;
                const float contrib = fminf(newalpha, 1.f) - acc.w;
                acc.x = fmaf(smp.x, contrib, acc.x); acc.y = fmaf(smp.y, contrib, acc.y); acc.z = fmaf(smp.z, contrib, acc.z); acc.w += contrib;
                if (newalpha >= 1.f) done = true;
            }
        }
        t += a.stepsize;
        pos = pos + raydir * a.stepsize;
    }
    if (live) *reinterpret_cast<float4*>(a.out + ((static_cast<size_t>(n) * a.H + h) * a.W + w) * 4) = acc;
}

}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" int tpx_raymarch_preview(const float* tpl, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                                    const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius,
                                    float stepsize, float fadescale, float fadeexp, float* out, void* stream) {
    TPX_CHECK(tpl != nullptr && primpos != nullptr && primrot != nullptr && primscale != nullptr && campos != nullptr && camrot != nullptr && focal != nullptr &&
                  princpt != nullptr && out != nullptr,
              TPX_ERR_ARG, "raymarch_preview: null argument");
    TPX_CHECK(N > 0 && K > 0 && S >= 2 && S <= 64 && H > 0 && W > 0 && N <= 65535, TPX_ERR_SHAPE, "raymarch: bad geometry (N %d K %d S %d %d x %d)", N, K, S, H, W);
    TPX_CHECK(stepsize > 0.f && volradius > 0.f, TPX_ERR_ARG, "raymarch: step size and volume radius must be positive");
    TPX_CHECK((reinterpret_cast<uintptr_t>(tpl) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, TPX_ERR_ARG, "raymarch: template / output must be 16-B aligned");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    RayMarchArgs a{tpl, primpos, primrot, primscale, campos, camrot, focal, princpt, out, N, K, S, H, W, volradius, stepsize, fadescale, fadeexp};
    const dim3 grid((W + RM_BX - 1) / RM_BX, (H + RM_BY - 1) / RM_BY, N), block(RM_BX, RM_BY);
    raymarch_preview_kernel<<<grid, block, 0, st>>>(a);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}
