// Ray-march preview of the primitive volume (SURVEY.md §8f-1, second half): the reference renders every 10th denoising step
// and the final turntable through `RayMarcher.forward` (dva/ray_marcher.py:142-229) = `compute_raydirs` (dva/mvp/extensions/
// utils/utils_kernel.cu:15-55) + `mvpraymarch` with the "fixedorder" hierarchy (dva/mvp/extensions/mvpraymarch/
// mvpraymarch_subset_kernel.h:14-101, utils.h:728-824, primtransf.h:104-131, primsampler.h:44-66, primaccum.h:63-79),
// an sm_70 torch extension.  One kernel here does both:
//   * ray set-up per pixel (origin / volradius, direction through the pinhole, slab range of the unit cube);
//   * per warp (the reference's 8 x 4-pixel warp of an 8 x 16 block — the hit list is a per-warp object in the reference and so
//     part of the result) the list of primitives whose box is hit by ANY ray of the warp, in the reference's tree order (ascending
//     index rotated by 2^ceil(log2 K) - K; see the hit-list scan), capped at 512 like the reference's shared-memory list.  The
//     reference walks a trivial (2K - 1)-node tree whose boxes prune next to nothing for unsorted primitives; here the 32 lanes first
//     cull the primitives' bounding spheres against the warp's ray cone (64 sphere tests per lane at K = 2048) and only the
//     survivors get the exact per-ray slab test;
//   * the fixed-step march: start at the last step before the ray's first hit, visit the listed primitives at every step
//     (strictly-inside test in the primitive's frame, trilinear channels-last sample, alpha faded by exp(-fadescale * sum |y|^fadeexp)
//     with the fast-math intrinsics the reference is compiled with), additive alpha with saturation at 1.
// The first 96 listed primitives' transforms live in shared memory (the march re-reads them at every step).
// The same kernel, instantiated with GRAD, is the backward (raymarch_subset_backward_kernel, mvpraymarch_subset_kernel.h:103-217, with
// forwarddir = true): it rebuilds the hit list, re-marches from the same first step through the SAME device code (so every inside test,
// saturation and step count is the forward's), and per listed primitive and step applies PrimAccumAdditive::forwardbackward_prim
// (primaccum.h:81-98), PrimSamplerTW<false>::backward (primsampler.h:68-91) and PrimTransfSRT::backward (primtransf.h:155-179):
//   * the template gradient is a trilinear scatter, one sm_90 vector reduction (atomicAdd(float4*) -> RED.E.ADD.F32x4) per corner;
//   * the 15 transform partials are summed over the warp with shuffles (all 32 lanes visit the same primitive at the same step) and
//     lanes 0..14 each issue one reduction.
// Subsampled rays (ray_subsample_factor > 1): output pixel (j, i) traces the ray through image pixel (x0 + stride j, y0 + stride i).
// Views (tpx_raymarch_preview_views): image n reads primitive set n / views and camera n, so a turntable of one primitive set is one
// launch over one template.
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
    float* out;              // [N, H, W, 4]  (forward)
    int N, K, S, H, W;       // H, W: the marched (subsampled) image
    float volradius, stepsize, fadescale, fadeexp;
    int stride;              // image pixel = offset + stride * output pixel
    const int* offsets;      // [N, 2] (x0, y0), or null for (0, 0)
    float* raysat;           // forward: [N, H, W, 3] colour of the saturating sample, (-1,-1,-1) if none; may be null.  backward: read
    const float* grad_out;   // backward: [N, H, W, 4]
    float* grad_tpl;         // backward, accumulated: [N, K, S, S, S, 4]
    float* grad_pos;         // [N, K, 3]
    float* grad_rot;         // [N, K, 3, 3]
    float* grad_scale;       // [N, K, 3]
    int views;               // image n marches primitive set n / views (the [N, K, ...] arrays above hold N / views sets)
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

template <bool GRAD>
__global__ void __launch_bounds__(RM_BX * RM_BY) raymarch_kernel(const RayMarchArgs a) {
    __shared__ int s_list[4][RM_MAXHIT];
    __shared__ float s_prim[4][RM_CACHE][16];
    const int lin = threadIdx.y * RM_BX + threadIdx.x;
    const int warp = lin >> 5, lane = lin & 31;
    int w = blockIdx.x * RM_BX + threadIdx.x, h = blockIdx.y * RM_BY + threadIdx.y;
    const int n = blockIdx.z, np = n / a.views;   // image (camera, output) and primitive set
    const bool live = w < a.W && h < a.H;
    w = min(w, a.W - 1);
    h = min(h, a.H - 1);                 // threads outside the image march a duplicate of the border ray (as in the reference)

    // ---- ray (compute_raydirs_forward_kernel) ----
    float3 raypos = ld3(a.campos + n * 3);
    raypos = make_float3(raypos.x / a.volradius, raypos.y / a.volradius, raypos.z / a.volradius);
    const int ox = a.offsets ? a.offsets[n * 2] : 0, oy = a.offsets ? a.offsets[n * 2 + 1] : 0;
    const float px = (static_cast<float>(ox + a.stride * w) - a.princpt[n * 2]) / a.focal[n * 2];
    const float py = (static_cast<float>(oy + a.stride * h) - a.princpt[n * 2 + 1]) / a.focal[n * 2 + 1];
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

    // ---- hit list (ray_subset_fixedbvh semantics: any ray of the warp, the tree's leaf order, first RM_MAXHIT) ----
    // The reference walks the implicit heap of build_accel(fixedorder=True) depth-first, left child first, and appends each leaf as it
    // is reached; leaf node i is primitive i - (K - 1).  Left to right, the leaves are the deeper level's first, so the list order is
    // ascending order rotated by r = 2^ceil(log2 K) - K: r, ..., K - 1, 0, ..., r - 1 (ascending when K is a power of two).  Scan
    // position j visits primitive (j + r) mod K.  The order decides which primitives a warp over the cap keeps and which primitive a
    // saturating step's colour comes from.
    const int rot = (1 << (32 - __clz(a.K - 1))) - a.K;
    int nhit = 0;
    float rtmin = INFINITY, rtmax = -INFINITY;
    for (int k0 = 0; k0 < a.K; k0 += 32) {
        const int kc = k0 + lane + rot < a.K ? k0 + lane + rot : k0 + lane + rot - a.K;
        bool cand = false;
        if (k0 + lane < a.K) {
            const size_t o = static_cast<size_t>(np) * a.K + kc;
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
            const int k = k0 + b + rot < a.K ? k0 + b + rot : k0 + b + rot - a.K;
            const Prim p = load_prim(a, np, k);
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
        const Prim p = load_prim(a, np, s_list[warp][j]);
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
    const size_t pix = (static_cast<size_t>(n) * a.H + h) * a.W + w;
    float3 satrgb = make_float3(-1.f, -1.f, -1.f);   // forward: PrimAccumAdditive's raysat; backward: read back
    float4 dL = make_float4(0.f, 0.f, 0.f, 0.f);     // backward: upstream gradient of this ray (zero for the border duplicates)
    if (GRAD) {
        satrgb = ld3(a.raysat + pix * 3);
        if (live) dL = *reinterpret_cast<const float4*>(a.grad_out + pix * 4);
    }
    const bool rsat = satrgb.x > -1.f;               // the ray saturates somewhere (the reference's test, primaccum.h:92)
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
                p = load_prim(a, np, k);
            }
            const float3 xmt = pos - p.t;
            const float3 y = (p.r0 * xmt.x + p.r1 * xmt.y + p.r2 * xmt.z) * p.s;
            const bool inside = y.x > -1.f && y.x < 1.f && y.y > -1.f && y.y < 1.f && y.z > -1.f && y.z < 1.f;
            const bool eval = inside && active && !done;
            float gs[15];                                // backward: d/dscale (3), d/drot (9, row-major), d/dpos (3) of this sample
            if (GRAD) {
#pragma unroll
                for (int i = 0; i < 15; ++i) gs[i] = 0.f;
            }
            if (eval) {
                // trilinear channels-last sample (grid_sample_chlast_forward; strictly inside, so all eight corners exist)
                const float ix = (y.x + 1.f) * 0.5f * hs, iy = (y.y + 1.f) * 0.5f * hs, iz = (y.z + 1.f) * 0.5f * hs;
                const int x0 = min(static_cast<int>(floorf(ix)), S - 2), y0 = min(static_cast<int>(floorf(iy)), S - 2), z0 = min(static_cast<int>(floorf(iz)), S - 2);
                const float ax = ix - x0, ay = iy - y0, az = iz - z0;
                const float4* tp = reinterpret_cast<const float4*>(a.tpl) + (static_cast<size_t>(np) * a.K + k) * S * S * S + (z0 * S + y0) * S + x0;
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
                if (GRAD) {
                    // PrimAccumAdditive::forwardbackward_prim: this sample saturates iff the forward's newalpha >= 1 (same operands)
                    const bool sat = newalpha >= 1.f;
                    const float wgt_rgb = sat ? 1.f - acc.w : __fmul_rn(alpha, a.stepsize);
                    const float dla = sat ? 0.f
                                          : a.stepsize * ((smp.x - (rsat ? satrgb.x : 0.f)) * dL.x + (smp.y - (rsat ? satrgb.y : 0.f)) * dL.y +
                                                          (smp.z - (rsat ? satrgb.z : 0.f)) * dL.z + (rsat ? 0.f : dL.w));
                    // PrimSamplerTW<false>::backward: fade, then the trilinear scatter and its position gradient
                    const float cf = -(a.fadescale * a.fadeexp) * alpha * dla;
                    const float fe1 = a.fadeexp - 1.f;
                    float3 dy = make_float3(cf * __powf(fabsf(y.x), fe1) * (y.x > 0.f ? 1.f : -1.f), cf * __powf(fabsf(y.y), fe1) * (y.y > 0.f ? 1.f : -1.f),
                                            cf * __powf(fabsf(y.z), fe1) * (y.z > 0.f ? 1.f : -1.f));
                    const float4 g = make_float4(wgt_rgb * dL.x, wgt_rgb * dL.y, wgt_rgb * dL.z, dla * fade);
                    float4* gtp = reinterpret_cast<float4*>(a.grad_tpl) + (static_cast<size_t>(np) * a.K + k) * S * S * S + (z0 * S + y0) * S + x0;
                    float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        const int dz = c >> 2, dy_ = (c >> 1) & 1, dx = c & 1;
                        const float wx = dx ? ax : 1.f - ax, wy = dy_ ? ay : 1.f - ay, wz = dz ? az : 1.f - az;
                        const float4 v = __ldg(tp + (dz * S + dy_) * S + dx);
                        const float gv = v.x * g.x + v.y * g.y + v.z * g.z + v.w * g.w;
                        gx += (dx ? gv : -gv) * wy * wz;
                        gy += (dy_ ? gv : -gv) * wx * wz;
                        gz += (dz ? gv : -gv) * wx * wy;
                        const float wgt = wx * wy * wz;
                        if (live) atomicAdd(gtp + (dz * S + dy_) * S + dx, make_float4(g.x * wgt, g.y * wgt, g.z * wgt, g.w * wgt));
                    }
                    dy.x += gx * (0.5f * hs); dy.y += gy * (0.5f * hs); dy.z += gz * (0.5f * hs);
                    // PrimTransfSRT::backward
                    const float3 rx = p.r0 * xmt.x + p.r1 * xmt.y + p.r2 * xmt.z;
                    gs[0] = rx.x * dy.x; gs[1] = rx.y * dy.y; gs[2] = rx.z * dy.z;
                    dy = dy * p.s;
                    gs[3] = xmt.x * dy.x; gs[4] = xmt.x * dy.y; gs[5] = xmt.x * dy.z;
                    gs[6] = xmt.y * dy.x; gs[7] = xmt.y * dy.y; gs[8] = xmt.y * dy.z;
                    gs[9] = xmt.z * dy.x; gs[10] = xmt.z * dy.y; gs[11] = xmt.z * dy.z;
                    gs[12] = -dot3(p.r0, dy); gs[13] = -dot3(p.r1, dy); gs[14] = -dot3(p.r2, dy);
                }
                acc.x = fmaf(smp.x, contrib, acc.x); acc.y = fmaf(smp.y, contrib, acc.y); acc.z = fmaf(smp.z, contrib, acc.z); acc.w += contrib;
                if (newalpha >= 1.f) {
                    if (!GRAD) satrgb = make_float3(smp.x, smp.y, smp.z);
                    done = true;
                }
            }
            if (GRAD && __any_sync(0xffffffffu, eval)) {
                // one warp-wide sum per partial; lane i < 15 then holds partial i and issues its reduction
                float mine = 0.f;
#pragma unroll
                for (int i = 0; i < 15; ++i) {
                    float v = gs[i];
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    if (lane == i) mine = v;
                }
                const size_t o = static_cast<size_t>(np) * a.K + k;
                float* dst = lane < 3 ? a.grad_scale + o * 3 + lane : lane < 12 ? a.grad_rot + o * 9 + (lane - 3) : a.grad_pos + o * 3 + (lane - 12);
                if (lane < 15 && mine != 0.f) atomicAdd(dst, mine);
            }
        }
        t += a.stepsize;
        pos = pos + raydir * a.stepsize;
    }
    if (!GRAD && live) {
        *reinterpret_cast<float4*>(a.out + pix * 4) = acc;
        if (a.raysat) { a.raysat[pix * 3] = satrgb.x; a.raysat[pix * 3 + 1] = satrgb.y; a.raysat[pix * 3 + 2] = satrgb.z; }
    }
}

int raymarch_check(const RayMarchArgs& a, int H, int W) {
    TPX_CHECK(a.tpl != nullptr && a.primpos != nullptr && a.primrot != nullptr && a.primscale != nullptr && a.campos != nullptr && a.camrot != nullptr &&
                  a.focal != nullptr && a.princpt != nullptr,
              TPX_ERR_ARG, "raymarch: null argument");
    TPX_CHECK(a.N > 0 && a.K > 0 && a.S >= 2 && a.S <= 64 && H > 0 && W > 0 && a.N <= 65535, TPX_ERR_SHAPE, "raymarch: bad geometry (N %d K %d S %d %d x %d)", a.N,
              a.K, a.S, H, W);
    TPX_CHECK(a.stride >= 1 && a.H >= 1 && a.W >= 1, TPX_ERR_SHAPE, "raymarch: stride %d leaves a %d x %d image of %d x %d", a.stride, a.H, a.W, H, W);
    TPX_CHECK(a.views >= 1 && a.N % a.views == 0, TPX_ERR_SHAPE, "raymarch: %d views do not divide %d images", a.views, a.N);
    TPX_CHECK(a.stepsize > 0.f && a.volradius > 0.f, TPX_ERR_ARG, "raymarch: step size and volume radius must be positive");
    TPX_CHECK((reinterpret_cast<uintptr_t>(a.tpl) & 15) == 0, TPX_ERR_ARG, "raymarch: template must be 16-B aligned");
    return TPX_OK;
}

template <bool GRAD>
int raymarch_launch(const RayMarchArgs& a, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    const dim3 grid((a.W + RM_BX - 1) / RM_BX, (a.H + RM_BY - 1) / RM_BY, a.N), block(RM_BX, RM_BY);
    raymarch_kernel<GRAD><<<grid, block, 0, st>>>(a);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" int tpx_raymarch_preview(const float* tpl, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                                    const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius,
                                    float stepsize, float fadescale, float fadeexp, float* out, void* stream) {
    return tpx_raymarch_forward(tpl, primpos, primrot, primscale, campos, camrot, focal, princpt, N, K, S, H, W, volradius, stepsize, fadescale, fadeexp, 1,
                                nullptr, out, nullptr, stream);
}

extern "C" int tpx_raymarch_preview_views(const float* tpl, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                                          const float* camrot, const float* focal, const float* princpt, int N, int views, int K, int S, int H, int W,
                                          float volradius, float stepsize, float fadescale, float fadeexp, float* out, void* stream) {
    const RayMarchArgs a{tpl, primpos, primrot, primscale, campos, camrot, focal, princpt, out, N, K, S, H, W, volradius, stepsize, fadescale, fadeexp,
                         1, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, views};
    TPX_CHECK(out != nullptr, TPX_ERR_ARG, "raymarch: null argument");
    if (const int rc = raymarch_check(a, H, W)) return rc;
    TPX_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, TPX_ERR_ARG, "raymarch: output must be 16-B aligned");
    TPX_DEVICE_GUARD();
    return raymarch_launch<false>(a, stream);
}

extern "C" int tpx_raymarch_forward(const float* tpl, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                                    const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius,
                                    float stepsize, float fadescale, float fadeexp, int stride, const int* offsets, float* out, float* raysat_out, void* stream) {
    const int h = stride >= 1 ? H / stride : 0, w = stride >= 1 ? W / stride : 0;
    const RayMarchArgs a{tpl, primpos, primrot, primscale, campos, camrot, focal, princpt, out, N, K, S, h, w, volradius, stepsize, fadescale, fadeexp,
                         stride, offsets, raysat_out, nullptr, nullptr, nullptr, nullptr, nullptr, 1};
    TPX_CHECK(out != nullptr, TPX_ERR_ARG, "raymarch: null argument");
    if (const int rc = raymarch_check(a, H, W)) return rc;
    TPX_CHECK((reinterpret_cast<uintptr_t>(out) & 15) == 0, TPX_ERR_ARG, "raymarch: output must be 16-B aligned");
    TPX_DEVICE_GUARD();
    return raymarch_launch<false>(a, stream);
}

extern "C" int tpx_raymarch_backward(const float* tpl, const float* primpos, const float* primrot, const float* primscale, const float* campos,
                                     const float* camrot, const float* focal, const float* princpt, int N, int K, int S, int H, int W, float volradius,
                                     float stepsize, float fadescale, float fadeexp, int stride, const int* offsets, const float* raysat,
                                     const float* grad_rgba, float* grad_tpl, float* grad_primpos, float* grad_primrot, float* grad_primscale, void* stream) {
    const int h = stride >= 1 ? H / stride : 0, w = stride >= 1 ? W / stride : 0;
    const RayMarchArgs a{tpl, primpos, primrot, primscale, campos, camrot, focal, princpt, nullptr, N, K, S, h, w, volradius, stepsize, fadescale, fadeexp,
                         stride, offsets, const_cast<float*>(raysat), grad_rgba, grad_tpl, grad_primpos, grad_primrot, grad_primscale, 1};
    TPX_CHECK(raysat != nullptr && grad_rgba != nullptr && grad_tpl != nullptr && grad_primpos != nullptr && grad_primrot != nullptr && grad_primscale != nullptr,
              TPX_ERR_ARG, "raymarch: null argument");
    if (const int rc = raymarch_check(a, H, W)) return rc;
    TPX_CHECK((reinterpret_cast<uintptr_t>(grad_rgba) & 15) == 0 && (reinterpret_cast<uintptr_t>(grad_tpl) & 15) == 0, TPX_ERR_ARG,
              "raymarch: output gradient / template gradient must be 16-B aligned");
    TPX_DEVICE_GUARD();
    return raymarch_launch<true>(a, stream);
}
