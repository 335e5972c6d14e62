// Texture bake (the back half of extract_texmesh, inference.py:163-211): UV-space rasteriser and attribute interpolation standing
// behind nvdiffrast's dr.rasterize / dr.interpolate as called there, and the nearest-texel seam padding standing behind the
// scipy / scikit-learn block.  The fused texel query that sits between them is primsdf_bake_kernel in primsdf.cu.  Plain FP32 /
// integer SIMT: this is coverage testing and gather work.
#include "bake_interp.cuh"
#include "kernels.cuh"

namespace tpx {

namespace {
// =====================================================================================================================
// Rasteriser.  Contract (the tests hold it to a float64 restatement):
//   * texel (row i, col j) is sampled at its centre; row 0 is v = 0.  Everything is evaluated in texel units relative to the
//     centre, X = u W - (j + 1/2), Y = v H - (i + 1/2) (one fused rounding each): the NDC form x = 2 u - 1 against
//     (j + 1/2) / W 2 - 1 scaled by W H / 4, which changes neither a sign nor a barycentric ratio;
//   * the edge function of edge (a, b) at the centre is cross(a - p, b - p), evaluated with the endpoints ordered by (x, y) and
//     negated when that swapped them, so the two triangles sharing an edge see exactly opposite values: a centre on a shared
//     edge belongs to both, a centre beside it to exactly one, never to none;
//   * orientation is the sign of cross(v1 - v0, v2 - v0); zero (or non-finite) area and out-of-range indices skip the triangle;
//     a texel is covered iff all three oriented edge functions are >= 0; the lowest covering triangle index wins (atomicMin);
//   * (u, v) = (e12, e20) / (e01 + e12 + e20): the weights of vertices 0 and 1.
// One thread per triangle walks bounding boxes of up to RB_SMALL texels; larger boxes are handed to the whole block, and
// to the RB_SPLIT blocks along grid.y, which take interleaved row bands of them.
// =====================================================================================================================
constexpr int RB_THREADS = 256;
constexpr int RB_SMALL = 1024;
constexpr int RB_SPLIT = 16;
constexpr unsigned RB_EMPTY = 0xffffffffu;

struct RastTri {
    float x[3], y[3];
    float sign;             // +1 / -1: orientation
    int j0, j1, i0, i1;     // conservative texel bounding box, clipped to the atlas (empty if j1 < j0 or i1 < i0)
};

__device__ __forceinline__ bool load_tri(const float* __restrict__ vt, long long Nt, const int* __restrict__ ft, long long t, int H, int W, RastTri& r) {
    const float Wf = static_cast<float>(W), Hf = static_cast<float>(H);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int idx = ft[3 * t + c];
        if (idx < 0 || idx >= Nt) return false;
        r.x[c] = vt[2 * static_cast<long long>(idx)];
        r.y[c] = vt[2 * static_cast<long long>(idx) + 1];
    }
    const float ax = __fmul_rn(__fsub_rn(r.x[1], r.x[0]), Wf), ay = __fmul_rn(__fsub_rn(r.y[1], r.y[0]), Hf);
    const float bx = __fmul_rn(__fsub_rn(r.x[2], r.x[0]), Wf), by = __fmul_rn(__fsub_rn(r.y[2], r.y[0]), Hf);
    const float area = __fmaf_rn(ax, by, -__fmul_rn(ay, bx));
    if (!(fabsf(area) > 0.f) || isinf(area)) return false;      // zero area, NaN or overflow
    r.sign = area > 0.f ? 1.f : -1.f;
    const float xmin = fminf(r.x[0], fminf(r.x[1], r.x[2])) * Wf - 0.5f, xmax = fmaxf(r.x[0], fmaxf(r.x[1], r.x[2])) * Wf - 0.5f;
    const float ymin = fminf(r.y[0], fminf(r.y[1], r.y[2])) * Hf - 0.5f, ymax = fmaxf(r.y[0], fmaxf(r.y[1], r.y[2])) * Hf - 0.5f;
    r.j0 = __float2int_rd(fminf(fmaxf(xmin, 0.f), Wf));
    r.j1 = min(__float2int_ru(fminf(fmaxf(xmax, -1.f), Wf)), W - 1);
    r.i0 = __float2int_rd(fminf(fmaxf(ymin, 0.f), Hf));
    r.i1 = min(__float2int_ru(fminf(fmaxf(ymax, -1.f), Hf)), H - 1);
    return true;
}

__device__ __forceinline__ float edge_fn(float ax, float ay, float bx, float by, float cx, float cy, float Wf, float Hf) {
    const bool swap = bx < ax || (bx == ax && by < ay);
    const float lx = swap ? bx : ax, ly = swap ? by : ay, hx = swap ? ax : bx, hy = swap ? ay : by;
    const float Ax = __fmaf_rn(lx, Wf, -cx), Ay = __fmaf_rn(ly, Hf, -cy);
    const float Bx = __fmaf_rn(hx, Wf, -cx), By = __fmaf_rn(hy, Hf, -cy);
    const float e = __fmaf_rn(Ax, By, -__fmul_rn(Ay, Bx));
    return swap ? -e : e;
}

// oriented edge functions of triangle r at the centre of texel (i, j): e[0] opposite vertex 0 (edge 1-2), e[1] opposite vertex 1, e[2]
__device__ __forceinline__ void tri_edges(const RastTri& r, int i, int j, float Wf, float Hf, float e[3]) {
    const float cx = static_cast<float>(j) + 0.5f, cy = static_cast<float>(i) + 0.5f;
    e[0] = r.sign * edge_fn(r.x[1], r.y[1], r.x[2], r.y[2], cx, cy, Wf, Hf);
    e[1] = r.sign * edge_fn(r.x[2], r.y[2], r.x[0], r.y[0], cx, cy, Wf, Hf);
    e[2] = r.sign * edge_fn(r.x[0], r.y[0], r.x[1], r.y[1], cx, cy, Wf, Hf);
}

__device__ __forceinline__ void test_texel(const RastTri& r, unsigned t, int i, int j, int W, float Wf, float Hf, unsigned* __restrict__ winner) {
    float e[3];
    tri_edges(r, i, j, Wf, Hf, e);
    if (e[0] >= 0.f && e[1] >= 0.f && e[2] >= 0.f) atomicMin(winner + static_cast<size_t>(i) * W + j, t);
}

__global__ void __launch_bounds__(RB_THREADS) uv_raster_kernel(const float* __restrict__ vt, long long Nt, const int* __restrict__ ft, long long F, int H, int W,
                                                               unsigned* __restrict__ winner) {
    __shared__ int s_large[RB_THREADS];
    __shared__ int s_n;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const float Wf = static_cast<float>(W), Hf = static_cast<float>(H);
    const long long t = static_cast<long long>(blockIdx.x) * RB_THREADS + threadIdx.x;
    RastTri r;
    if (t < F && load_tri(vt, Nt, ft, t, H, W, r) && r.j1 >= r.j0 && r.i1 >= r.i0) {
        const long long n = static_cast<long long>(r.j1 - r.j0 + 1) * (r.i1 - r.i0 + 1);
        if (n > RB_SMALL) {
            s_large[atomicAdd(&s_n, 1)] = threadIdx.x;
        } else if (blockIdx.y == 0) {
            for (int i = r.i0; i <= r.i1; ++i)
                for (int j = r.j0; j <= r.j1; ++j) test_texel(r, static_cast<unsigned>(t), i, j, W, Wf, Hf, winner);
        }
    }
    __syncthreads();
    const int n_large = s_n;            // the order of the list varies from run to run; atomicMin makes the result independent of it
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int WARPS = RB_THREADS / 32;
    for (int q = 0; q < n_large; ++q) {
        const long long tl = static_cast<long long>(blockIdx.x) * RB_THREADS + s_large[q];
        load_tri(vt, Nt, ft, tl, H, W, r);
        for (int i = r.i0 + blockIdx.y * WARPS + warp; i <= r.i1; i += WARPS * RB_SPLIT)
            for (int j = r.j0 + lane; j <= r.j1; j += 32) test_texel(r, static_cast<unsigned>(tl), i, j, W, Wf, Hf, winner);
    }
}

// winner -> rast (u, v, 0, id + 1); empty texels get zeros and winner -1
__global__ void __launch_bounds__(RB_THREADS) uv_resolve_kernel(const float* __restrict__ vt, long long Nt, const int* __restrict__ ft, int H, int W,
                                                                int* __restrict__ winner, float4* __restrict__ rast) {
    const long long p = static_cast<long long>(blockIdx.x) * RB_THREADS + threadIdx.x;
    if (p >= static_cast<long long>(H) * W) return;
    const unsigned t = static_cast<unsigned>(winner[p]);
    RastTri r;
    if (t == RB_EMPTY || !load_tri(vt, Nt, ft, t, H, W, r)) {
        winner[p] = -1;
        rast[p] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    float e[3];
    tri_edges(r, static_cast<int>(p / W), static_cast<int>(p % W), static_cast<float>(W), static_cast<float>(H), e);
    const float sum = __fadd_rn(__fadd_rn(e[0], e[1]), e[2]);
    rast[p] = make_float4(__fdiv_rn(e[0], sum), __fdiv_rn(e[1], sum), 0.f, static_cast<float>(t + 1u));
}

__global__ void __launch_bounds__(RB_THREADS) rast_interpolate_kernel(const float* __restrict__ attr, long long Nv, int C, const int* __restrict__ tri, long long F,
                                                                      const float4* __restrict__ rast, long long n, float* __restrict__ out) {
    const long long p = static_cast<long long>(blockIdx.x) * RB_THREADS + threadIdx.x;
    if (p >= n) return;
    const float4 r = rast[p];
    const int t = rast_triangle(r.w);
    float* o = out + p * C;
    long long i0 = -1, i1 = -1, i2 = -1;
    if (t >= 0 && t < F) { i0 = tri[3 * static_cast<long long>(t)]; i1 = tri[3 * static_cast<long long>(t) + 1]; i2 = tri[3 * static_cast<long long>(t) + 2]; }
    if (i0 < 0 || i1 < 0 || i2 < 0 || i0 >= Nv || i1 >= Nv || i2 >= Nv) {
        for (int c = 0; c < C; ++c) o[c] = 0.f;
        return;
    }
    const float *a0 = attr + i0 * C, *a1 = attr + i1 * C, *a2 = attr + i2 * C;
    for (int c = 0; c < C; ++c) o[c] = bary_interp(r.x, r.y, a0[c], a1[c], a2[c]);
}

// =====================================================================================================================
// Seam padding (inference.py:200-211).  Every texel outside the mask whose L1 (4-connected) distance to the mask is <= P takes the
// value of the Euclidean-nearest mask texel; ties go to the smallest (row, col).  This equals the reference's result exactly:
//   * binary_dilation with the default cross element iterated P times grows the mask by the L1 ball of radius P, so its
//     inpaint_region is { not mask, L1 distance <= P };
//   * its search set (mask minus the 3-fold erosion of mask) contains every mask texel with a non-mask 4-neighbour, and the
//     Euclidean-nearest mask texel of a non-mask texel always has one: otherwise its neighbour toward the query would be a mask
//     texel strictly closer.  So nearest-in-search-set = nearest-in-mask;
//   * L1 distance <= P bounds the Euclidean distance by P, so the nearest mask texel lies within |dx|, |dy| <= P.
// Two exact integer passes: per row, the signed offset to the nearest mask column within +-P (left wins a tie); per column,
// the minimum over |dy| <= P of dy^2 + dx^2 (rows ascending, strict <: the smallest row wins, then the smaller column).  Where the
// kd-tree of the reference meets equidistant texels its choice is unspecified; this one is fixed.
// =====================================================================================================================
constexpr short IP_NONE = 0x7fff;
constexpr int IP_MAX_PAD = 8192;

__global__ void __launch_bounds__(RB_THREADS) inpaint_rows_kernel(const uint8_t* __restrict__ mask, int H, int W, int P, short* __restrict__ rowd) {
    const long long p = static_cast<long long>(blockIdx.x) * RB_THREADS + threadIdx.x;
    if (p >= static_cast<long long>(H) * W) return;
    const int j = static_cast<int>(p % W);
    const uint8_t* row = mask + (p - j);
    short best = IP_NONE;
    for (int d = 0; d <= P; ++d) {
        if (j - d >= 0 && row[j - d]) { best = static_cast<short>(-d); break; }
        if (j + d < W && row[j + d]) { best = static_cast<short>(d); break; }
    }
    rowd[p] = best;
}

__global__ void __launch_bounds__(RB_THREADS) inpaint_cols_kernel(const uint8_t* __restrict__ mask, const short* __restrict__ rowd, int H, int W, int C, int P,
                                                                  float* __restrict__ feats, int* __restrict__ src) {
    const long long p = static_cast<long long>(blockIdx.x) * RB_THREADS + threadIdx.x;
    if (p >= static_cast<long long>(H) * W) return;
    const int i = static_cast<int>(p / W), j = static_cast<int>(p % W);
    int best_d2 = 0x7fffffff, best_l1 = 0x7fffffff, best_src = -1;
    if (!mask[p]) {
        for (int r = max(i - P, 0); r <= min(i + P, H - 1); ++r) {
            const int dx = rowd[static_cast<size_t>(r) * W + j];
            if (dx == IP_NONE) continue;
            const int dy = r - i;
            const int d2 = dy * dy + dx * dx;
            best_l1 = min(best_l1, abs(dy) + abs(dx));
            if (d2 < best_d2) { best_d2 = d2; best_src = r * W + j + dx; }
        }
        if (best_l1 > P) best_src = -1;
    }
    if (src != nullptr) src[p] = best_src;
    if (best_src < 0) return;
    const float* s = feats + static_cast<size_t>(best_src) * C;     // a mask texel: never written by this kernel
    float* o = feats + static_cast<size_t>(p) * C;
    for (int c = 0; c < C; ++c) o[c] = s[c];
}

bool atlas_ok(int H, int W) { return H >= 1 && W >= 1 && H <= 8192 && W <= 8192; }
unsigned texel_blocks(int H, int W) { return static_cast<unsigned>((static_cast<long long>(H) * W + RB_THREADS - 1) / RB_THREADS); }
}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" {

int tpx_uv_rasterize(const float* vt, int64_t Nt, const int32_t* ft, int64_t F, int H, int W, float* rast, int32_t* winner, void* stream) {
    TPX_CHECK(rast != nullptr && winner != nullptr && (F == 0 || (vt != nullptr && ft != nullptr)), TPX_ERR_ARG, "uv_rasterize: null argument");
    TPX_CHECK(atlas_ok(H, W), TPX_ERR_SHAPE, "uv_rasterize: atlas %d x %d (1..8192 each)", H, W);
    // channel 3 of rast carries triangle id + 1 as a float, exact up to 2^24
    TPX_CHECK(F >= 0 && F < (1LL << 24) && Nt >= 0 && Nt < (1LL << 31), TPX_ERR_SHAPE, "uv_rasterize: %lld triangles / %lld vertices (F < 2^24, Nt < 2^31)",
              (long long)F, (long long)Nt);
    TPX_CHECK((reinterpret_cast<uintptr_t>(rast) & 15) == 0, TPX_ERR_ARG, "uv_rasterize: rast must be 16-B aligned");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    TPX_CUDA(cudaMemsetAsync(winner, 0xff, static_cast<size_t>(H) * W * sizeof(int), st));
    if (F > 0) {
        const dim3 grid(static_cast<unsigned>((F + RB_THREADS - 1) / RB_THREADS), RB_SPLIT);
        uv_raster_kernel<<<grid, RB_THREADS, 0, st>>>(vt, Nt, ft, F, H, W, reinterpret_cast<unsigned*>(winner));
        TPX_LAUNCH_CHECK();
    }
    uv_resolve_kernel<<<texel_blocks(H, W), RB_THREADS, 0, st>>>(vt, Nt, ft, H, W, winner, reinterpret_cast<float4*>(rast));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_rast_interpolate(const float* attr, int64_t Nv, int C, const int32_t* tri, int64_t F, const float* rast, int H, int W, float* out, void* stream) {
    TPX_CHECK(rast != nullptr && out != nullptr && (F == 0 || Nv == 0 || (attr != nullptr && tri != nullptr)), TPX_ERR_ARG, "rast_interpolate: null argument");
    TPX_CHECK(atlas_ok(H, W), TPX_ERR_SHAPE, "rast_interpolate: atlas %d x %d (1..8192 each)", H, W);
    TPX_CHECK(C >= 1 && C <= 4096 && F >= 0 && Nv >= 0, TPX_ERR_SHAPE, "rast_interpolate: bad sizes (C %d, F %lld, Nv %lld)", C, (long long)F, (long long)Nv);
    TPX_CHECK((reinterpret_cast<uintptr_t>(rast) & 15) == 0, TPX_ERR_ARG, "rast_interpolate: rast must be 16-B aligned");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    rast_interpolate_kernel<<<texel_blocks(H, W), RB_THREADS, 0, st>>>(attr, Nv, C, tri, F, reinterpret_cast<const float4*>(rast), static_cast<long long>(H) * W, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

size_t tpx_texture_inpaint_bytes(int H, int W) { return atlas_ok(H, W) ? ((static_cast<size_t>(H) * W * sizeof(short) + 255) & ~static_cast<size_t>(255)) : 0; }

int tpx_texture_inpaint(float* feats, const uint8_t* mask, int H, int W, int C, int pad, void* ws, size_t ws_bytes, int32_t* src, void* stream) {
    TPX_CHECK(feats != nullptr && mask != nullptr && ws != nullptr, TPX_ERR_ARG, "texture_inpaint: null argument");
    TPX_CHECK(atlas_ok(H, W), TPX_ERR_SHAPE, "texture_inpaint: atlas %d x %d (1..8192 each)", H, W);
    TPX_CHECK(C >= 1 && C <= 4096 && pad >= 0 && pad <= IP_MAX_PAD, TPX_ERR_SHAPE, "texture_inpaint: bad sizes (C %d, pad %d; pad 0..%d)", C, pad, IP_MAX_PAD);
    TPX_CHECK(ws_bytes >= tpx_texture_inpaint_bytes(H, W) && (reinterpret_cast<uintptr_t>(ws) & 1) == 0, TPX_ERR_ARG,
              "texture_inpaint: workspace too small or misaligned");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    short* rowd = static_cast<short*>(ws);
    inpaint_rows_kernel<<<texel_blocks(H, W), RB_THREADS, 0, st>>>(mask, H, W, pad, rowd);
    TPX_LAUNCH_CHECK();
    inpaint_cols_kernel<<<texel_blocks(H, W), RB_THREADS, 0, st>>>(mask, rowd, H, W, C, pad, feats, src);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // extern "C"
