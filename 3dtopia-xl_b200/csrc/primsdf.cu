// PrimSDF point query (SURVEY.md §8f-1, the consumer of the VAE output layout):
//   reference: models/primsdf.py:52-109 (forward, grid_sample_feat, prim_weight); called on 256^3 = 16.8 M points in
//   8192-point chunks by extract_texmesh (inference.py:108-116) through a dense [points x prims] weight matrix.
// Here: one thread per point, the primitives' (1/scale, pos) streamed through shared memory; a point visits every
// primitive once (box test in registers), samples only the few that cover it (trilinear, align_corners=True, from the
// L2-resident feature volumes) and never materialises the weight matrix.  FP32 SIMT: this is gather/compare work,
// not tensor-core work.
#include "bake_interp.cuh"
#include "kernels.cuh"

namespace tpx {

namespace {
constexpr int PS_THREADS = 256;
constexpr int PS_CHUNK = 1024;   // primitives staged per pass (16 KB of float4)

// ---- pieces shared by the exhaustive and the grid-binned kernels (identical arithmetic => identical results) ----------------------
// DF is the per-primitive channel stride of feat, NC <= DF the number of leading channels accumulated: the SDF-grid kernel
// accumulates channel 0 alone with exactly the channel-0 arithmetic of the full query.
template <int NC>
struct PointAcc {
    float acc[NC];
    float wsum;
};

// box weight w = 1 - |l|_inf of primitive v (scale, tx, ty, tz) at the point, and the local position l = (x - pos) / scale it was
// decided on.  The point and the backward decide coverage (w > 0) here and nowhere else.  The reference divides (primsdf.py:70, :106);
// the reciprocal multiply is at most one ulp of l from that.  Where |w| < 0.1 l is recomputed with the correctly rounded division:
// there w cancels to a few ulps of l, coverage is decided, and where a point's weights sum to about the 1e-6 of the normalisation
// (primsdf.py:108) one ulp of w moves the output by up to ~1e-4.  Above it one ulp of l (6e-8) is under 6e-7 of w.
__device__ __forceinline__ float prim_box(float px, float py, float pz, const float4 v, float& lx, float& ly, float& lz) {
    const float inv = 1.0f / v.x;
    const float dx = px - v.y, dy = py - v.z, dz = pz - v.w;
    lx = __fmul_rn(dx, inv); ly = __fmul_rn(dy, inv); lz = __fmul_rn(dz, inv);
    float w = 1.0f - fmaxf(fabsf(lx), fmaxf(fabsf(ly), fabsf(lz)));
    if (fabsf(w) < 0.1f) {
        lx = __fdiv_rn(dx, v.x); ly = __fdiv_rn(dy, v.x); lz = __fdiv_rn(dz, v.x);
        w = 1.0f - fmaxf(fabsf(lx), fmaxf(fabsf(ly), fabsf(lz)));
    }
    return w;
}

// trilinear cell of a covered local position in feat[k] viewed as [DF, D(z), H(y), W(x)], align_corners=True; |l| < 1 so no
// padding case.  off is the flat offset of the (x0, y0, z0) corner, a = the fractions along x, y, z.
struct TriCell {
    int off;
    float ax, ay, az;
};
__device__ __forceinline__ TriCell tri_cell(float lx, float ly, float lz, int S, float half_span) {
    const float fx = (lx + 1.0f) * half_span, fy = (ly + 1.0f) * half_span, fz = (lz + 1.0f) * half_span;
    const int x0 = min(static_cast<int>(fx), S - 2), y0 = min(static_cast<int>(fy), S - 2), z0 = min(static_cast<int>(fz), S - 2);
    return TriCell{(z0 * S + y0) * S + x0, fx - x0, fy - y0, fz - z0};
}

// Every product is rounded or fused as written (no compiler contraction), so the sdf channel comes out bit-identical whether one
// channel (the SDF grid) or all six (the point query) are accumulated: u (1 - t) + v t = fma(1 - t, u, t v).
__device__ __forceinline__ float tri_sample(const float* __restrict__ fc, const TriCell& t, int S) {
    const float bx = 1.f - t.ax, by = 1.f - t.ay, bz = 1.f - t.az;
    const float c00 = __fmaf_rn(bx, fc[0], __fmul_rn(t.ax, fc[1]));
    const float c01 = __fmaf_rn(bx, fc[S], __fmul_rn(t.ax, fc[S + 1]));
    const float c10 = __fmaf_rn(bx, fc[S * S], __fmul_rn(t.ax, fc[S * S + 1]));
    const float c11 = __fmaf_rn(bx, fc[S * S + S], __fmul_rn(t.ax, fc[S * S + S + 1]));
    return __fmaf_rn(bz, __fmaf_rn(by, c00, __fmul_rn(t.ay, c01)), __fmul_rn(t.az, __fmaf_rn(by, c10, __fmul_rn(t.ay, c11))));
}

// visit primitive k for the point (px,py,pz): box weight, and — if it covers the point — its trilinear sample
template <int NC, int DF>
__device__ __forceinline__ void visit_prim(PointAcc<NC>& a, float px, float py, float pz, const float4 v /* scale, tx, ty, tz */, int k,
                                           const float* __restrict__ feat, int S, int S3, float half_span) {
    float lx, ly, lz;
    const float w = prim_box(px, py, pz, v, lx, ly, lz);
    if (w > 0.f) {
        a.wsum += w;
        const TriCell t = tri_cell(lx, ly, lz, S, half_span);
        const float* f = feat + static_cast<size_t>(k) * DF * S3 + t.off;
#pragma unroll
        for (int c = 0; c < NC; ++c) a.acc[c] = fmaf(w, tri_sample(f + c * S3, t, S), a.acc[c]);
    }
}

// Nearest voxel of primitive v to an uncovered point (inference).  It is one of the 2x2x2 lattice neighbours of the (clamped) local
// position.  They are ranked the way the reference ranks all S^3 candidates (primsdf.py:93-96): fp32 L2 distance to pos + scale *
// linspace grid, first flat index wins a tie — a far point often has two candidates whose fp32 distances coincide.  e = x - voxel.
struct NearVoxel {
    int xi, yi, zi;
    float dist, ex, ey, ez;
};
__device__ __forceinline__ float lin_coord(int i, int S) {   // torch.linspace(-1, 1, S)[i]
    const float step = 2.0f / static_cast<float>(S - 1);
    return i < S / 2 ? -1.f + step * static_cast<float>(i) : 1.f - step * static_cast<float>(S - 1 - i);
}
__device__ __forceinline__ NearVoxel nearest_voxel(float px, float py, float pz, const float4 v, int S, float half_span) {
    const float sc = v.x;
    const float lx = (px - v.y) / sc, ly = (py - v.z) / sc, lz = (pz - v.w) / sc;
    const int x0 = min(max(static_cast<int>(floorf((lx + 1.f) * half_span)), 0), S - 2);
    const int y0 = min(max(static_cast<int>(floorf((ly + 1.f) * half_span)), 0), S - 2);
    const int z0 = min(max(static_cast<int>(floorf((lz + 1.f) * half_span)), 0), S - 2);
    NearVoxel r{x0, y0, z0, INFINITY, 0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const int cz = z0 + (c >> 2), cy = y0 + ((c >> 1) & 1), cx = x0 + (c & 1);
        const float ex = px - __fadd_rn(v.y, __fmul_rn(sc, lin_coord(cx, S)));
        const float ey = py - __fadd_rn(v.z, __fmul_rn(sc, lin_coord(cy, S)));
        const float ez = pz - __fadd_rn(v.w, __fmul_rn(sc, lin_coord(cz, S)));
        const float d = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez)));
        if (d < r.dist) r = NearVoxel{cx, cy, cz, d, ex, ey, ez};
    }
    return r;
}

template <int NC, int DF>
__device__ __forceinline__ void finish_point(const PointAcc<NC>& a, float px, float py, float pz, int best_k, const float* __restrict__ srt,
                                             const float* __restrict__ feat, int K, int S, int S3, float half_span, int inference, float* __restrict__ o) {
    if (a.wsum > 0.f) {
        const float inv = 1.0f / (a.wsum + 1e-6f);
        o[0] = a.acc[0] * inv;
#pragma unroll
        for (int c = 1; c < NC; ++c) o[c] = fminf(fmaxf(a.acc[c] * inv, 0.f), 1.f);
        return;
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) o[c] = 0.f;
    if (inference && K > 0) {
        // SDF of an uncovered point: nearest voxel of the nearest primitive, same sign, plus the L2 distance to it
        const float4 v = *reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(best_k));
        const NearVoxel nv = nearest_voxel(px, py, pz, v, S, half_span);
        const float sdf = feat[static_cast<size_t>(best_k) * DF * S3 + (nv.zi * S + nv.yi) * S + nv.xi];
        const float sgn = sdf > 0.f ? 1.f : (sdf < 0.f ? -1.f : 0.f);
        o[0] = sdf + nv.dist * sgn;
    }
}

// exhaustive version: every point visits every primitive (kept as the exactness reference of the binned kernel and as its fallback)
template <int DF>
__global__ void __launch_bounds__(PS_THREADS) primsdf_query_kernel(const float* __restrict__ x, const float* __restrict__ srt,
                                                                   const float* __restrict__ feat, long long n, int K, int S, int inference,
                                                                   float* __restrict__ out) {
    __shared__ float4 s_prim[PS_CHUNK];   // (scale, tx, ty, tz)
    const long long i = static_cast<long long>(blockIdx.x) * PS_THREADS + threadIdx.x;
    const bool live = i < n;
    float px = 0.f, py = 0.f, pz = 0.f;
    if (live) { px = x[3 * i]; py = x[3 * i + 1]; pz = x[3 * i + 2]; }
    PointAcc<DF> a;
#pragma unroll
    for (int c = 0; c < DF; ++c) a.acc[c] = 0.f;
    a.wsum = 0.f;
    float best_d2 = INFINITY;
    int best_k = 0;
    const int S3 = S * S * S;
    const float half_span = 0.5f * static_cast<float>(S - 1);
    for (int k0 = 0; k0 < K; k0 += PS_CHUNK) {
        const int kc = min(PS_CHUNK, K - k0);
        __syncthreads();
        for (int t = threadIdx.x; t < kc; t += PS_THREADS) s_prim[t] = *reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(k0 + t));
        __syncthreads();
        if (!live) continue;
        for (int t = 0; t < kc; ++t) {
            const float4 p = s_prim[t];
            const float dx = px - p.y, dy = py - p.z, dz = pz - p.w;
            const float d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < best_d2) { best_d2 = d2; best_k = k0 + t; }
            visit_prim<DF, DF>(a, px, py, pz, p, k0 + t, feat, S, S3, half_span);
        }
    }
    if (!live) return;
    finish_point<DF, DF>(a, px, py, pz, best_k, srt, feat, K, S, S3, half_span, inference, out + static_cast<size_t>(i) * DF);
}

// =====================================================================================================================
// Grid-binned query.  A G^3 grid over the bounding box of the primitives' boxes (united with [-1,1]^3) carries two
// ascending index lists per cell, built on the device from srt:
//   cover[c] : primitives whose box [pos - scale, pos + scale] meets the cell            (a superset of those covering a point of c)
//   near[c]  : primitives that can be the nearest centre for SOME point of the cell:      mindist(c, pos_k) <= min_j maxdist(c, pos_j)
// A point walks cover[cell] (same visit_prim, same ascending order => the same sums as the exhaustive kernel) and, only if nothing
// covers it, near[cell] for the nearest centre (same strict-< scan in ascending index => the same argmin).  Points outside
// the grid, or a grid whose lists overflowed the workspace, take the exhaustive loop.
// Layout of the workspace: GridHdr | counts[2 C] | offsets[2 C + 2] | entries[cap]      (C = G^3)
// =====================================================================================================================
constexpr int PG_G = 32;
constexpr int PG_CELLS = PG_G * PG_G * PG_G;
struct GridHdr {
    float ox, oy, oz, inv_h, h;
    int total_cover, total_near, overflow, cap, K;
};

__global__ void __launch_bounds__(256) grid_bounds_kernel(const float* __restrict__ srt, int K, GridHdr* __restrict__ hdr, int cap) {
    __shared__ float s_lo[3][256], s_hi[3][256];
    float lo[3] = {-1.f, -1.f, -1.f}, hi[3] = {1.f, 1.f, 1.f};
    for (int k = threadIdx.x; k < K; k += 256) {
        const float4 v = *reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(k));
        const float s = fabsf(v.x);
        const float c[3] = {v.y, v.z, v.w};
#pragma unroll
        for (int d = 0; d < 3; ++d) { lo[d] = fminf(lo[d], c[d] - s); hi[d] = fmaxf(hi[d], c[d] + s); }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) { s_lo[d][threadIdx.x] = lo[d]; s_hi[d][threadIdx.x] = hi[d]; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = 1; t < 256; ++t)
            for (int d = 0; d < 3; ++d) { lo[d] = fminf(lo[d], s_lo[d][t]); hi[d] = fmaxf(hi[d], s_hi[d][t]); }
        const float ext = fmaxf(hi[0] - lo[0], fmaxf(hi[1] - lo[1], hi[2] - lo[2])) * 1.0001f + 1e-6f;
        hdr->ox = lo[0]; hdr->oy = lo[1]; hdr->oz = lo[2];
        hdr->h = ext / PG_G;
        hdr->inv_h = PG_G / ext;
        hdr->total_cover = 0; hdr->total_near = 0; hdr->overflow = 0; hdr->cap = cap; hdr->K = K;
    }
}

// one warp per cell; FILL = 0: count both lists, FILL = 1: write them (ascending k, ordered warp compaction)
template <int FILL>
__global__ void __launch_bounds__(256) grid_lists_kernel(const float* __restrict__ srt, int K, const GridHdr* __restrict__ hdr, int* __restrict__ counts,
                                                         const int* __restrict__ offsets, int* __restrict__ entries) {
    extern __shared__ float4 s_srt[];      // all K primitives
    for (int k = threadIdx.x; k < K; k += blockDim.x) s_srt[k] = *reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(k));
    __syncthreads();
    const int cell = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (cell >= PG_CELLS) return;
    const int lane = threadIdx.x & 31;
    const float h = hdr->h;
    const int cz = cell / (PG_G * PG_G), cy = (cell / PG_G) % PG_G, cx = cell % PG_G;
    const float lo[3] = {hdr->ox + cx * h, hdr->oy + cy * h, hdr->oz + cz * h};
    const float hi[3] = {lo[0] + h, lo[1] + h, lo[2] + h};
    // pass A: upper bound of the nearest-centre distance over the cell = min_k maxdist(cell, pos_k)
    float ub2 = INFINITY;
    for (int k = lane; k < K; k += 32) {
        const float4 v = s_srt[k];
        const float c[3] = {v.y, v.z, v.w};
        float m2 = 0.f;
#pragma unroll
        for (int d = 0; d < 3; ++d) { const float m = fmaxf(fabsf(c[d] - lo[d]), fabsf(c[d] - hi[d])); m2 += m * m; }
        ub2 = fminf(ub2, m2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ub2 = fminf(ub2, __shfl_xor_sync(0xffffffffu, ub2, o));
    ub2 = ub2 * 1.0001f + 1e-9f;            // margin over fp32 rounding of the per-point distances
    int n_cover = 0, n_near = 0;
    const int off_c = FILL ? offsets[cell] : 0, off_n = FILL ? offsets[PG_CELLS + cell] : 0;
    const int cap = hdr->cap;
    for (int k0 = 0; k0 < K; k0 += 32) {
        const int k = k0 + lane;
        bool cover = false, near = false;
        if (k < K) {
            const float4 v = s_srt[k];
            const float s = fabsf(v.x) * 1.0001f + 1e-6f;
            const float c[3] = {v.y, v.z, v.w};
            cover = true;
            float d2 = 0.f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                cover = cover && (c[d] + s >= lo[d]) && (c[d] - s <= hi[d]);
                const float g = fmaxf(fmaxf(lo[d] - c[d], c[d] - hi[d]), 0.f);
                d2 += g * g;
            }
            near = d2 <= ub2;
        }
        const unsigned mc = __ballot_sync(0xffffffffu, cover), mn = __ballot_sync(0xffffffffu, near);
        if (FILL) {
            const unsigned below = (1u << lane) - 1u;
            if (cover) { const int pos = off_c + n_cover + __popc(mc & below); if (pos < cap) entries[pos] = k; }
            if (near) { const int pos = off_n + n_near + __popc(mn & below); if (pos < cap) entries[pos] = k; }
        }
        n_cover += __popc(mc);
        n_near += __popc(mn);
    }
    if (!FILL && lane == 0) { counts[cell] = n_cover; counts[PG_CELLS + cell] = n_near; }
}

// exclusive scan of the 2 C counts (single block), totals and the overflow flag
__global__ void __launch_bounds__(1024) grid_scan_kernel(const int* __restrict__ counts, int* __restrict__ offsets, GridHdr* __restrict__ hdr) {
    __shared__ int s_tot[1024];
    constexpr int N = 2 * PG_CELLS, PER = N / 1024;
    const int t = threadIdx.x;
    int local = 0;
    for (int i = 0; i < PER; ++i) local += counts[t * PER + i];
    s_tot[t] = local;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
        const int v = t >= o ? s_tot[t - o] : 0;
        __syncthreads();
        s_tot[t] += v;
        __syncthreads();
    }
    int run = s_tot[t] - local;
    for (int i = 0; i < PER; ++i) { offsets[t * PER + i] = run; run += counts[t * PER + i]; }
    if (t == 1023) {
        offsets[N] = run;
        hdr->total_cover = offsets[PG_CELLS];
        hdr->total_near = run - offsets[PG_CELLS];
        hdr->overflow = run > hdr->cap ? 1 : 0;
    }
}

// The walk of one point: every primitive (no grid, a point outside it or an over-full grid) or the cover list of the point's cell,
// in ascending k, calling visit(k, srt[k]) on each; then, only on a cell walk where covered() is false and `nearest` is set, the
// cell's near list.  Returns the nearest centre (strict <, ascending k: the first of equals) over the primitives scanned for it.
// The query and its backward both walk through here, so a (point, primitive) pair counts in both or in neither.
template <class Visit, class Covered>
__device__ __forceinline__ int walk_point(float px, float py, float pz, const float* __restrict__ srt, const GridHdr* __restrict__ hdr,
                                          const int* __restrict__ offsets, const int* __restrict__ entries, int K, bool nearest, Visit&& visit,
                                          Covered&& covered) {
    float best_d2 = INFINITY;
    int best_k = 0;
    bool inside = false;
    int cell = 0;
    if (hdr != nullptr) {
        const float gx = (px - hdr->ox) * hdr->inv_h, gy = (py - hdr->oy) * hdr->inv_h, gz = (pz - hdr->oz) * hdr->inv_h;
        inside = gx >= 0.f && gy >= 0.f && gz >= 0.f && gx < static_cast<float>(PG_G) && gy < static_cast<float>(PG_G) && gz < static_cast<float>(PG_G) &&
                 hdr->overflow == 0;
        if (inside) cell = (static_cast<int>(gz) * PG_G + static_cast<int>(gy)) * PG_G + static_cast<int>(gx);
    }
    if (!inside) {          // exhaustive loop (rare: points outside the primitives' bounding box / oversized lists / no grid)
        for (int k = 0; k < K; ++k) {
            const float4 p = __ldg(reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(k)));
            const float dx = px - p.y, dy = py - p.z, dz = pz - p.w;
            const float d2 = dx * dx + dy * dy + dz * dz;
            if (d2 < best_d2) { best_d2 = d2; best_k = k; }
            visit(k, p);
        }
    } else {
        const int c0 = offsets[cell], c1 = offsets[cell + 1];
        for (int e = c0; e < c1; ++e) {
            const int k = entries[e];
            const float4 p = __ldg(reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(k)));
            visit(k, p);
        }
        if (!covered() && nearest) {
            const int n0 = offsets[PG_CELLS + cell], n1 = offsets[PG_CELLS + cell + 1];
            for (int e = n0; e < n1; ++e) {
                const int k = entries[e];
                const float4 p = __ldg(reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(k)));
                const float dx = px - p.y, dy = py - p.z, dz = pz - p.w;
                const float d2 = dx * dx + dy * dy + dz * dz;
                if (d2 < best_d2) { best_d2 = d2; best_k = k; }
            }
        }
    }
    return best_k;
}

// one point of the binned query; hdr == nullptr (no grid) takes the exhaustive loop
template <int NC, int DF>
__device__ __forceinline__ void query_point_binned(float px, float py, float pz, const float* __restrict__ srt, const float* __restrict__ feat,
                                                   const GridHdr* __restrict__ hdr, const int* __restrict__ offsets, const int* __restrict__ entries, int K,
                                                   int S, int inference, float* __restrict__ o) {
    PointAcc<NC> a;
#pragma unroll
    for (int c = 0; c < NC; ++c) a.acc[c] = 0.f;
    a.wsum = 0.f;
    const int S3 = S * S * S;
    const float half_span = 0.5f * static_cast<float>(S - 1);
    const int best_k = walk_point(
        px, py, pz, srt, hdr, offsets, entries, K, inference != 0,
        [&](int k, const float4 p) { visit_prim<NC, DF>(a, px, py, pz, p, k, feat, S, S3, half_span); }, [&] { return a.wsum > 0.f; });
    finish_point<NC, DF>(a, px, py, pz, best_k, srt, feat, K, S, S3, half_span, inference, o);
}

template <int DF>
__global__ void __launch_bounds__(PS_THREADS) primsdf_query_grid_kernel(const float* __restrict__ x, const float* __restrict__ srt,
                                                                        const float* __restrict__ feat, const GridHdr* __restrict__ hdr,
                                                                        const int* __restrict__ offsets, const int* __restrict__ entries, long long n, int K,
                                                                        int S, int inference, float* __restrict__ out) {
    const long long i = static_cast<long long>(blockIdx.x) * PS_THREADS + threadIdx.x;
    if (i >= n) return;
    query_point_binned<DF, DF>(x[3 * i], x[3 * i + 1], x[3 * i + 2], srt, feat, hdr, offsets, entries, K, S, inference, out + static_cast<size_t>(i) * DF);
}

// =====================================================================================================================
// Backward of the point query (models/primsdf.py:52-109 under autograd; the loss of dva/losses.py:102-148 fits through it).
// One thread per point, walking exactly the primitives the forward walked (walk_point, prim_box, nearest_voxel):
//   pass 1: the forward's wsum, raw normalised output o_c and nearest-primitive choice, with its arithmetic;
//   the upstream gradient g of channels 1..5 is zeroed where o_c lies outside [0, 1] (torch.clip passes the bounds);
//   pass 2: the covering primitives again, emitting with W = wsum + 1e-6:
//     dL/dv_jc = g_c w_j / W, scattered to the 8 trilinear corners of channel c of feat[j];
//     dL/dw_j = sum_c g_c (v_jc - o_c) / W;
//     dL/dl_j = sum_c (g_c w_j / W) dv_jc/dl - dL/dw_j sign(l_jd) [|l_jd| = max] / (tied axes);
//     dL/dx += dL/dl_j / s_j, dL/dpos_j -= dL/dl_j / s_j, dL/ds_j -= (dL/dl_j . l_j) / s_j.
//   An uncovered point at inference (sdf = f + d sign(f), d = |x - c|, c the nearest voxel, u = (x - c) / d, 0 at d = 0):
//     dL/dfeat_geo[k,v] += g_0, dL/dx += g_0 sign(f) u, dL/dpos_k -= g_0 sign(f) u, dL/ds_k -= g_0 sign(f) (u . grid_v).
// grad_x is owned by the point's thread; grad_srt / grad_feat are fp32 reductions (RED.E.ADD.F32), so their last bits depend on
// the order in which points arrive.  Any of the three may be null.  Two blocks per SM cap the registers at 128 without spills.
// =====================================================================================================================
template <int DF>
__global__ void __launch_bounds__(PS_THREADS, 2) primsdf_backward_kernel(const float* __restrict__ x, const float* __restrict__ srt, const float* __restrict__ feat,
                                                                      const GridHdr* __restrict__ hdr, const int* __restrict__ offsets,
                                                                      const int* __restrict__ entries, long long n, int K, int S, int inference,
                                                                      const float* __restrict__ grad_out, float* __restrict__ grad_x,
                                                                      float* __restrict__ grad_srt, float* __restrict__ grad_feat) {
    const long long i = static_cast<long long>(blockIdx.x) * PS_THREADS + threadIdx.x;
    if (i >= n) return;
    const float px = x[3 * i], py = x[3 * i + 1], pz = x[3 * i + 2];
    const int S3 = S * S * S;
    const float half_span = 0.5f * static_cast<float>(S - 1);
    PointAcc<DF> a;
#pragma unroll
    for (int c = 0; c < DF; ++c) a.acc[c] = 0.f;
    a.wsum = 0.f;
    const int best_k = walk_point(
        px, py, pz, srt, hdr, offsets, entries, K, inference != 0,
        [&](int k, const float4 p) { visit_prim<DF, DF>(a, px, py, pz, p, k, feat, S, S3, half_span); }, [&] { return a.wsum > 0.f; });
    float g[DF];
#pragma unroll
    for (int c = 0; c < DF; ++c) g[c] = grad_out[static_cast<size_t>(i) * DF + c];
    float gpx = 0.f, gpy = 0.f, gpz = 0.f;
    if (a.wsum > 0.f) {
        const float inv = 1.0f / (a.wsum + 1e-6f);
        float o[DF];
#pragma unroll
        for (int c = 0; c < DF; ++c) {
            o[c] = a.acc[c] * inv;
            if (c > 0 && !(o[c] >= 0.f && o[c] <= 1.f)) g[c] = 0.f;
        }
        walk_point(
            px, py, pz, srt, hdr, offsets, entries, K, false,
            [&](int k, const float4 p) {
                float lx, ly, lz;
                const float w = prim_box(px, py, pz, p, lx, ly, lz);
                if (!(w > 0.f)) return;
                const TriCell t = tri_cell(lx, ly, lz, S, half_span);
                const float bx = 1.f - t.ax, by = 1.f - t.ay, bz = 1.f - t.az;
                const size_t base = static_cast<size_t>(k) * DF * S3 + t.off;
                const float wn = w * inv;
                float gw = 0.f, dax = 0.f, day = 0.f, daz = 0.f;   // dL/dw_j * W and dL/d(ax, ay, az)
#pragma unroll
                for (int c = 0; c < DF; ++c) {
                    const float* fc = feat + base + static_cast<size_t>(c) * S3;
                    const float f000 = fc[0], f001 = fc[1], f010 = fc[S], f011 = fc[S + 1];
                    const float f100 = fc[S * S], f101 = fc[S * S + 1], f110 = fc[S * S + S], f111 = fc[S * S + S + 1];
                    const float c00 = bx * f000 + t.ax * f001, c01 = bx * f010 + t.ax * f011;
                    const float c10 = bx * f100 + t.ax * f101, c11 = bx * f110 + t.ax * f111;
                    const float e0 = by * c00 + t.ay * c01, e1 = by * c10 + t.ay * c11;
                    gw += g[c] * ((bz * e0 + t.az * e1) - o[c]);
                    const float gv = g[c] * wn;
                    if (gv == 0.f) continue;
                    dax += gv * (bz * (by * (f001 - f000) + t.ay * (f011 - f010)) + t.az * (by * (f101 - f100) + t.ay * (f111 - f110)));
                    day += gv * (bz * (c01 - c00) + t.az * (c11 - c10));
                    daz += gv * (e1 - e0);
                    if (grad_feat != nullptr) {
                        float* gf = grad_feat + base + static_cast<size_t>(c) * S3;
                        atomicAdd(gf, gv * bz * by * bx);                 atomicAdd(gf + 1, gv * bz * by * t.ax);
                        atomicAdd(gf + S, gv * bz * t.ay * bx);           atomicAdd(gf + S + 1, gv * bz * t.ay * t.ax);
                        atomicAdd(gf + S * S, gv * t.az * by * bx);       atomicAdd(gf + S * S + 1, gv * t.az * by * t.ax);
                        atomicAdd(gf + S * S + S, gv * t.az * t.ay * bx); atomicAdd(gf + S * S + S + 1, gv * t.az * t.ay * t.ax);
                    }
                }
                // the inf-norm's derivative splits a tie evenly between the tied axes; at the centre (l = 0) it is 0
                const float m = fmaxf(fabsf(lx), fmaxf(fabsf(ly), fabsf(lz)));
                const bool tx = fabsf(lx) == m, ty = fabsf(ly) == m, tz = fabsf(lz) == m;
                const float q = gw * inv / static_cast<float>(static_cast<int>(tx) + static_cast<int>(ty) + static_cast<int>(tz));
                const float is = 1.0f / p.x;
                const float glx = (dax * half_span - (tx && lx != 0.f ? (lx > 0.f ? q : -q) : 0.f)) * is;
                const float gly = (day * half_span - (ty && ly != 0.f ? (ly > 0.f ? q : -q) : 0.f)) * is;
                const float glz = (daz * half_span - (tz && lz != 0.f ? (lz > 0.f ? q : -q) : 0.f)) * is;
                gpx += glx; gpy += gly; gpz += glz;
                if (grad_srt != nullptr) {
                    float* gs = grad_srt + 4 * static_cast<size_t>(k);
                    atomicAdd(gs, -(glx * lx + gly * ly + glz * lz));
                    atomicAdd(gs + 1, -glx); atomicAdd(gs + 2, -gly); atomicAdd(gs + 3, -glz);
                }
            },
            [] { return true; });
    } else if (inference && K > 0) {
        const float4 v = *reinterpret_cast<const float4*>(srt + 4 * static_cast<size_t>(best_k));
        const NearVoxel nv = nearest_voxel(px, py, pz, v, S, half_span);
        const size_t vi = static_cast<size_t>(best_k) * DF * S3 + (nv.zi * S + nv.yi) * S + nv.xi;
        const float f = feat[vi];
        if (grad_feat != nullptr && g[0] != 0.f) atomicAdd(grad_feat + vi, g[0]);
        const float h = (f > 0.f ? g[0] : (f < 0.f ? -g[0] : 0.f)) / nv.dist;       // g_0 sign(f) / d
        if (nv.dist > 0.f && h != 0.f) {
            const float ux = h * nv.ex, uy = h * nv.ey, uz = h * nv.ez;
            gpx = ux; gpy = uy; gpz = uz;
            if (grad_srt != nullptr) {
                float* gs = grad_srt + 4 * static_cast<size_t>(best_k);
                atomicAdd(gs, -(ux * lin_coord(nv.xi, S) + uy * lin_coord(nv.yi, S) + uz * lin_coord(nv.zi, S)));
                atomicAdd(gs + 1, -ux); atomicAdd(gs + 2, -uy); atomicAdd(gs + 3, -uz);
            }
        }
    }
    if (grad_x != nullptr) { grad_x[3 * i] += gpx; grad_x[3 * i + 1] += gpy; grad_x[3 * i + 2] += gpz; }
}

// sdf channel of the query on the R^3 lattice (coords[i], coords[j], coords[k]); grid[(i R + j) R + k] (inference.py:108-116:
// meshgrid(indexing='ij'), reshape(R,R,R)); the points are never materialised
__global__ void __launch_bounds__(PS_THREADS) primsdf_sdf_grid_kernel(const float* __restrict__ coords, int R, const float* __restrict__ srt,
                                                                      const float* __restrict__ feat, const GridHdr* __restrict__ hdr,
                                                                      const int* __restrict__ offsets, const int* __restrict__ entries, int K, int S,
                                                                      int inference, float* __restrict__ grid) {
    const long long idx = static_cast<long long>(blockIdx.x) * PS_THREADS + threadIdx.x;
    const long long n = static_cast<long long>(R) * R * R;
    if (idx >= n) return;
    const int k = static_cast<int>(idx % R), j = static_cast<int>((idx / R) % R), i = static_cast<int>(idx / (static_cast<long long>(R) * R));
    query_point_binned<1, 6>(coords[i], coords[j], coords[k], srt, feat, hdr, offsets, entries, K, S, inference, grid + idx);
}
// fused texel query of the texture bake (inference.py:173-198: dr.interpolate of the positions, the masked PrimSDF.forward in 8192-point
// chunks, the scatter through the mask, * 255): one thread per atlas texel reads its rast entry, interpolates the 3-D position with the
// device function tpx_rast_interpolate uses, runs the 6-channel binned query forward runs (inference = 0: the nearest-primitive
// fallback only defines the discarded sdf of uncovered points) and writes feats = 255 (R, G, B, 0, roughness, metallic) and the mask.
__global__ void __launch_bounds__(PS_THREADS) primsdf_bake_kernel(const float4* __restrict__ rast, long long n, const float* __restrict__ v, long long Nv,
                                                                  const int* __restrict__ f, long long F, const float* __restrict__ srt,
                                                                  const float* __restrict__ feat, const GridHdr* __restrict__ hdr,
                                                                  const int* __restrict__ offsets, const int* __restrict__ entries, int K, int S,
                                                                  float* __restrict__ feats, uint8_t* __restrict__ mask) {
    const long long p = static_cast<long long>(blockIdx.x) * PS_THREADS + threadIdx.x;
    if (p >= n) return;
    const float4 r = rast[p];
    const int t = rast_triangle(r.w);
    float o[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    uint8_t covered = 0;
    if (t >= 0 && t < F) {
        const long long i0 = f[3 * static_cast<long long>(t)], i1 = f[3 * static_cast<long long>(t) + 1], i2 = f[3 * static_cast<long long>(t) + 2];
        if (i0 >= 0 && i1 >= 0 && i2 >= 0 && i0 < Nv && i1 < Nv && i2 < Nv) {
            const float *a0 = v + 3 * i0, *a1 = v + 3 * i1, *a2 = v + 3 * i2;
            query_point_binned<6, 6>(bary_interp(r.x, r.y, a0[0], a1[0], a2[0]), bary_interp(r.x, r.y, a0[1], a1[1], a2[1]),
                                     bary_interp(r.x, r.y, a0[2], a1[2], a2[2]), srt, feat, hdr, offsets, entries, K, S, 0, o);
            covered = 1;
        }
    }
    float* out = feats + p * 6;
    out[0] = __fmul_rn(o[1], 255.f); out[1] = __fmul_rn(o[2], 255.f); out[2] = __fmul_rn(o[3], 255.f);
    out[3] = 0.f;
    out[4] = __fmul_rn(o[4], 255.f); out[5] = __fmul_rn(o[5], 255.f);
    mask[p] = covered;
}

struct GridPtrs { GridHdr* hdr; int* counts; int* offsets; int* entries; long long cap; };
GridPtrs grid_carve(const void* ws, size_t bytes) {
    if (ws == nullptr) return GridPtrs{nullptr, nullptr, nullptr, nullptr, 0};
    uint8_t* b = static_cast<uint8_t*>(const_cast<void*>(ws));
    GridPtrs g;
    g.hdr = reinterpret_cast<GridHdr*>(b);
    g.counts = reinterpret_cast<int*>(b + 256);
    g.offsets = g.counts + 2 * PG_CELLS;
    g.entries = g.offsets + 2 * PG_CELLS + 2;
    const size_t fixed = 256 + static_cast<size_t>(4 * PG_CELLS + 2) * 4;
    g.cap = bytes > fixed ? static_cast<long long>((bytes - fixed) / 4) : 0;
    return g;
}
}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" {

int tpx_primsdf_query(const float* x, const float* srt, const float* feat, int64_t n, int K, int S, int dim_feat, int inference, float* out, void* stream) {
    if (n == 0) return TPX_OK;
    TPX_CHECK(n > 0 && x != nullptr && srt != nullptr && feat != nullptr && out != nullptr, TPX_ERR_ARG, "primsdf_query: null argument or negative n");
    TPX_CHECK(dim_feat == 6, TPX_ERR_SHAPE, "primsdf_query: dim_feat %d (kernel covers the released 6-channel layout)", dim_feat);
    TPX_CHECK(S >= 2 && S <= 32 && K >= 0, TPX_ERR_SHAPE, "primsdf_query: bad primitive geometry (S %d, K %d)", S, K);
    TPX_CHECK((reinterpret_cast<uintptr_t>(srt) & 15) == 0, TPX_ERR_ARG, "primsdf_query: srt must be 16-B aligned");
    const long long blocks = (n + PS_THREADS - 1) / PS_THREADS;
    TPX_CHECK(blocks < (1LL << 31), TPX_ERR_SHAPE, "primsdf_query: too many points");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    primsdf_query_kernel<6><<<static_cast<unsigned>(blocks), PS_THREADS, 0, st>>>(x, srt, feat, n, K, S, inference, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

size_t tpx_primsdf_grid_bytes(int64_t cap_entries) {
    if (cap_entries <= 0) return 0;
    return sizeof(GridHdr) + 256 + static_cast<size_t>(2 * PG_CELLS) * 4 + static_cast<size_t>(2 * PG_CELLS + 2) * 4 + static_cast<size_t>(cap_entries) * 4;
}

int tpx_primsdf_grid_build(const float* srt, int K, void* grid_ws, size_t grid_bytes, void* stream) {
    TPX_CHECK(srt != nullptr && grid_ws != nullptr, TPX_ERR_ARG, "primsdf_grid_build: null argument");
    TPX_CHECK(K > 0 && K <= 4096, TPX_ERR_SHAPE, "primsdf_grid_build: K %d (1..4096 primitives fit the builder's shared memory)", K);
    TPX_CHECK((reinterpret_cast<uintptr_t>(srt) & 15) == 0 && (reinterpret_cast<uintptr_t>(grid_ws) & 255) == 0, TPX_ERR_ARG, "primsdf_grid_build: alignment");
    const GridPtrs g = grid_carve(grid_ws, grid_bytes);
    TPX_CHECK(g.cap >= 1024, TPX_ERR_ARG, "primsdf_grid_build: workspace too small");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    const int cap = g.cap > 0x7fffffffLL ? 0x7fffffff : static_cast<int>(g.cap);
    grid_bounds_kernel<<<1, 256, 0, st>>>(srt, K, g.hdr, cap);
    TPX_LAUNCH_CHECK();
    const size_t smem = static_cast<size_t>(K) * 16;
    static bool attr_set = false;
    if (!attr_set) {
        TPX_CUDA(cudaFuncSetAttribute(grid_lists_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 16));
        TPX_CUDA(cudaFuncSetAttribute(grid_lists_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 16));
        attr_set = true;
    }
    grid_lists_kernel<0><<<PG_CELLS / 8, 256, smem, st>>>(srt, K, g.hdr, g.counts, g.offsets, g.entries);
    TPX_LAUNCH_CHECK();
    grid_scan_kernel<<<1, 1024, 0, st>>>(g.counts, g.offsets, g.hdr);
    TPX_LAUNCH_CHECK();
    grid_lists_kernel<1><<<PG_CELLS / 8, 256, smem, st>>>(srt, K, g.hdr, g.counts, g.offsets, g.entries);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_primsdf_query_grid(const float* x, const float* srt, const float* feat, const void* grid_ws, size_t grid_bytes, int64_t n, int K, int S, int dim_feat,
                           int inference, float* out, void* stream) {
    if (n == 0) return TPX_OK;
    TPX_CHECK(n > 0 && x != nullptr && srt != nullptr && feat != nullptr && out != nullptr && grid_ws != nullptr, TPX_ERR_ARG,
              "primsdf_query_grid: null argument or negative n");
    TPX_CHECK(dim_feat == 6, TPX_ERR_SHAPE, "primsdf_query: dim_feat %d (kernel covers the released 6-channel layout)", dim_feat);
    TPX_CHECK(S >= 2 && S <= 32 && K > 0, TPX_ERR_SHAPE, "primsdf_query: bad primitive geometry (S %d, K %d)", S, K);
    const long long blocks = (n + PS_THREADS - 1) / PS_THREADS;
    TPX_CHECK(blocks < (1LL << 31), TPX_ERR_SHAPE, "primsdf_query: too many points");
    TPX_DEVICE_GUARD();
    const GridPtrs g = grid_carve(grid_ws, grid_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    primsdf_query_grid_kernel<6><<<static_cast<unsigned>(blocks), PS_THREADS, 0, st>>>(x, srt, feat, g.hdr, g.offsets, g.entries, n, K, S, inference, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_primsdf_query_backward(const float* x, const float* srt, const float* feat, const void* grid_ws, size_t grid_bytes, int64_t n, int K, int S,
                               int dim_feat, int inference, const float* grad_out, float* grad_x, float* grad_srt, float* grad_feat, void* stream) {
    if (n == 0) return TPX_OK;
    TPX_CHECK(n > 0 && x != nullptr && srt != nullptr && feat != nullptr && grad_out != nullptr, TPX_ERR_ARG,
              "primsdf_query_backward: null argument or negative n");
    TPX_CHECK(dim_feat == 6, TPX_ERR_SHAPE, "primsdf_query_backward: dim_feat %d (kernel covers the released 6-channel layout)", dim_feat);
    TPX_CHECK(S >= 2 && S <= 32 && K >= 0 && (K > 0 || grid_ws == nullptr), TPX_ERR_SHAPE, "primsdf_query_backward: bad primitive geometry (S %d, K %d)", S, K);
    TPX_CHECK((reinterpret_cast<uintptr_t>(srt) & 15) == 0, TPX_ERR_ARG, "primsdf_query_backward: srt must be 16-B aligned");
    const long long blocks = (n + PS_THREADS - 1) / PS_THREADS;
    TPX_CHECK(blocks < (1LL << 31), TPX_ERR_SHAPE, "primsdf_query_backward: too many points");
    TPX_DEVICE_GUARD();
    if (grad_x == nullptr && grad_srt == nullptr && grad_feat == nullptr) return TPX_OK;
    const GridPtrs g = grid_carve(grid_ws, grid_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    primsdf_backward_kernel<6><<<static_cast<unsigned>(blocks), PS_THREADS, 0, st>>>(x, srt, feat, g.hdr, g.offsets, g.entries, n, K, S, inference, grad_out,
                                                                                     grad_x, grad_srt, grad_feat);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_primsdf_sdf_grid(const float* coords, int R, const float* srt, const float* feat, const void* grid_ws, size_t grid_bytes, int K, int S, int dim_feat,
                         int inference, float* grid_out, void* stream) {
    TPX_CHECK(coords != nullptr && srt != nullptr && feat != nullptr && grid_out != nullptr, TPX_ERR_ARG, "primsdf_sdf_grid: null argument");
    TPX_CHECK(dim_feat == 6, TPX_ERR_SHAPE, "primsdf_sdf_grid: dim_feat %d (kernel covers the released 6-channel layout)", dim_feat);
    TPX_CHECK(S >= 2 && S <= 32 && K >= 0 && (K > 0 || grid_ws == nullptr), TPX_ERR_SHAPE, "primsdf_sdf_grid: bad primitive geometry (S %d, K %d)", S, K);
    TPX_CHECK(R >= 1 && R <= 2048, TPX_ERR_SHAPE, "primsdf_sdf_grid: resolution %d (1..2048)", R);
    TPX_CHECK((reinterpret_cast<uintptr_t>(srt) & 15) == 0, TPX_ERR_ARG, "primsdf_sdf_grid: srt must be 16-B aligned");
    TPX_DEVICE_GUARD();
    const GridPtrs g = grid_carve(grid_ws, grid_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    const long long blocks = (static_cast<long long>(R) * R * R + PS_THREADS - 1) / PS_THREADS;
    primsdf_sdf_grid_kernel<<<static_cast<unsigned>(blocks), PS_THREADS, 0, st>>>(coords, R, srt, feat, g.hdr, g.offsets, g.entries, K, S, inference, grid_out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_primsdf_bake(const float* rast, int H, int W, const float* v, int64_t Nv, const int32_t* f, int64_t F, const float* srt, const float* feat,
                     const void* grid_ws, size_t grid_bytes, int K, int S, int dim_feat, float* feats, uint8_t* mask, void* stream) {
    TPX_CHECK(rast != nullptr && feats != nullptr && mask != nullptr && srt != nullptr && feat != nullptr && (F == 0 || Nv == 0 || (v != nullptr && f != nullptr)),
              TPX_ERR_ARG, "primsdf_bake: null argument");
    TPX_CHECK(dim_feat == 6, TPX_ERR_SHAPE, "primsdf_bake: dim_feat %d (kernel covers the released 6-channel layout)", dim_feat);
    TPX_CHECK(S >= 2 && S <= 32 && K >= 0 && (K > 0 || grid_ws == nullptr), TPX_ERR_SHAPE, "primsdf_bake: bad primitive geometry (S %d, K %d)", S, K);
    TPX_CHECK(H >= 1 && W >= 1 && H <= 8192 && W <= 8192 && F >= 0 && Nv >= 0, TPX_ERR_SHAPE, "primsdf_bake: atlas %d x %d (1..8192 each), F %lld, Nv %lld", H, W,
              (long long)F, (long long)Nv);
    TPX_CHECK((reinterpret_cast<uintptr_t>(srt) & 15) == 0 && (reinterpret_cast<uintptr_t>(rast) & 15) == 0, TPX_ERR_ARG, "primsdf_bake: srt and rast must be 16-B aligned");
    TPX_DEVICE_GUARD();
    const GridPtrs g = grid_carve(grid_ws, grid_bytes);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    const long long n = static_cast<long long>(H) * W;
    primsdf_bake_kernel<<<static_cast<unsigned>((n + PS_THREADS - 1) / PS_THREADS), PS_THREADS, 0, st>>>(reinterpret_cast<const float4*>(rast), n, v, Nv, f, F, srt, feat, g.hdr,
                                                                                                       g.offsets, g.entries, K, S, feats, mask);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // extern "C"
