// Marching cubes over a dense fp32 volume (DESIGN.md §1 f-5): the GPU stand-in for `mcubes.marching_cubes(grid, 0.0)` in
// extract_texmesh (inference.py:106-124), which the reference runs on the CPU after copying the 256^3 SDF grid to the host.
// The output is deterministic: every vertex and triangle position comes from prefix sums, never from atomics.
//   count : (a) one thread per lattice point: crossing-edge mask of the 3 edges it owns and, if it is a cell's lowest corner,
//           the cell's case byte (both kept in the workspace); per-block vertex / triangle totals;
//           (b) one block scans the block totals into int64 offsets and writes V, F.
//   emit  : (c) one thread per point: block scan of its vertex count, the point's first vertex id, its vertex positions;
//           (d) one thread per point: block scan of its cell's triangle count, the triangles (vertex ids of the owners).
// Workspace: McHdr (256 B) | code[N] u16 (mask | case << 8) | vbase[N] i32 | blk_v[nb] i32 | blk_f[nb] i32 | off_v[nb] i64 | off_f[nb] i64
#include "kernels.cuh"
#include "mc_tables.cuh"

namespace tpx {

namespace {
constexpr int MC_THREADS = 256;
constexpr int MC_SCAN_THREADS = 1024;
constexpr long long MC_INDEX_LIMIT = 1LL << 31;

struct McHdr {
    long long V, F;
};

struct McPtrs {
    McHdr* hdr;
    uint16_t* code;
    int* vbase;
    int* blk_v;
    int* blk_f;
    long long* off_v;
    long long* off_f;
    size_t total;
};

McPtrs mc_carve(void* ws, long long N, long long nb) {
    Carve c{static_cast<uint8_t*>(ws)};
    McPtrs p;
    p.hdr = c.take<McHdr>(1);
    p.code = c.take<uint16_t>(N);
    p.vbase = c.take<int>(N);
    p.blk_v = c.take<int>(nb);
    p.blk_f = c.take<int>(nb);
    p.off_v = c.take<long long>(nb);
    p.off_f = c.take<long long>(nb);
    p.total = c.off;
    return p;
}

// exclusive block-wide prefix sum of v (MC_THREADS threads); *total receives the block's sum
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < MC_THREADS / 32 ? s_warp[lane] : 0;
#pragma unroll
        for (int o = 1; o < MC_THREADS / 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < MC_THREADS / 32) s_warp[lane] = w;      // inclusive warp totals
    }
    __syncthreads();
    *total = s_warp[MC_THREADS / 32 - 1];
    return x - v + (warp > 0 ? s_warp[warp - 1] : 0);
}

__device__ __forceinline__ int block_sum(int v, int* s_warp) {
    int total;
    block_exclusive_scan(v, s_warp, &total);
    return total;
}

// (a) classification and counts
__global__ void __launch_bounds__(MC_THREADS) mc_count_kernel(const float* __restrict__ vol, int X, int Y, int Z, float iso, uint16_t* __restrict__ code,
                                                              int* __restrict__ blk_v, int* __restrict__ blk_f) {
    __shared__ int8_t s_cnt[256];
    __shared__ int s_warp[MC_THREADS / 32];
    s_cnt[threadIdx.x] = kMcTriCount[threadIdx.x];
    __syncthreads();
    const int N = X * Y * Z, YZ = Y * Z;
    const int p = blockIdx.x * MC_THREADS + threadIdx.x;
    int nv = 0, nt = 0;
    if (p < N) {
        const int i = p / YZ, r = p - i * YZ, j = r / Z, k = r - j * Z;
        const bool bx = i + 1 < X, by = j + 1 < Y, bz = k + 1 < Z;
        const bool in0 = __ldg(vol + p) < iso;
        unsigned m = 0;
        if (bx && ((__ldg(vol + p + YZ) < iso) != in0)) m |= 1u;
        if (by && ((__ldg(vol + p + Z) < iso) != in0)) m |= 2u;
        if (bz && ((__ldg(vol + p + 1) < iso) != in0)) m |= 4u;
        unsigned c = 0;
        if (bx && by && bz) {
#pragma unroll
            for (int n = 0; n < 8; ++n) {
                const int off = (n & 1) * YZ + ((n >> 1) & 1) * Z + (n >> 2);
                c |= static_cast<unsigned>(__ldg(vol + p + off) < iso) << n;
            }
            nt = s_cnt[c];
        }
        code[p] = static_cast<uint16_t>(m | (c << 8));
        nv = __popc(m);
    }
    const int tv = block_sum(nv, s_warp);
    __syncthreads();
    const int tf = block_sum(nt, s_warp);
    if (threadIdx.x == 0) { blk_v[blockIdx.x] = tv; blk_f[blockIdx.x] = tf; }
}

// (b) exclusive scan of the per-block totals (one block; nb < 2^23) into int64 offsets; totals to the header and to counts
__global__ void __launch_bounds__(MC_SCAN_THREADS) mc_scan_kernel(const int* __restrict__ blk_v, const int* __restrict__ blk_f, int nb,
                                                                  long long* __restrict__ off_v, long long* __restrict__ off_f, McHdr* __restrict__ hdr,
                                                                  long long* __restrict__ counts) {
    __shared__ long long s_v[MC_SCAN_THREADS], s_f[MC_SCAN_THREADS];
    const int t = threadIdx.x;
    const int per = (nb + MC_SCAN_THREADS - 1) / MC_SCAN_THREADS;
    const int b0 = min(t * per, nb), b1 = min(b0 + per, nb);
    long long lv = 0, lf = 0;
    for (int b = b0; b < b1; ++b) { lv += blk_v[b]; lf += blk_f[b]; }
    s_v[t] = lv;
    s_f[t] = lf;
    __syncthreads();
    for (int o = 1; o < MC_SCAN_THREADS; o <<= 1) {
        const long long av = t >= o ? s_v[t - o] : 0, af = t >= o ? s_f[t - o] : 0;
        __syncthreads();
        s_v[t] += av;
        s_f[t] += af;
        __syncthreads();
    }
    long long rv = s_v[t] - lv, rf = s_f[t] - lf;
    for (int b = b0; b < b1; ++b) {
        off_v[b] = rv;
        off_f[b] = rf;
        rv += blk_v[b];
        rf += blk_f[b];
    }
    if (t == MC_SCAN_THREADS - 1) {
        hdr->V = s_v[t];
        hdr->F = s_f[t];
        counts[0] = s_v[t];
        counts[1] = s_f[t];
    }
}

// (c) vertices: id order = (point, axis); position origin + spacing * (p + t e_a), t = (iso - f(p)) / (f(p + e_a) - f(p)) in fp32
__global__ void __launch_bounds__(MC_THREADS) mc_vertex_kernel(const float* __restrict__ vol, int X, int Y, int Z, float iso, float3 origin, float3 spacing,
                                                               const uint16_t* __restrict__ code, const long long* __restrict__ off_v,
                                                               const McHdr* __restrict__ hdr, int* __restrict__ vbase, float* __restrict__ verts) {
    __shared__ int s_warp[MC_THREADS / 32];
    if (hdr->V >= MC_INDEX_LIMIT || hdr->F >= MC_INDEX_LIMIT) return;    // the caller sees the counts and reports the overflow
    const int N = X * Y * Z, YZ = Y * Z;
    const int p = blockIdx.x * MC_THREADS + threadIdx.x;
    const unsigned m = p < N ? (code[p] & 7u) : 0u;
    int total;
    const int excl = block_exclusive_scan(__popc(m), s_warp, &total);
    if (m == 0) return;
    int id = static_cast<int>(off_v[blockIdx.x] + excl);
    vbase[p] = id;
    const int i = p / YZ, r = p - i * YZ, j = r / Z, k = r - j * Z;
    const float f0 = __ldg(vol + p);
    const int stride[3] = {YZ, Z, 1};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        if (!((m >> a) & 1u)) continue;
        const float f1 = __ldg(vol + p + stride[a]);
        const float t = (iso - f0) / (f1 - f0);
        float pos[3] = {static_cast<float>(i), static_cast<float>(j), static_cast<float>(k)};
        pos[a] += t;
        float* v = verts + 3 * static_cast<size_t>(id);
        v[0] = fmaf(spacing.x, pos[0], origin.x);
        v[1] = fmaf(spacing.y, pos[1], origin.y);
        v[2] = fmaf(spacing.z, pos[2], origin.z);
        ++id;
    }
}

// (d) triangles in (cell, table slot) order; the vertex of edge e is vertex (popc of lower-axis crossings) of its owner point
__global__ void __launch_bounds__(MC_THREADS) mc_face_kernel(int X, int Y, int Z, const uint16_t* __restrict__ code, const long long* __restrict__ off_f,
                                                             const McHdr* __restrict__ hdr, const int* __restrict__ vbase, long long* __restrict__ faces) {
    __shared__ int8_t s_cnt[256];
    __shared__ int8_t s_tri[256 * 3 * kMcMaxTris];
    __shared__ int s_owner[12];
    __shared__ int8_t s_axis[12];
    __shared__ int s_warp[MC_THREADS / 32];
    if (hdr->V >= MC_INDEX_LIMIT || hdr->F >= MC_INDEX_LIMIT) return;
    const int N = X * Y * Z, YZ = Y * Z;
    s_cnt[threadIdx.x] = kMcTriCount[threadIdx.x];
    for (int e = threadIdx.x; e < 256 * 3 * kMcMaxTris; e += MC_THREADS) s_tri[e] = (&kMcTriEdges[0][0])[e];
    if (threadIdx.x < 12) {
        const int c = kMcEdgeOwner[threadIdx.x];
        s_owner[threadIdx.x] = (c & 1) * YZ + ((c >> 1) & 1) * Z + (c >> 2);
        s_axis[threadIdx.x] = kMcEdgeAxis[threadIdx.x];
    }
    __syncthreads();
    const int p = blockIdx.x * MC_THREADS + threadIdx.x;
    const int c = p < N ? (code[p] >> 8) : 0;
    const int nt = s_cnt[c];
    int total;
    const int excl = block_exclusive_scan(nt, s_warp, &total);
    if (nt == 0) return;
    long long* out = faces + 3 * (off_f[blockIdx.x] + excl);
    const int8_t* tri = s_tri + c * 3 * kMcMaxTris;
    for (int q = 0; q < 3 * nt; ++q) {
        const int e = tri[q];
        const int o = p + s_owner[e];
        const unsigned lower = (1u << s_axis[e]) - 1u;
        out[q] = static_cast<long long>(vbase[o]) + __popc(code[o] & 7u & lower);
    }
}

int mc_check(const float* vol, long long X, long long Y, long long Z, const void* ws, size_t ws_bytes, long long* N, long long* nb) {
    TPX_CHECK(vol != nullptr && ws != nullptr, TPX_ERR_ARG, "marching_cubes: null volume or workspace");
    TPX_CHECK(X >= 2 && Y >= 2 && Z >= 2, TPX_ERR_SHAPE, "marching_cubes: volume [%lld, %lld, %lld]: every dimension must be >= 2", X, Y, Z);
    TPX_CHECK(X < MC_INDEX_LIMIT && Y < MC_INDEX_LIMIT && Z < MC_INDEX_LIMIT && X * Y < MC_INDEX_LIMIT && X * Y * Z < MC_INDEX_LIMIT, TPX_ERR_SHAPE,
              "marching_cubes: volume [%lld, %lld, %lld] has 2^31 or more points", X, Y, Z);
    *N = X * Y * Z;
    *nb = (*N + MC_THREADS - 1) / MC_THREADS;
    TPX_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, TPX_ERR_ARG, "marching_cubes: workspace must be 256-B aligned");
    const size_t need = mc_carve(nullptr, *N, *nb).total;
    TPX_CHECK(ws_bytes >= need, TPX_ERR_ARG, "marching_cubes: workspace of %zu bytes, %zu needed", ws_bytes, need);
    return TPX_OK;
}
}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" {

size_t tpx_mc_workspace_bytes(int64_t X, int64_t Y, int64_t Z) {
    if (X < 2 || Y < 2 || Z < 2 || X >= MC_INDEX_LIMIT || Y >= MC_INDEX_LIMIT || Z >= MC_INDEX_LIMIT || X * Y >= MC_INDEX_LIMIT || X * Y * Z >= MC_INDEX_LIMIT)
        return 0;
    const long long N = X * Y * Z;
    return mc_carve(nullptr, N, (N + MC_THREADS - 1) / MC_THREADS).total;
}

int tpx_mc_count(const float* vol, int64_t X, int64_t Y, int64_t Z, float iso, void* ws, size_t ws_bytes, int64_t* counts, void* stream) {
    long long N, nb;
    const int rc = mc_check(vol, X, Y, Z, ws, ws_bytes, &N, &nb);
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr, TPX_ERR_ARG, "marching_cubes: null counts");
    TPX_DEVICE_GUARD();
    const McPtrs w = mc_carve(ws, N, nb);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    mc_count_kernel<<<static_cast<unsigned>(nb), MC_THREADS, 0, st>>>(vol, static_cast<int>(X), static_cast<int>(Y), static_cast<int>(Z), iso, w.code, w.blk_v,
                                                                      w.blk_f);
    TPX_LAUNCH_CHECK();
    mc_scan_kernel<<<1, MC_SCAN_THREADS, 0, st>>>(w.blk_v, w.blk_f, static_cast<int>(nb), w.off_v, w.off_f, w.hdr, reinterpret_cast<long long*>(counts));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_mc_emit(const float* vol, int64_t X, int64_t Y, int64_t Z, float iso, float ox, float oy, float oz, float sx, float sy, float sz, void* ws, size_t ws_bytes,
                float* verts, int64_t* faces, void* stream) {
    long long N, nb;
    const int rc = mc_check(vol, X, Y, Z, ws, ws_bytes, &N, &nb);
    if (rc != TPX_OK) return rc;
    TPX_DEVICE_GUARD();
    const McPtrs w = mc_carve(ws, N, nb);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_VAE_MISC, st);
    const int x = static_cast<int>(X), y = static_cast<int>(Y), z = static_cast<int>(Z);
    mc_vertex_kernel<<<static_cast<unsigned>(nb), MC_THREADS, 0, st>>>(vol, x, y, z, iso, make_float3(ox, oy, oz), make_float3(sx, sy, sz), w.code, w.off_v, w.hdr,
                                                                       w.vbase, verts);
    TPX_LAUNCH_CHECK();
    mc_face_kernel<<<static_cast<unsigned>(nb), MC_THREADS, 0, st>>>(x, y, z, w.code, w.off_f, w.hdr, w.vbase, reinterpret_cast<long long*>(faces));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // extern "C"
