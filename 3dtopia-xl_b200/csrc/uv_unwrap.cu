// Box-projection UV unwrap and the primitive noise filter (DESIGN.md §1 f-8): the fast-unwrap branch of extract_texmesh
// (inference.py:140-150, utils/uv_unwrap.py:65-685) and its first block (inference.py:90-103), on the device.
//   * vertex normals: face normals (v1 - v0) x (v2 - v0), summed per vertex in the order of the reference's three scatter_add_
//     calls (all corner-0 contributions by ascending face, then corner 1, then corner 2): the corners are sorted by vertex with a
//     stable radix sort over the corner-major list, and one thread sums each vertex's run.  No float atomics.
//   * unwrap: bbox, cube-face slice and projection, per-vertex tangents (the same sorted runs), per-slice mean tangents and angle
//     (one block per slice, fp64 sums in a fixed tree), rotation and joint rescale, two overlap passes over a uniform UV grid per
//     slice (sorted cell keys; each face scans the cells within 3 r of its centre and stores 1 into the flag of the face the
//     reference moves, so duplicate hits are idempotent), placement (slot-12 order from an exclusive scan), and unique rows from a
//     64-bit (u, v) key sort.
// Min / max reductions are atomics on order-preserving ints (exact); sums have a fixed order; every output position comes from a sort
// or a scan, so repeated calls on any stream give identical bytes.  Built with -fmad=false (build.py) with explicit _rn arithmetic, so
// that the numpy test oracle (unwrap.py) can follow the same operations.
#include <cub/cub.cuh>

#include "kernels.cuh"

namespace tpx {

namespace {
typedef unsigned long long u64;
constexpr int UW_THREADS = 256;
constexpr int UW_RED_THREADS = 1024;
constexpr long long UW_FACE_LIMIT = (1LL << 31) / 3;
constexpr int UW_NTAPS = 6;

unsigned blocks(long long n) { return static_cast<unsigned>((n + UW_THREADS - 1) / UW_THREADS); }
int bits_for(long long n) {
    int b = 1;
    while ((1LL << b) < n) ++b;
    return b;
}
// cells per side of the per-slice overlap grid: about four faces per cell if every face fell into one slice
int grid_side(long long F) {
    long long g = 1;
    while (g * g * 4 < F && g < 1024) ++g;
    return static_cast<int>(g);
}

// state the kernels exchange through the workspace
struct UwHdr {
    int bmin[3], bmax[3];    // bbox of the vertices (order-preserving ints)
    int divmax[3];           // max |coord| along the chosen axis, per corner slot
    int rmin[6], rmax[6];    // joint min / max of the rotated uv per slice
    int smin[6][2], smax[6][2];   // per-axis min / max of slots 6..11
    float rc[6], rs[6];      // cos / sin of the slice angle
    float angle[6];
    int bad;                 // faces with an index outside [0, V)
    long long U;             // unique uv rows (-1 for malformed input)
};

struct Ws {
    UwHdr* hdr;
    int* T;                  // validated faces int32 [F,3]
    int *ck[2], *cv[2];      // corner keys (vertex) / values (face), sorted
    int* vstart;             // [V+1] start of each vertex's run
    float* fvec;             // per-face vector [F,3] (face normal, then tangent)
    float *vtan, *vexp;      // per-vertex tangent, expected tangent [V,3]
    int* slice;              // [F]
    float* uvp;              // projected uv before the divisor [F,6]
    float* uv;               // projected uv [F,6]
    float* uvr;              // rotated, rescaled uv [F,6]
    float *cu, *cvv, *rad;   // uv centre and radius [F]
    int* assign;             // [F]
    unsigned *gk[2];         // grid keys
    int* gv[2];              // grid values (face)
    int* cstart;             // [6 G^2 + 1]
    int* flag;               // [F]
    int *is12, *pos12;       // [F]
    float* placed;           // [F,6]
    u64* uk[2];              // unique keys [3F]
    int* uvv[2];             // unique values (corner) [3F]
    int *head, *hscan;       // [3F]
    int* inv;                // [3F]
    u64* ukey;               // [3F] the unique keys, in order
    void* cub;
    size_t cub_bytes;
};

size_t cub_need(long long V, long long F, int G) {
    const long long n3 = 3 * F;
    size_t need = 0, b = 0;
    cub::DoubleBuffer<int> di(nullptr, nullptr);
    cub::DoubleBuffer<unsigned> du(nullptr, nullptr);
    cub::DoubleBuffer<u64> dk(nullptr, nullptr);
    if (cub::DeviceRadixSort::SortPairs(nullptr, b, di, di, static_cast<int>(n3), 0, bits_for(V + 1)) == cudaSuccess) need = b > need ? b : need;
    if (cub::DeviceRadixSort::SortPairs(nullptr, b, du, di, static_cast<int>(F), 0, bits_for(6LL * G * G + 1)) == cudaSuccess) need = b > need ? b : need;
    if (cub::DeviceRadixSort::SortPairs(nullptr, b, dk, di, static_cast<int>(n3), 0, 64) == cudaSuccess) need = b > need ? b : need;
    if (cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const int*>(nullptr), static_cast<int*>(nullptr), static_cast<int>(F)) == cudaSuccess)
        need = b > need ? b : need;
    if (cub::DeviceScan::InclusiveSum(nullptr, b, static_cast<const int*>(nullptr), static_cast<int*>(nullptr), static_cast<int>(n3)) == cudaSuccess)
        need = b > need ? b : need;
    return align_up(need + 4096, 256);
}

Ws carve(void* base, long long V, long long F, int G, size_t cub_bytes, size_t* total) {
    Carve c{static_cast<uint8_t*>(base)};
    Ws w{};
    const long long n3 = 3 * F, nc = 6LL * G * G + 1;
    w.hdr = c.take<UwHdr>(1);
    w.T = c.take<int>(n3);
    for (int i = 0; i < 2; ++i) {
        w.ck[i] = c.take<int>(n3);
        w.cv[i] = c.take<int>(n3);
    }
    w.vstart = c.take<int>(V + 1);
    w.fvec = c.take<float>(n3);
    w.vtan = c.take<float>(3 * V);
    w.vexp = c.take<float>(3 * V);
    w.slice = c.take<int>(F);
    w.uvp = c.take<float>(6 * F);
    w.uv = c.take<float>(6 * F);
    w.uvr = c.take<float>(6 * F);
    w.cu = c.take<float>(F);
    w.cvv = c.take<float>(F);
    w.rad = c.take<float>(F);
    w.assign = c.take<int>(F);
    for (int i = 0; i < 2; ++i) {
        w.gk[i] = c.take<unsigned>(F);
        w.gv[i] = c.take<int>(F);
    }
    w.cstart = c.take<int>(nc);
    w.flag = c.take<int>(F);
    w.is12 = c.take<int>(F);
    w.pos12 = c.take<int>(F);
    w.placed = c.take<float>(6 * F);
    for (int i = 0; i < 2; ++i) {
        w.uk[i] = c.take<u64>(n3);
        w.uvv[i] = c.take<int>(n3);
    }
    w.head = c.take<int>(n3);
    w.hscan = c.take<int>(n3);
    w.inv = c.take<int>(n3);
    w.ukey = c.take<u64>(n3);
    w.cub_bytes = cub_bytes;
    w.cub = c.take<uint8_t>(static_cast<long long>(cub_bytes));
    *total = c.off;
    return w;
}

// ------------------------------------------------------------------------------------------------------------ small helpers
__device__ __forceinline__ int ord_f32(float x) {
    const int b = __float_as_int(x);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float unord_f32(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float dvd(float a, float b) { return __fdiv_rn(a, b); }
// torch.clamp: NaN stays NaN
__device__ __forceinline__ float clamp_min(float x, float lo) { return x != x ? x : (x < lo ? lo : x); }
__device__ __forceinline__ float clamp01(float x) { return x != x ? x : (x < 0.0f ? 0.0f : (x > 1.0f ? 1.0f : x)); }
__device__ __forceinline__ float dot3(const float* a, const float* b) { return add(add(mul(a[0], b[0]), mul(a[1], b[1])), mul(a[2], b[2])); }
// F.normalize(x, eps): x / max(|x|, eps), |x| = sqrt((x0^2 + x1^2) + x2^2)
__device__ __forceinline__ void normalize3(float* x, float eps) {
    const float n = clamp_min(__fsqrt_rn(dot3(x, x)), eps);
    x[0] = dvd(x[0], n), x[1] = dvd(x[1], n), x[2] = dvd(x[2], n);
}
// F.normalize(x, -1) as the reference calls it for the expected tangent (uv_unwrap.py:414-419): -1 is p, not dim, so the divisor is
// max(1 / ((1/|x0| + 1/|x1|) + 1/|x2|), 1e-12), and a zero component makes it 1e-12
__device__ __forceinline__ void normalize_pm1(float* x) {
    const float n = clamp_min(dvd(1.0f, add(add(dvd(1.0f, fabsf(x[0])), dvd(1.0f, fabsf(x[1]))), dvd(1.0f, fabsf(x[2])))), 1e-12f);
    x[0] = dvd(x[0], n), x[1] = dvd(x[1], n), x[2] = dvd(x[2], n);
}
__device__ __forceinline__ void cross3(const float* a, const float* b, float* o) {
    o[0] = sub(mul(a[1], b[2]), mul(a[2], b[1]));
    o[1] = sub(mul(a[2], b[0]), mul(a[0], b[2]));
    o[2] = sub(mul(a[0], b[1]), mul(a[1], b[0]));
}

// ------------------------------------------------------------------------------------------------------------ shared stages
__global__ void __launch_bounds__(UW_THREADS) faces_kernel(const int* __restrict__ fin, long long F, long long V, int* __restrict__ T, int* bad) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    bool ok = true;
    int t[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        t[k] = fin[3 * f + k];
        ok = ok && t[k] >= 0 && t[k] < V;
    }
    if (!ok) atomicAdd(bad, 1);
#pragma unroll
    for (int k = 0; k < 3; ++k) T[3 * f + k] = ok ? t[k] : 0;   // clamped so no later stage reads out of bounds
}

// corner h = c F + f (corner-major): key = its vertex, value = its face; a stable sort then orders each vertex's run as the
// reference's scatter_add_ calls visit it
__global__ void __launch_bounds__(UW_THREADS) corner_keys_kernel(const int* __restrict__ T, long long F, int* __restrict__ key, int* __restrict__ val) {
    const long long h = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (h >= 3 * F) return;
    const long long c = h / F, f = h - c * F;
    key[h] = T[3 * f + c];
    val[h] = static_cast<int>(f);
}

// vstart[v] = first sorted corner with key >= v, v in [0, V]
__global__ void __launch_bounds__(UW_THREADS) run_start_kernel(const int* __restrict__ key, long long n, long long V, int* __restrict__ start) {
    const long long v = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (v > V) return;
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (key[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    start[v] = static_cast<int>(lo);
}

__global__ void __launch_bounds__(UW_THREADS) face_normal_kernel(const float* __restrict__ P, const int* __restrict__ T, long long F, float* __restrict__ out) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const float* p0 = P + 3 * T[3 * f];
    const float* p1 = P + 3 * T[3 * f + 1];
    const float* p2 = P + 3 * T[3 * f + 2];
    float a[3], b[3], n[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) a[d] = sub(p1[d], p0[d]), b[d] = sub(p2[d], p0[d]);
    cross3(a, b, n);
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * f + d] = n[d];
}

// compute_vertex_normal (uv_unwrap.py:65-85): the run's face normals summed in order; |n|^2 <= 1e-20 -> (0,0,1); normalised
__global__ void __launch_bounds__(UW_THREADS) vertex_normal_kernel(const int* __restrict__ start, const int* __restrict__ face, const float* __restrict__ fn,
                                                                   long long V, float* __restrict__ out) {
    const long long v = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (v >= V) return;
    float s[3] = {0.0f, 0.0f, 0.0f};
    for (int i = start[v]; i < start[v + 1]; ++i) {
        const float* n = fn + 3 * static_cast<long long>(face[i]);
        s[0] = add(s[0], n[0]), s[1] = add(s[1], n[1]), s[2] = add(s[2], n[2]);
    }
    if (!(dot3(s, s) > 1e-20f)) s[0] = 0.0f, s[1] = 0.0f, s[2] = 1.0f;
    normalize3(s, 1e-12f);
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * v + d] = s[d];
}

// ------------------------------------------------------------------------------------------------------------ stage 2: projection
__global__ void __launch_bounds__(UW_THREADS) bbox_kernel(const float* __restrict__ P, long long V, UwHdr* hdr) {
    const long long v = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (v >= V) return;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const int o = ord_f32(P[3 * v + d]);
        atomicMin(&hdr->bmin[d], o);
        atomicMax(&hdr->bmax[d], o);
    }
}

// _box_assign_vertex_to_cube_face (uv_unwrap.py:87-179) up to the divisor: slice = first argmax of (x, -x, y, -y, z, -z) of the
// normalised summed vertex normals; (u, v) from the slice's table; per corner slot the max |coord| along the slice's axis
__global__ void __launch_bounds__(UW_THREADS) project_kernel(const float* __restrict__ P, const float* __restrict__ N, const int* __restrict__ T, long long F,
                                                             UwHdr* hdr, int* __restrict__ slice, float* __restrict__ uvp) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    float lo[3], ext[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        lo[d] = unord_f32(hdr->bmin[d]);
        ext[d] = sub(unord_f32(hdr->bmax[d]), lo[d]);
    }
    float fnrm[3] = {0.0f, 0.0f, 0.0f};
    float q[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const long long v = T[3 * f + k];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            q[k][d] = sub(mul(2.0f, dvd(sub(P[3 * v + d], lo[d]), ext[d])), 1.0f);
            fnrm[d] = k == 0 ? N[3 * v + d] : add(fnrm[d], N[3 * v + d]);
        }
    }
    normalize3(fnrm, 1e-6f);
    const float dots[6] = {fnrm[0], -fnrm[0], fnrm[1], -fnrm[1], fnrm[2], -fnrm[2]};
    int s = 0;
#pragma unroll
    for (int i = 1; i < 6; ++i)
        if (dots[i] > dots[s]) s = i;
    slice[f] = s;
    const int ax = s >> 1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float u, v;
        if (s <= 1) u = q[k][1], v = -q[k][2];
        else if (s <= 3) u = q[k][0], v = -q[k][2];
        else if (s == 4) u = q[k][0], v = q[k][1];
        else u = q[k][0], v = -q[k][1];
        uvp[6 * f + 2 * k] = u;
        uvp[6 * f + 2 * k + 1] = v;
        atomicMax(&hdr->divmax[k], ord_f32(fabsf(q[k][ax])));
    }
}

__global__ void __launch_bounds__(UW_THREADS) project_div_kernel(const float* __restrict__ uvp, long long F, const UwHdr* hdr, float* __restrict__ uv) {
    const long long i = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (i >= 6 * F) return;
    const int k = static_cast<int>((i % 6) >> 1);
    uv[i] = clamp01(mul(add(dvd(uvp[i], unord_f32(hdr->divmax[k])), 1.0f), 0.5f));
}

// ------------------------------------------------------------------------------------------------------------ stage 3: rotation
// calculate_tangents (uv_unwrap.py:349-395), per face: (dpos1 duv2.y - dpos2 duv1.y) / max(duv1.x duv2.y - duv1.y duv2.x, 1e-6)
__global__ void __launch_bounds__(UW_THREADS) face_tangent_kernel(const float* __restrict__ P, const int* __restrict__ T, const float* __restrict__ uv, long long F,
                                                                  float* __restrict__ out) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const float* t = uv + 6 * f;
    const float d1x = sub(t[2], t[0]), d1y = sub(t[3], t[1]), d2x = sub(t[4], t[0]), d2y = sub(t[5], t[1]);
    const float den = clamp_min(sub(mul(d1x, d2y), mul(d1y, d2x)), 1e-6f);
    const float* p0 = P + 3 * T[3 * f];
    const float* p1 = P + 3 * T[3 * f + 1];
    const float* p2 = P + 3 * T[3 * f + 2];
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * f + d] = dvd(sub(mul(sub(p1[d], p0[d]), d2y), mul(sub(p2[d], p0[d]), d1y)), den);
}

// per vertex: the run's tangents summed in order, / count, normalised, made perpendicular to the normal, normalised; and the
// expected tangent n x ((-y, x, 0) x n) divided by its (-1)-norm (normalize_pm1)
__global__ void __launch_bounds__(UW_THREADS) vertex_tangent_kernel(const int* __restrict__ start, const int* __restrict__ face, const float* __restrict__ ft,
                                                                    const float* __restrict__ P, const float* __restrict__ N, long long V,
                                                                    float* __restrict__ vtan, float* __restrict__ vexp) {
    const long long v = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (v >= V) return;
    float s[3] = {0.0f, 0.0f, 0.0f}, cnt = 0.0f;
    for (int i = start[v]; i < start[v + 1]; ++i) {
        const float* t = ft + 3 * static_cast<long long>(face[i]);
        s[0] = add(s[0], t[0]), s[1] = add(s[1], t[1]), s[2] = add(s[2], t[2]);
        cnt = add(cnt, 1.0f);
    }
    const float n[3] = {N[3 * v], N[3 * v + 1], N[3 * v + 2]};
    s[0] = dvd(s[0], cnt), s[1] = dvd(s[1], cnt), s[2] = dvd(s[2], cnt);
    normalize3(s, 1e-12f);
    const float dn = dot3(s, n);
#pragma unroll
    for (int d = 0; d < 3; ++d) s[d] = sub(s[d], mul(dn, n[d]));
    normalize3(s, 1e-12f);
    const float ps[3] = {-P[3 * v + 1], P[3 * v], 0.0f};
    float c1[3], e[3];
    cross3(ps, n, c1);
    cross3(n, c1, e);
    normalize_pm1(e);
#pragma unroll
    for (int d = 0; d < 3; ++d) vtan[3 * v + d] = s[d], vexp[3 * v + d] = e[d];
}

// one block per slice: the mean over faces x corners of both tangent sets (fp64 sums in a fixed order, rounded to fp32), the
// angle atan2(a.x e.y - a.y e.x, a . e) and its cosine / sine (uv_unwrap.py:429-446)
__global__ void __launch_bounds__(UW_RED_THREADS) slice_angle_kernel(const int* __restrict__ T, const int* __restrict__ slice, long long F,
                                                                     const float* __restrict__ vtan, const float* __restrict__ vexp, UwHdr* hdr) {
    __shared__ double red[UW_RED_THREADS / 32][7];
    const int s = blockIdx.x;
    double acc[7] = {0, 0, 0, 0, 0, 0, 0};
    for (long long f = threadIdx.x; f < F; f += UW_RED_THREADS) {
        if (slice[f] != s) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const long long v = T[3 * f + k];
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                acc[d] = __dadd_rn(acc[d], static_cast<double>(vtan[3 * v + d]));
                acc[3 + d] = __dadd_rn(acc[3 + d], static_cast<double>(vexp[3 * v + d]));
            }
        }
        acc[6] = __dadd_rn(acc[6], 3.0);
    }
#pragma unroll
    for (int j = 0; j < 7; ++j)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] = __dadd_rn(acc[j], __shfl_down_sync(0xffffffffu, acc[j], o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0)
#pragma unroll
        for (int j = 0; j < 7; ++j) red[warp][j] = acc[j];
    __syncthreads();
    if (warp != 0) return;
#pragma unroll
    for (int j = 0; j < 7; ++j) {
        acc[j] = red[lane][j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[j] = __dadd_rn(acc[j], __shfl_down_sync(0xffffffffu, acc[j], o));
    }
    if (lane != 0) return;
    float a[3], e[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        a[d] = __double2float_rn(__ddiv_rn(acc[d], acc[6]));
        e[d] = __double2float_rn(__ddiv_rn(acc[3 + d], acc[6]));
    }
    const float ang = atan2f(sub(mul(a[0], e[1]), mul(a[1], e[0])), dot3(a, e));
    hdr->angle[s] = acc[6] > 0 ? ang : 0.0f;
    hdr->rc[s] = cosf(ang);
    hdr->rs[s] = sinf(ang);
}

__global__ void __launch_bounds__(UW_THREADS) rotate_kernel(const float* __restrict__ uv, const int* __restrict__ slice, long long F, UwHdr* hdr,
                                                            float* __restrict__ uvr) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int s = slice[f];
    const float c = hdr->rc[s], sn = hdr->rs[s];
    int lo = 0x7fffffff, hi = static_cast<int>(0x80000000);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float u = sub(mul(uv[6 * f + 2 * k], 2.0f), 1.0f), v = sub(mul(uv[6 * f + 2 * k + 1], 2.0f), 1.0f);
        const float ru = add(mul(c, u), mul(-sn, v)), rv = add(mul(sn, u), mul(c, v));
        uvr[6 * f + 2 * k] = ru;
        uvr[6 * f + 2 * k + 1] = rv;
        lo = min(lo, min(ord_f32(ru), ord_f32(rv)));
        hi = max(hi, max(ord_f32(ru), ord_f32(rv)));
    }
    atomicMin(&hdr->rmin[s], lo);
    atomicMax(&hdr->rmax[s], hi);
}

// rescale by the slice's joint min / max; then the overlap test's centre (mean of the corners) and radius (max corner distance)
__global__ void __launch_bounds__(UW_THREADS) rescale_kernel(const int* __restrict__ slice, long long F, const UwHdr* hdr, float* __restrict__ uvr,
                                                             float* __restrict__ cu, float* __restrict__ cv, float* __restrict__ rad, int* __restrict__ assign) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int s = slice[f];
    const float lo = unord_f32(hdr->rmin[s]), ext = sub(unord_f32(hdr->rmax[s]), lo);
    float t[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) uvr[6 * f + i] = t[i] = dvd(sub(uvr[6 * f + i], lo), ext);
    const float mu = dvd(add(add(t[0], t[2]), t[4]), 3.0f), mv = dvd(add(add(t[1], t[3]), t[5]), 3.0f);
    float r = 0.0f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float du = sub(t[2 * k], mu), dv = sub(t[2 * k + 1], mv);
        const float d = __fsqrt_rn(add(mul(du, du), mul(dv, dv)));
        r = k == 0 ? d : (d > r || d != d ? d : r);
    }
    cu[f] = mu, cv[f] = mv, rad[f] = r;
    assign[f] = s;
}

// ------------------------------------------------------------------------------------------------------------ stage 4: overlaps
__device__ __forceinline__ int cell_of(float c, int G) {
    const float x = floorf(mul(c, static_cast<float>(G)));
    return x != x ? 0 : static_cast<int>(fminf(fmaxf(x, 0.0f), static_cast<float>(G - 1)));
}

__global__ void __launch_bounds__(UW_THREADS) grid_key_kernel(const int* __restrict__ assign, const float* __restrict__ cu, const float* __restrict__ cv, long long F,
                                                              int pass, int G, unsigned* __restrict__ key, int* __restrict__ val) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int i = assign[f] - 6 * pass;
    const unsigned GG = static_cast<unsigned>(G) * G;
    key[f] = (i >= 0 && i < 6) ? i * GG + cell_of(cv[f], G) * G + cell_of(cu[f], G) : 6 * GG;
    val[f] = static_cast<int>(f);
}

__global__ void __launch_bounds__(UW_THREADS) cell_start_kernel(const unsigned* __restrict__ key, long long n, long long ncell, int* __restrict__ start) {
    const long long c = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (c > ncell) return;
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (key[mid] < c) lo = mid + 1;
        else hi = mid;
    }
    start[c] = static_cast<int>(lo);
}

// tri_winding (uv_unwrap.py:9-17): rows 1 and 2 swapped when the determinant of [[u, v, 1]] is negative
__device__ __forceinline__ void wound(const float* t, double* w) {
    const double u0 = t[0], v0 = t[1], u1 = t[2], v1 = t[3], u2 = t[4], v2 = t[5];
    const double det = __dsub_rn(__dmul_rn(__dsub_rn(u1, u0), __dsub_rn(v2, v0)), __dmul_rn(__dsub_rn(v1, v0), __dsub_rn(u2, u0)));
    const bool flip = det < 0.0;
    w[0] = u0, w[1] = v0;
    w[2] = flip ? u2 : u1, w[3] = flip ? v2 : v1;
    w[4] = flip ? u1 : u2, w[5] = flip ? v1 : v2;
}
// chk_edge: the point is "outside" the edge a -> b unless det [[a,1],[b,1],[p,1]] > 1e-6 (a NaN det is outside)
__device__ __forceinline__ bool outside(double ax, double ay, double bx, double by, double px, double py) {
    const double det = __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(py, ay)), __dmul_rn(__dsub_rn(by, ay), __dsub_rn(px, ax)));
    return !(det > 1e-6);
}
// an edge of a separates b when all three points of b are outside it; edges (0,1), (2,0), (1,2) as torch.roll gives them
__device__ __forceinline__ bool separates(const double* a, const double* b) {
    const int e0[3] = {0, 2, 1}, e1[3] = {1, 0, 2};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const double ax = a[2 * e0[i]], ay = a[2 * e0[i] + 1], bx = a[2 * e1[i]], by = a[2 * e1[i] + 1];
        if (outside(ax, ay, bx, by, b[0], b[1]) && outside(ax, ay, bx, by, b[2], b[3]) && outside(ax, ay, bx, by, b[4], b[5])) return true;
    }
    return false;
}

__global__ void __launch_bounds__(UW_THREADS) overlap_kernel(const unsigned* __restrict__ key, const int* __restrict__ val, long long F, int pass, int G,
                                                             const int* __restrict__ cstart, const float* __restrict__ cu, const float* __restrict__ cv,
                                                             const float* __restrict__ rad, const float* __restrict__ uvr, const float* __restrict__ P,
                                                             const int* __restrict__ T, int* __restrict__ flag) {
    const long long p = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (p >= F) return;
    const unsigned GG = static_cast<unsigned>(G) * G;
    const unsigned k = key[p];
    if (k >= 6 * GG) return;
    const int i = static_cast<int>(k / GG);
    const int slice = i + 6 * pass;
    const int a = val[p];
    const float ua = cu[a], va = cv[a], r3 = mul(rad[a], 3.0f);
    if (!(r3 >= 0.0f)) return;
    const int x0 = max(cell_of(sub(ua, r3), G) - 1, 0), x1 = min(cell_of(add(ua, r3), G) + 1, G - 1);
    const int y0 = max(cell_of(sub(va, r3), G) - 1, 0), y1 = min(cell_of(add(va, r3), G) + 1, G - 1);
    double wa[6];
    wound(uvr + 6 * static_cast<long long>(a), wa);
    const int ax = slice < 2 ? 0 : (slice < 4 ? 1 : 2);
    const bool use_max = slice & 1;
    for (int y = y0; y <= y1; ++y) {
        const long long row = static_cast<long long>(i) * GG + static_cast<long long>(y) * G;
        for (int j = cstart[row + x0]; j < cstart[row + x1 + 1]; ++j) {
            const int b = val[j];
            if (b == a) continue;
            const float du = sub(cu[b], ua), dv = sub(cv[b], va);
            if (!(__fsqrt_rn(add(mul(du, du), mul(dv, dv))) <= r3)) continue;
            double wb[6];
            wound(uvr + 6 * static_cast<long long>(b), wb);
            if (separates(wa, wb) || separates(wb, wa)) continue;
            // the face the reference moves: first = min id, second = max id; mark_first compares their 3-D centroids on `ax`
            const int lo = min(a, b), hi = max(a, b);
            float c[2];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const long long f = q ? hi : lo;
                c[q] = dvd(add(add(P[3 * T[3 * f] + ax], P[3 * T[3 * f + 1] + ax]), P[3 * T[3 * f + 2] + ax]), 3.0f);
            }
            const bool mark = use_max ? c[0] > c[1] : c[0] < c[1];
            flag[mark ? hi : lo] = 1;
        }
    }
}

__global__ void __launch_bounds__(UW_THREADS) shift_kernel(const int* __restrict__ flag, long long F, int* __restrict__ assign) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    if (flag[f]) assign[f] = min(assign[f] + 6, 12);
}

// ------------------------------------------------------------------------------------------------------------ stage 5: placement
__global__ void __launch_bounds__(UW_THREADS) slot_minmax_kernel(const int* __restrict__ assign, const float* __restrict__ uvr, long long F, UwHdr* hdr,
                                                                 int* __restrict__ is12) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int a = assign[f];
    is12[f] = a >= 12;
    if (a < 6 || a >= 12) return;
#pragma unroll
    for (int d = 0; d < 2; ++d) {
        int lo = 0x7fffffff, hi = static_cast<int>(0x80000000);
#pragma unroll
        for (int k = 0; k < 3; ++k) lo = min(lo, ord_f32(uvr[6 * f + 2 * k + d])), hi = max(hi, ord_f32(uvr[6 * f + 2 * k + d]));
        atomicMin(&hdr->smin[a - 6][d], lo);
        atomicMax(&hdr->smax[a - 6][d], hi);
    }
}

struct PlaceConsts {
    float pad_mul, pad_add;   // 1 - 2 p, p
    float fin_mul, fin_add;   // 1 - 2 p 0.5, p 0.5
    double pad;               // p
};

// _distribute_individual_uvs_in_atlas (uv_unwrap.py:457-570) and the unique key of every corner
__global__ void __launch_bounds__(UW_THREADS) place_kernel(const int* __restrict__ assign, const float* __restrict__ uvr, const int* __restrict__ is12,
                                                           const int* __restrict__ pos12, long long F, UwHdr* hdr, PlaceConsts pc, float* __restrict__ placed,
                                                           u64* __restrict__ ukey, int* __restrict__ uval) {
    const long long f = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int a = assign[f];
    float t[6];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int d = 0; d < 2; ++d) {
            float x = uvr[6 * f + 2 * k + d];
            if (a >= 6 && a < 12) {
                const float lo = unord_f32(hdr->smin[a - 6][d]);
                x = dvd(sub(x, lo), clamp_min(sub(unord_f32(hdr->smax[a - 6][d]), lo), 0.5f));
            }
            t[2 * k + d] = clamp01(add(mul(x, pc.pad_mul), pc.pad_add));
        }
    float ox, oy, dx, dy;
    if (a >= 12) {
        const long long n12 = F ? static_cast<long long>(pos12[F - 1]) + is12[F - 1] : 0;
        const double mult = sqrt(static_cast<double>(n12) / (0.5 * (1.0 / 3.0)));
        const long long nw = static_cast<long long>(ceil(0.5 * mult));
        const long long nh = static_cast<long long>(ceil(static_cast<double>(n12) / static_cast<double>(nw)));
        const double width = 1.0 / static_cast<double>(nw), height = 1.0 / static_cast<double>(nh);
        const float clip = static_cast<float>(fmin(width, height) * 1.5);
        const float sm[2] = {static_cast<float>(1.0 - pc.pad * static_cast<double>(nw) * 0.5), static_cast<float>(1.0 - pc.pad * static_cast<double>(nh) * 0.5)};
        const float sa[2] = {static_cast<float>(pc.pad * static_cast<double>(nw) * 0.25), static_cast<float>(pc.pad * static_cast<double>(nh) * 0.25)};
        const float wh[2] = {static_cast<float>(width), static_cast<float>(height)};
        const int idx = pos12[f];
        const float cell[2] = {static_cast<float>(idx % nw), static_cast<float>(idx / nw)};
#pragma unroll
        for (int d = 0; d < 2; ++d) {
            const float lo = fminf(fminf(t[d], t[2 + d]), t[4 + d]), hi = fmaxf(fmaxf(t[d], t[2 + d]), t[4 + d]);
            const float ext = clamp_min(sub(hi, lo), clip);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float x = dvd(sub(t[2 * k + d], lo), ext);
                x = clamp01(add(mul(x, sm[d]), sa[d]));
                x = add(mul(x, wh[d]), mul(cell[d], wh[d]));
                t[2 * k + d] = clamp01(add(mul(x, pc.fin_mul), pc.fin_add));
            }
        }
        ox = 0.5f, oy = static_cast<float>(1.0 / 3.0 * 2.0), dx = 2.0f, dy = 3.0f;
    } else {
        const int m = a % 6;
        const double gx = m % 3, gy = m / 3;
        if (a < 6) ox = static_cast<float>(1.0 / 3.0 * gx), oy = static_cast<float>(1.0 / 3.0 * gy), dx = dy = 3.0f;
        else ox = static_cast<float>(1.0 / 6.0 * gx), oy = static_cast<float>(1.0 / 6.0 * gy + 1.0 / 3.0 * 2.0), dx = dy = 6.0f;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float u = add(dvd(t[2 * k], dx), ox), v = add(dvd(t[2 * k + 1], dy), oy);
        placed[6 * f + 2 * k] = u;
        placed[6 * f + 2 * k + 1] = v;
        ukey[3 * f + k] = (static_cast<u64>(__float_as_uint(u)) << 32) | __float_as_uint(v);
        uval[3 * f + k] = static_cast<int>(3 * f + k);
    }
}

// ------------------------------------------------------------------------------------------------------------ stage 6: unique
__global__ void __launch_bounds__(UW_THREADS) head_kernel(const u64* __restrict__ key, long long n, int* __restrict__ head) {
    const long long p = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (p >= n) return;
    head[p] = p == 0 || key[p] != key[p - 1];
}

__global__ void __launch_bounds__(UW_THREADS) unique_kernel(const u64* __restrict__ key, const int* __restrict__ val, const int* __restrict__ head,
                                                            const int* __restrict__ scan, long long n, int* __restrict__ inv, u64* __restrict__ ukey) {
    const long long p = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (p >= n) return;
    const int u = scan[p] - 1;
    inv[val[p]] = u;
    if (head[p]) ukey[u] = key[p];
}

__global__ void hdr_init_kernel(UwHdr* h) {
    const int lo = 0x7fffffff, hi = static_cast<int>(0x80000000);
    for (int d = 0; d < 3; ++d) h->bmin[d] = lo, h->bmax[d] = hi, h->divmax[d] = hi;
    for (int s = 0; s < 6; ++s) {
        h->rmin[s] = lo, h->rmax[s] = hi, h->angle[s] = 0.0f;
        for (int d = 0; d < 2; ++d) h->smin[s][d] = lo, h->smax[s][d] = hi;
    }
    h->bad = 0;
    h->U = 0;
}

__global__ void unique_count_kernel(const int* __restrict__ scan, long long n, UwHdr* hdr) {
    hdr->U = hdr->bad ? -1 : (n ? scan[n - 1] : 0);
}

__global__ void __launch_bounds__(UW_THREADS) emit_kernel(const u64* __restrict__ ukey, const int* __restrict__ inv, long long n, const UwHdr* hdr,
                                                          float* __restrict__ uv, long long* __restrict__ vidx) {
    const long long p = blockIdx.x * static_cast<long long>(UW_THREADS) + threadIdx.x;
    if (p >= n) return;
    vidx[p] = inv[p];
    if (p < hdr->U) {
        uv[2 * p] = __uint_as_float(static_cast<unsigned>(ukey[p] >> 32));
        uv[2 * p + 1] = __uint_as_float(static_cast<unsigned>(ukey[p]));
    }
}

// ------------------------------------------------------------------------------------------------------------ noise filter
constexpr int NF_THREADS = 256;
// inference.py:90-103: d_ij = sqrt(sum((p_i - p_j)^2)) + (i == j); nn = first argmin; keep = d_nn < s_i + s_nn
__global__ void __launch_bounds__(NF_THREADS) noise_filter_kernel(const float* __restrict__ srt, int K, uint8_t* __restrict__ keep, int* __restrict__ nn_out) {
    __shared__ float sp[NF_THREADS][3];
    const int i = blockIdx.x * NF_THREADS + threadIdx.x;
    float pi[3] = {0.0f, 0.0f, 0.0f};
    if (i < K)
#pragma unroll
        for (int d = 0; d < 3; ++d) pi[d] = srt[4 * i + 1 + d];
    float best = 0.0f;
    int nn = -1;
    for (int j0 = 0; j0 < K; j0 += NF_THREADS) {
        __syncthreads();
        if (j0 + threadIdx.x < K)
#pragma unroll
            for (int d = 0; d < 3; ++d) sp[threadIdx.x][d] = srt[4 * (j0 + threadIdx.x) + 1 + d];
        __syncthreads();
        const int jn = min(NF_THREADS, K - j0);
        for (int jj = 0; jj < jn; ++jj) {
            const float dx = sub(pi[0], sp[jj][0]), dy = sub(pi[1], sp[jj][1]), dz = sub(pi[2], sp[jj][2]);
            float d = __fsqrt_rn(add(add(mul(dx, dx), mul(dy, dy)), mul(dz, dz)));
            if (j0 + jj == i) d = add(d, 1.0f);
            if (nn < 0 || d < best) best = d, nn = j0 + jj;
        }
    }
    if (i >= K) return;
    keep[i] = best < add(srt[4 * i], srt[4 * nn]);
    if (nn_out) nn_out[i] = nn;
}
}  // namespace

// ------------------------------------------------------------------------------------------------------------ entry points
namespace {
int uw_check(long long V, long long F) {
    TPX_CHECK(V >= 1 && F >= 1 && V < (1LL << 31) - 1 && F < UW_FACE_LIMIT, TPX_ERR_ARG, "uv unwrap: need 1 <= V < 2^31 - 1 and 1 <= F < 2^31 / 3 (V=%lld F=%lld)", V, F);
    return TPX_OK;
}

// faces in, corners sorted by vertex, vertex runs
int uw_prologue(const Ws& w, const int* faces, long long V, long long F, cudaStream_t st) {
    const long long n3 = 3 * F;
    faces_kernel<<<blocks(F), UW_THREADS, 0, st>>>(faces, F, V, w.T, &w.hdr->bad);
    TPX_LAUNCH_CHECK();
    corner_keys_kernel<<<blocks(n3), UW_THREADS, 0, st>>>(w.T, F, w.ck[0], w.cv[0]);
    TPX_LAUNCH_CHECK();
    cub::DoubleBuffer<int> dk(w.ck[0], w.ck[1]), dv(w.cv[0], w.cv[1]);
    size_t b = w.cub_bytes;
    TPX_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, b, dk, dv, static_cast<int>(n3), 0, bits_for(V + 1), st));
    run_start_kernel<<<blocks(V + 1), UW_THREADS, 0, st>>>(dk.Current(), n3, V, w.vstart);
    TPX_LAUNCH_CHECK();
    if (dk.Current() != w.ck[0]) {     // keep the sorted runs in the fixed buffers
        TPX_CUDA(cudaMemcpyAsync(w.ck[0], dk.Current(), n3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
        TPX_CUDA(cudaMemcpyAsync(w.cv[0], dv.Current(), n3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
    }
    return TPX_OK;
}

int uw_setup(void* ws, size_t ws_bytes, long long V, long long F, Ws* out) {
    const int G = grid_side(F);
    size_t total = 0;
    carve(nullptr, V, F, G, 0, &total);
    const size_t cb = cub_need(V, F, G);
    TPX_CHECK(ws_bytes >= total + align_up(cb, 256), TPX_ERR_ARG, "uv unwrap: workspace of %zu bytes, need %zu", ws_bytes, total + align_up(cb, 256));
    TPX_CHECK(ws != nullptr && (reinterpret_cast<uintptr_t>(ws) & 255) == 0, TPX_ERR_ARG, "uv unwrap: workspace must be 256-B aligned");
    *out = carve(ws, V, F, G, cb, &total);
    return TPX_OK;
}

}  // namespace

extern "C" {

size_t tpx_uv_unwrap_workspace_bytes(int64_t V, int64_t F) {
    if (V < 1 || F < 1 || V >= (1LL << 31) - 1 || F >= UW_FACE_LIMIT) return 0;
    size_t total = 0;
    const int G = grid_side(F);
    carve(nullptr, V, F, G, 0, &total);
    return total + align_up(cub_need(V, F, G), 256);
}

int tpx_vertex_normals(const float* verts_dev, int64_t V, const int32_t* faces_dev, int64_t F, void* ws, size_t ws_bytes, float* normals_dev, void* stream) {
    if (int rc = uw_check(V, F)) return rc;
    TPX_CHECK(verts_dev && faces_dev && normals_dev, TPX_ERR_ARG, "tpx_vertex_normals: null pointer");
    TPX_DEVICE_GUARD();   // first: the workspace check sizes the CUB scratch, a CUDA query
    Ws w;
    if (int rc = uw_setup(ws, ws_bytes, V, F, &w)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TPX_CUDA(cudaMemsetAsync(&w.hdr->bad, 0, sizeof(int), st));
    if (int rc = uw_prologue(w, faces_dev, V, F, st)) return rc;
    face_normal_kernel<<<blocks(F), UW_THREADS, 0, st>>>(verts_dev, w.T, F, w.fvec);
    TPX_LAUNCH_CHECK();
    vertex_normal_kernel<<<blocks(V), UW_THREADS, 0, st>>>(w.vstart, w.cv[0], w.fvec, V, normals_dev);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_uv_unwrap(const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F, double island_padding, void* ws,
                  size_t ws_bytes, int64_t* count_dev, void** taps_host, void* stream) {
    if (int rc = uw_check(V, F)) return rc;
    TPX_CHECK(verts_dev && normals_dev && faces_dev && count_dev, TPX_ERR_ARG, "tpx_uv_unwrap: null pointer");
    TPX_CHECK(island_padding >= 0.0 && island_padding < 0.5, TPX_ERR_ARG, "tpx_uv_unwrap: island_padding %g outside [0, 0.5)", island_padding);
    TPX_DEVICE_GUARD();
    Ws w;
    if (int rc = uw_setup(ws, ws_bytes, V, F, &w)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n3 = 3 * F;
    const int G = grid_side(F);
    const long long ncell = 6LL * G * G;
    hdr_init_kernel<<<1, 1, 0, st>>>(w.hdr);
    TPX_LAUNCH_CHECK();
    if (int rc = uw_prologue(w, faces_dev, V, F, st)) return rc;
    // stage 2
    bbox_kernel<<<blocks(V), UW_THREADS, 0, st>>>(verts_dev, V, w.hdr);
    TPX_LAUNCH_CHECK();
    project_kernel<<<blocks(F), UW_THREADS, 0, st>>>(verts_dev, normals_dev, w.T, F, w.hdr, w.slice, w.uvp);
    TPX_LAUNCH_CHECK();
    project_div_kernel<<<blocks(6 * F), UW_THREADS, 0, st>>>(w.uvp, F, w.hdr, w.uv);
    TPX_LAUNCH_CHECK();
    // stage 3
    face_tangent_kernel<<<blocks(F), UW_THREADS, 0, st>>>(verts_dev, w.T, w.uv, F, w.fvec);
    TPX_LAUNCH_CHECK();
    vertex_tangent_kernel<<<blocks(V), UW_THREADS, 0, st>>>(w.vstart, w.cv[0], w.fvec, verts_dev, normals_dev, V, w.vtan, w.vexp);
    TPX_LAUNCH_CHECK();
    slice_angle_kernel<<<6, UW_RED_THREADS, 0, st>>>(w.T, w.slice, F, w.vtan, w.vexp, w.hdr);
    TPX_LAUNCH_CHECK();
    rotate_kernel<<<blocks(F), UW_THREADS, 0, st>>>(w.uv, w.slice, F, w.hdr, w.uvr);
    TPX_LAUNCH_CHECK();
    rescale_kernel<<<blocks(F), UW_THREADS, 0, st>>>(w.slice, F, w.hdr, w.uvr, w.cu, w.cvv, w.rad, w.assign);
    TPX_LAUNCH_CHECK();
    // stage 4: two passes (a third could only move faces already clamped to slot 12)
    for (int pass = 0; pass < 2; ++pass) {
        grid_key_kernel<<<blocks(F), UW_THREADS, 0, st>>>(w.assign, w.cu, w.cvv, F, pass, G, w.gk[0], w.gv[0]);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<unsigned> dk(w.gk[0], w.gk[1]);
        cub::DoubleBuffer<int> dv(w.gv[0], w.gv[1]);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, b, dk, dv, static_cast<int>(F), 0, bits_for(ncell + 1), st));
        cell_start_kernel<<<blocks(ncell + 1), UW_THREADS, 0, st>>>(dk.Current(), F, ncell, w.cstart);
        TPX_LAUNCH_CHECK();
        TPX_CUDA(cudaMemsetAsync(w.flag, 0, F * sizeof(int), st));
        overlap_kernel<<<blocks(F), UW_THREADS, 0, st>>>(dk.Current(), dv.Current(), F, pass, G, w.cstart, w.cu, w.cvv, w.rad, w.uvr, verts_dev, w.T, w.flag);
        TPX_LAUNCH_CHECK();
        shift_kernel<<<blocks(F), UW_THREADS, 0, st>>>(w.flag, F, w.assign);
        TPX_LAUNCH_CHECK();
    }
    // stage 5
    slot_minmax_kernel<<<blocks(F), UW_THREADS, 0, st>>>(w.assign, w.uvr, F, w.hdr, w.is12);
    TPX_LAUNCH_CHECK();
    {
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceScan::ExclusiveSum(w.cub, b, w.is12, w.pos12, static_cast<int>(F), st));
    }
    PlaceConsts pc;
    pc.pad = island_padding;
    pc.pad_mul = static_cast<float>(1.0 - 2.0 * island_padding);
    pc.pad_add = static_cast<float>(island_padding);
    pc.fin_mul = static_cast<float>(1.0 - 2.0 * island_padding * 0.5);
    pc.fin_add = static_cast<float>(island_padding * 0.5);
    place_kernel<<<blocks(F), UW_THREADS, 0, st>>>(w.assign, w.uvr, w.is12, w.pos12, F, w.hdr, pc, w.placed, w.uk[0], w.uvv[0]);
    TPX_LAUNCH_CHECK();
    // stage 6
    {
        cub::DoubleBuffer<u64> dk(w.uk[0], w.uk[1]);
        cub::DoubleBuffer<int> dv(w.uvv[0], w.uvv[1]);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, b, dk, dv, static_cast<int>(n3), 0, 64, st));
        head_kernel<<<blocks(n3), UW_THREADS, 0, st>>>(dk.Current(), n3, w.head);
        TPX_LAUNCH_CHECK();
        b = w.cub_bytes;
        TPX_CUDA(cub::DeviceScan::InclusiveSum(w.cub, b, w.head, w.hscan, static_cast<int>(n3), st));
        unique_kernel<<<blocks(n3), UW_THREADS, 0, st>>>(dk.Current(), dv.Current(), w.head, w.hscan, n3, w.inv, w.ukey);
        TPX_LAUNCH_CHECK();
        unique_count_kernel<<<1, 1, 0, st>>>(w.hscan, n3, w.hdr);
        TPX_LAUNCH_CHECK();
    }
    TPX_CUDA(cudaMemcpyAsync(count_dev, &w.hdr->U, sizeof(long long), cudaMemcpyDeviceToDevice, st));
    if (taps_host) {
        const void* src[UW_NTAPS] = {w.slice, w.uv, w.hdr->angle, w.uvr, w.assign, w.placed};
        const size_t bytes[UW_NTAPS] = {F * sizeof(int), 6 * F * sizeof(float), 6 * sizeof(float), 6 * F * sizeof(float), F * sizeof(int), 6 * F * sizeof(float)};
        for (int t = 0; t < UW_NTAPS; ++t)
            if (taps_host[t]) TPX_CUDA(cudaMemcpyAsync(taps_host[t], src[t], bytes[t], cudaMemcpyDeviceToDevice, st));
    }
    return TPX_OK;
}

int tpx_uv_unwrap_emit(int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* uv_dev, int64_t* vtex_idx_dev, void* stream) {
    if (int rc = uw_check(V, F)) return rc;
    TPX_CHECK(uv_dev && vtex_idx_dev, TPX_ERR_ARG, "tpx_uv_unwrap_emit: null pointer");
    TPX_DEVICE_GUARD();
    Ws w;
    if (int rc = uw_setup(const_cast<void*>(ws), ws_bytes, V, F, &w)) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    emit_kernel<<<blocks(3 * F), UW_THREADS, 0, st>>>(w.ukey, w.inv, 3 * F, w.hdr, uv_dev, reinterpret_cast<long long*>(vtex_idx_dev));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_prim_noise_filter(const float* srt_dev, int K, uint8_t* keep_dev, int32_t* nn_dev, void* stream) {
    TPX_CHECK(K >= 1 && srt_dev && keep_dev, TPX_ERR_ARG, "tpx_prim_noise_filter: need K >= 1 (K=%d) and non-null srt / keep", K);
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    noise_filter_kernel<<<(K + NF_THREADS - 1) / NF_THREADS, NF_THREADS, 0, st>>>(srt_dev, K, keep_dev, nn_dev);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // extern "C"

}  // namespace tpx
