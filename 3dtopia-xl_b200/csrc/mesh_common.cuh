// Pieces shared by the mesh clean-up / decimation (mesh_simplify.cu) and the isotropic remesher (mesh_remesh.cu): face input and
// output kernels, corner keys and the vertex CSR, the frozen-vertex state, the star flip test, the two-ring minimum acceptance, face remap / compaction, the host-side argument checks and the CUB helpers.  Everything sits in an anonymous
// namespace, so each translation unit that includes this gets its own copy; both are compiled with -fmad=false (build.py).
#pragma once
#include <cub/cub.cuh>

#include "kernels.cuh"

namespace tpx {

namespace {
typedef unsigned long long u64;
constexpr int MS_THREADS = 256;
constexpr long long MS_INDEX_LIMIT = 1LL << 31;
constexpr u64 KEY_NONE = ~0ull;
constexpr double SINGULAR_REL = 1e-10;

// CUB scratch: the onesweep radix sort needs a lookback table of a few bytes per key; the launch checks the real need against this
size_t cub_reserve(long long n3) { return align_up(static_cast<size_t>(n3) * 8 + (16u << 20), 256); }

unsigned blocks(long long n) { return static_cast<unsigned>((n + MS_THREADS - 1) / MS_THREADS); }
int key_bits(long long V) {
    int b = 1;
    while ((1LL << b) < V) ++b;
    return 32 + b;
}

// ------------------------------------------------------------------------------------------------------------ shared kernels
// int64 faces -> int32; bad counts faces with an index outside [0, V) or (unless allow_repeat) a repeated index
__global__ void __launch_bounds__(MS_THREADS) faces_in_kernel(const long long* __restrict__ fin, long long F, long long V, int* __restrict__ T, int* bad,
                                                              bool allow_repeat = false) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    const long long a = fin[3 * f], b = fin[3 * f + 1], c = fin[3 * f + 2];
    if (a < 0 || b < 0 || c < 0 || a >= V || b >= V || c >= V || (!allow_repeat && (a == b || b == c || c == a))) {
        atomicAdd(bad, 1);
        T[3 * f] = T[3 * f + 1] = T[3 * f + 2] = 0;
        return;
    }
    T[3 * f] = static_cast<int>(a);
    T[3 * f + 1] = static_cast<int>(b);
    T[3 * f + 2] = static_cast<int>(c);
}

// half-edge keys (min << 32 | max) and, when val != nullptr, the face id of each
__global__ void __launch_bounds__(MS_THREADS) edge_keys_kernel(const int* __restrict__ T, long long F, u64* __restrict__ key, int* __restrict__ val) {
    const long long h = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (h >= 3 * F) return;
    const long long f = h / 3;
    const int k = static_cast<int>(h - 3 * f);
    const unsigned u = static_cast<unsigned>(T[3 * f + k]), v = static_cast<unsigned>(T[3 * f + (k + 1) % 3]);
    key[h] = (static_cast<u64>(min(u, v)) << 32) | max(u, v);
    if (val) val[h] = static_cast<int>(f);
}

// the vertices the first F faces use (flag memset to 0 before)
__global__ void __launch_bounds__(MS_THREADS) ref_kernel(const int* __restrict__ T, const int* __restrict__ fkeep, long long F, int* __restrict__ vref) {
    const long long h = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (h >= 3 * F) return;
    if (fkeep == nullptr || fkeep[h / 3]) vref[T[h]] = 1;
}

// counts[0..1] = V_out, F_out from exclusive scans and their last flags (-1, -1 when the input was malformed)
__global__ void counts_kernel(const int* vref, const int* vpos, long long V, const int* fkeep, const int* fpos, long long F, long long F_fixed, const int* bad,
                              long long* counts) {
    const bool malformed = bad != nullptr && *bad != 0;
    counts[0] = malformed ? -1 : (V ? static_cast<long long>(vpos[V - 1]) + vref[V - 1] : 0);
    counts[1] = malformed ? -1 : (fkeep == nullptr ? F_fixed : (F ? static_cast<long long>(fpos[F - 1]) + fkeep[F - 1] : 0));
}

__global__ void __launch_bounds__(MS_THREADS) emit_verts_kernel(const float* __restrict__ P, const int* __restrict__ vref, const int* __restrict__ vpos, long long V,
                                                                float* __restrict__ out) {
    const long long v = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (v >= V || !vref[v]) return;
    const long long o = vpos[v];
    out[3 * o] = P[3 * v];
    out[3 * o + 1] = P[3 * v + 1];
    out[3 * o + 2] = P[3 * v + 2];
}

__global__ void __launch_bounds__(MS_THREADS) emit_faces_kernel(const int* __restrict__ T, const int* __restrict__ fkeep, const int* __restrict__ fpos,
                                                                const long long* __restrict__ nF, long long F, const int* __restrict__ vpos, long long* __restrict__ out) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= (nF ? *nF : F)) return;
    if (fkeep && !fkeep[f]) return;
    const long long o = fpos ? fpos[f] : f;
#pragma unroll
    for (int k = 0; k < 3; ++k) out[3 * o + k] = vpos[T[3 * f + k]];
}

// fp32 <-> int32 with the same order (atomicMin / atomicMax keys of boxes)
__device__ __forceinline__ int ord_f32(float x) {
    const int b = __float_as_int(x);
    return b >= 0 ? b : b ^ 0x7fffffff;
}
__device__ __forceinline__ float unord_f32(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

struct DecHdr {
    long long F;          // live faces (in T[buf])
    long long E;          // edges of the round (DeviceSelect::Unique)
    long long n_sel;      // accepted keys selected for trimming
    u64 thr;              // largest key collapsed this round
    int buf;              // which face buffer is live
    int n_acc;            // accepted edges this round
    int bad;              // malformed input faces
};

__device__ __forceinline__ void cross3(const double* p0, const double* p1, const double* p2, double* n) {
    const double e1x = __dsub_rn(p1[0], p0[0]), e1y = __dsub_rn(p1[1], p0[1]), e1z = __dsub_rn(p1[2], p0[2]);
    const double e2x = __dsub_rn(p2[0], p0[0]), e2y = __dsub_rn(p2[1], p0[1]), e2z = __dsub_rn(p2[2], p0[2]);
    n[0] = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
    n[1] = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
    n[2] = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
}

__device__ __forceinline__ void load3(const float* P, int v, double* p) {
    p[0] = P[3 * v];
    p[1] = P[3 * v + 1];
    p[2] = P[3 * v + 2];
}

// corner i of vertex v: the face id (low half of the sorted corner key) and the next (out) / previous (in) vertex of that face
__device__ __forceinline__ int corner(const u64* ck, const int* T, int v, int i, int* out, int* in) {
    const int f = static_cast<int>(static_cast<unsigned>(ck[i]));
    const int* t = T + 3 * static_cast<long long>(f);
    const int k = t[0] == v ? 0 : (t[1] == v ? 1 : 2);
    *out = t[k == 2 ? 0 : k + 1];
    *in = t[k == 0 ? 2 : k - 1];
    return f;
}

__global__ void __launch_bounds__(MS_THREADS) corner_keys_kernel(const int* __restrict__ T, long long F, u64* __restrict__ ck) {
    const long long h = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (h >= 3 * F) return;
    ck[h] = (static_cast<u64>(static_cast<unsigned>(T[h])) << 32) | static_cast<u64>(h / 3);
}

// vertex CSR over the sorted corner keys: [vstart[v], vend[v]) (both memset to 0 first)
__global__ void __launch_bounds__(MS_THREADS) csr_kernel(const u64* __restrict__ ck, long long n, int* __restrict__ vstart, int* __restrict__ vend) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= n) return;
    const unsigned v = static_cast<unsigned>(ck[i] >> 32);
    if (i == 0 || static_cast<unsigned>(ck[i - 1] >> 32) != v) vstart[v] = static_cast<int>(i);
    if (i == n - 1 || static_cast<unsigned>(ck[i + 1] >> 32) != v) vend[v] = static_cast<int>(i + 1);
}

// frozen flag and degree (distinct neighbours) of every vertex
__global__ void __launch_bounds__(MS_THREADS) vertex_state_kernel(const int* __restrict__ T, const u64* __restrict__ ck, const int* __restrict__ vstart,
                                                                  const int* __restrict__ vend, long long V, uint8_t* __restrict__ frozen, int* __restrict__ deg) {
    const long long vv = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (vv >= V) return;
    const int v = static_cast<int>(vv), s = vstart[v], n = vend[v] - s;
    bool ok = n > 0;
    int distinct = 0;
    for (int i = 0; i < n; ++i) {
        int oi, ii;
        corner(ck, T, v, s + i, &oi, &ii);
        int c_oo = 0, c_oi = 0;
        bool new_o = true, new_i = true;
        for (int j = 0; j < n; ++j) {
            int oj, ij;
            corner(ck, T, v, s + j, &oj, &ij);
            c_oo += oj == oi;
            c_oi += ij == oi;
            if (j < i && (oj == oi || ij == oi)) new_o = false;       // out_i seen among earlier outs or ins
            if (j <= i && oj == ii) new_i = false;                    // in_i seen among outs up to i
            if (j < i && ij == ii) new_i = false;                     // ... or among earlier ins
        }
        distinct += new_o;
        distinct += new_i && ii != oi;
        ok = ok && c_oo == 1 && c_oi == 1;
    }
    if (ok) {                                                         // one fan: the walk out -> in returns to corner 0 after n steps
        int o0, cur;
        corner(ck, T, v, s, &o0, &cur);
        int steps = 1;
        while (cur != o0 && steps <= n) {
            int j = 0, oj, ij;
            for (; j < n; ++j) {
                corner(ck, T, v, s + j, &oj, &ij);
                if (oj == cur) break;
            }
            cur = ij;
            ++steps;
        }
        ok = steps == n;
    }
    frozen[v] = !ok;
    deg[v] = distinct;
}

// no face of v's star but those containing `other` turns by 90 degrees or more when v moves to x (faces with a zero normal exempt)
__device__ __forceinline__ bool star_ok(const float* P, const int* T, const u64* ck, int s, int n, int v, int other, const float* x) {
    for (int i = 0; i < n; ++i) {
        const int* t = T + 3 * static_cast<long long>(static_cast<unsigned>(ck[s + i]));
        if (t[0] == other || t[1] == other || t[2] == other) continue;
        double p[3][3], m[3][3], no[3], nn[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            load3(P, t[k], p[k]);
#pragma unroll
            for (int d = 0; d < 3; ++d) m[k][d] = t[k] == v ? static_cast<double>(x[d]) : p[k][d];
        }
        cross3(p[0], p[1], p[2], no);
        if (no[0] == 0.0 && no[1] == 0.0 && no[2] == 0.0) continue;
        cross3(m[0], m[1], m[2], nn);
        if (!(__dadd_rn(__dadd_rn(__dmul_rn(no[0], nn[0]), __dmul_rn(no[1], nn[1])), __dmul_rn(no[2], nn[2])) > 0.0)) return false;
    }
    return true;
}

// m2 = m1 (copied before); m2[v] = min over v's neighbours of m1 too
__global__ void __launch_bounds__(MS_THREADS) edge_min2_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, const u64* __restrict__ m1, u64* m2) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E) return;
    const u64 ed = edges[e];
    const int a = static_cast<int>(ed >> 32), b = static_cast<int>(static_cast<unsigned>(ed));
    if (m1[b] != KEY_NONE) atomicMin(m2 + a, m1[b]);
    if (m1[a] != KEY_NONE) atomicMin(m2 + b, m1[a]);
}

__global__ void __launch_bounds__(MS_THREADS) edge_accept_kernel(const u64* __restrict__ edges, DecHdr* hdr, const u64* __restrict__ ekey, const u64* __restrict__ m2,
                                                                 int* __restrict__ aflag) {
    __shared__ int s_warp[MS_THREADS / 32];
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    int acc = 0;
    if (e < hdr->E) {
        const u64 ed = edges[e], key = ekey[e];
        const int a = static_cast<int>(ed >> 32), b = static_cast<int>(static_cast<unsigned>(ed));
        acc = key != KEY_NONE && m2[a] == key && m2[b] == key;
        aflag[e] = acc;
    }
    const int w = __popc(__ballot_sync(0xffffffffu, acc));
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int i = 0; i < MS_THREADS / 32; ++i) t += s_warp[i];
        if (t) atomicAdd(&hdr->n_acc, t);
    }
}

__global__ void __launch_bounds__(MS_THREADS) remap_kernel(int* __restrict__ T, long long F, const int* __restrict__ rep, int* __restrict__ fkeep) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int a = rep[T[3 * f]], b = rep[T[3 * f + 1]], c = rep[T[3 * f + 2]];
    T[3 * f] = a;
    T[3 * f + 1] = b;
    T[3 * f + 2] = c;
    fkeep[f] = a != b && b != c && c != a;
}

__global__ void __launch_bounds__(MS_THREADS) compact_faces_kernel(const int* __restrict__ T, long long F, const int* __restrict__ fkeep, const int* __restrict__ fpos,
                                                                   int* __restrict__ Tout, DecHdr* hdr, int buf) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f == 0) {
        hdr->F = F ? static_cast<long long>(fpos[F - 1]) + fkeep[F - 1] : 0;
        hdr->buf = buf;
    }
    if (f >= F || !fkeep[f]) return;
    const long long o = fpos[f];
    Tout[3 * o] = T[3 * f];
    Tout[3 * o + 1] = T[3 * f + 1];
    Tout[3 * o + 2] = T[3 * f + 2];
}

// the host-side argument checks of every mesh entry point
int mesh_args(const char* what, const float* verts, long long V, const long long* faces, long long F, void* ws, size_t ws_bytes, size_t need) {
    TPX_CHECK(V >= 0 && F >= 0 && V < MS_INDEX_LIMIT && F < MS_INDEX_LIMIT, TPX_ERR_SHAPE, "%s: %lld vertices / %lld faces: each must be below 2^31", what, V, F);
    TPX_CHECK((verts != nullptr || V == 0) && (faces != nullptr || F == 0) && ws != nullptr, TPX_ERR_ARG, "%s: null mesh or workspace", what);
    TPX_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, TPX_ERR_ARG, "%s: workspace must be 256-B aligned", what);
    TPX_CHECK(V > 0 || F == 0, TPX_ERR_ARG, "%s: %lld faces index an empty vertex array", what, F);
    TPX_CHECK(ws_bytes >= need, TPX_ERR_ARG, "%s: workspace of %zu bytes, %zu needed", what, ws_bytes, need);
    return TPX_OK;
}

// scan of n int flags into pos (exclusive)
int scan(const int* flags, int* pos, long long n, void* cub, size_t cub_bytes, cudaStream_t st) {
    if (n == 0) return TPX_OK;
    size_t b = cub_bytes;
    TPX_CUDA(cub::DeviceScan::ExclusiveSum(cub, b, flags, pos, n, st));
    return TPX_OK;
}

int sort_pairs(u64* k0, u64* k1, int* v0, int* v1, long long n, int bits, void* cub, size_t cub_bytes, cudaStream_t st, const u64** ko, const int** vo) {
    cub::DoubleBuffer<u64> dk(k0, k1);
    cub::DoubleBuffer<int> dv(v0, v1);
    if (n) {
        size_t b = cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortPairs(cub, b, dk, dv, n, 0, bits, st));
    }
    *ko = dk.Current();
    *vo = dv.Current();
    return TPX_OK;
}
}  // namespace

}  // namespace tpx
