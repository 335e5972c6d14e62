// Mesh clean-up and decimation (DESIGN.md §1 f-7): the GPU stand-in for the pymeshlab calls extract_texmesh makes between marching
// cubes and the unwrap (inference.py:126-129, utils/meshutils.py:63-193):
//   * remove_small_components — clean_mesh's remove_connected_component_by_face_number(min_f) / ..._by_diameter(min_d):
//     (a) faces -> int32, index checks; half-edge keys (min << 32 | max, face) sorted; (b) union-find over faces that share a key,
//     always hooking the larger root under the smaller, so each root is its component's smallest face id whatever the schedule;
//     (c) per-root face count and box (atomicMin / atomicMax on order-preserving ints), whole-mesh box; (d) keep flags, scans.
//   * decimate — quadric edge collapse in rounds of independent collapses; every round: corner keys (vertex << 32 | face) and
//     half-edge keys sorted, vertex CSR, frozen flags and degrees, edge list (unique keys), per-edge cost / placement / validity,
//     two minimum passes, accept, (last round) trim to the smallest keys, collapse, remap, stable face compaction.  The host reads
//     the accepted count back once per round.
// Every output position comes from a sort or a prefix sum, and every atomic is a min, max or count, so results are identical across
// calls and streams.  This file is compiled with -fmad=false (build.py) and spells its fp64 arithmetic with explicit _rn intrinsics: it
// is the numpy test oracle's (decimate.py) operation for operation, and a contracted product would change its last bits.
#include "mesh_common.cuh"

namespace tpx {

namespace {

// ------------------------------------------------------------------------------------------------------------ component filter
// root of x; parent[y] <= y always, path halving on the way (races only ever store an ancestor)
__device__ __forceinline__ int find_root(volatile int* parent, int x) {
    int cur = parent[x];
    if (cur != x) {
        int next, prev = x;
        while (cur > (next = parent[cur])) {
            parent[prev] = next;
            prev = cur;
            cur = next;
        }
    }
    return cur;
}

__global__ void __launch_bounds__(MS_THREADS) cc_init_kernel(long long F, int* __restrict__ parent, int* __restrict__ cnt, int* __restrict__ bmin,
                                                             int* __restrict__ bmax) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    parent[f] = static_cast<int>(f);
    cnt[f] = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) { bmin[3 * f + d] = INT_MAX; bmax[3 * f + d] = INT_MIN; }
}

// union of the faces of consecutive equal sorted keys: hook the larger root under the smaller with a CAS, retry on a lost race
__global__ void __launch_bounds__(MS_THREADS) cc_union_kernel(const u64* __restrict__ key, const int* __restrict__ val, long long n, int* parent) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i + 1 >= n || key[i] != key[i + 1]) return;
    volatile int* p = parent;
    int ra = find_root(p, val[i]), rb = find_root(p, val[i + 1]);
    while (ra != rb) {
        if (ra > rb) { const int t = ra; ra = rb; rb = t; }
        const int old = atomicCAS(parent + rb, rb, ra);
        if (old == rb) break;
        ra = find_root(p, ra);
        rb = find_root(p, old);
    }
}

// every face's root, its component's face count and box, and the box of all referenced vertices (warp-reduced first)
__global__ void __launch_bounds__(MS_THREADS) cc_stats_kernel(const int* __restrict__ T, const float* __restrict__ P, long long F, int* parent, int* __restrict__ cnt,
                                                              int* __restrict__ bmin, int* __restrict__ bmax, int* __restrict__ gbox) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    if (f < F) {
        volatile int* p = parent;
        int r = static_cast<int>(f);
        while (p[r] != r) r = p[r];
        p[f] = r;
        atomicAdd(cnt + r, 1);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float* v = P + 3 * static_cast<long long>(T[3 * f + k]);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const int o = ord_f32(v[d]);
                lo[d] = min(lo[d], o);
                hi[d] = max(hi[d], o);
            }
        }
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            atomicMin(bmin + 3 * r + d, lo[d]);
            atomicMax(bmax + 3 * r + d, hi[d]);
        }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = min(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
            hi[d] = max(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            atomicMin(gbox + d, lo[d]);
            atomicMax(gbox + 3 + d, hi[d]);
        }
    }
}

__device__ __forceinline__ double box_diag(const int* lo, const int* hi) {
    const double dx = __dsub_rn(static_cast<double>(unord_f32(hi[0])), static_cast<double>(unord_f32(lo[0])));
    const double dy = __dsub_rn(static_cast<double>(unord_f32(hi[1])), static_cast<double>(unord_f32(lo[1])));
    const double dz = __dsub_rn(static_cast<double>(unord_f32(hi[2])), static_cast<double>(unord_f32(lo[2])));
    return sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

__global__ void __launch_bounds__(MS_THREADS) cc_keep_kernel(const int* __restrict__ parent, const int* __restrict__ cnt, const int* __restrict__ bmin,
                                                             const int* __restrict__ bmax, const int* __restrict__ gbox, long long F, long long min_faces,
                                                             double min_diameter, int* __restrict__ fkeep) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int r = parent[f];
    const double lim = __dmul_rn(min_diameter, box_diag(gbox, gbox + 3));
    fkeep[f] = cnt[r] >= min_faces && !(box_diag(bmin + 3 * r, bmax + 3 * r) < lim);
}

// ------------------------------------------------------------------------------------------------------------ decimation
// x^T Q x at (x, y, z, 1), clamped below at 0
__device__ __forceinline__ double quadric_cost(const double* q, double x, double y, double z) {
    const double r0 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], x), __dmul_rn(q[1], y)), __dmul_rn(q[2], z)), q[3]);
    const double r1 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[1], x), __dmul_rn(q[4], y)), __dmul_rn(q[5], z)), q[6]);
    const double r2 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[2], x), __dmul_rn(q[5], y)), __dmul_rn(q[7], z)), q[8]);
    const double r3 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[3], x), __dmul_rn(q[6], y)), __dmul_rn(q[8], z)), q[9]);
    const double c = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r0, x), __dmul_rn(r1, y)), __dmul_rn(r2, z)), r3);
    return c > 0.0 ? c : 0.0;
}

__device__ __forceinline__ double cost_at(const double* q, const float* x) { return quadric_cost(q, x[0], x[1], x[2]); }

// placement x̄ (fp32) of the summed quadric q and its cost
__device__ __forceinline__ double placement(const double* q, const float* pa, const float* pb, float* x) {
    const double c00 = __dsub_rn(__dmul_rn(q[4], q[7]), __dmul_rn(q[5], q[5]));
    const double c01 = __dsub_rn(__dmul_rn(q[2], q[5]), __dmul_rn(q[1], q[7]));
    const double c02 = __dsub_rn(__dmul_rn(q[1], q[5]), __dmul_rn(q[2], q[4]));
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(q[0], c00), __dmul_rn(q[1], c01)), __dmul_rn(q[2], c02));
    const double tr = __dadd_rn(__dadd_rn(q[0], q[4]), q[7]);
    bool solved = fabs(det) > __dmul_rn(SINGULAR_REL, __dmul_rn(__dmul_rn(tr, tr), tr));
    if (solved) {
        const double c11 = __dsub_rn(__dmul_rn(q[0], q[7]), __dmul_rn(q[2], q[2]));
        const double c12 = __dsub_rn(__dmul_rn(q[1], q[2]), __dmul_rn(q[0], q[5]));
        const double c22 = __dsub_rn(__dmul_rn(q[0], q[4]), __dmul_rn(q[1], q[1]));
        const double b0 = -q[3], b1 = -q[6], b2 = -q[8];
        x[0] = __double2float_rn(__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(c00, b0), __dmul_rn(c01, b1)), __dmul_rn(c02, b2)), det));
        x[1] = __double2float_rn(__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(c01, b0), __dmul_rn(c11, b1)), __dmul_rn(c12, b2)), det));
        x[2] = __double2float_rn(__ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(c02, b0), __dmul_rn(c12, b1)), __dmul_rn(c22, b2)), det));
        solved = isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]);
    }
    if (solved) return cost_at(q, x);
#pragma unroll
    for (int d = 0; d < 3; ++d) x[d] = __double2float_rn(__dmul_rn(__dadd_rn(static_cast<double>(pa[d]), static_cast<double>(pb[d])), 0.5));
    double best = cost_at(q, x);
    const double ca = cost_at(q, pa);
    if (ca < best) { best = ca; x[0] = pa[0]; x[1] = pa[1]; x[2] = pa[2]; }
    const double cb = cost_at(q, pb);
    if (cb < best) { best = cb; x[0] = pb[0]; x[1] = pb[1]; x[2] = pb[2]; }
    return best;
}

// Q_v = sum over v's faces in ascending face index (the corner list order) of the area-weighted plane quadric
__global__ void __launch_bounds__(MS_THREADS) quadric_kernel(const float* __restrict__ P, const int* __restrict__ T, const u64* __restrict__ ck,
                                                             const int* __restrict__ vstart, const int* __restrict__ vend, long long V, double* __restrict__ Q) {
    const long long v = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (v >= V) return;
    double acc[10];
#pragma unroll
    for (int k = 0; k < 10; ++k) acc[k] = 0.0;
    for (int i = vstart[v]; i < vend[v]; ++i) {
        const int* t = T + 3 * static_cast<long long>(static_cast<unsigned>(ck[i]));
        double p0[3], p1[3], p2[3], c[3];
        load3(P, t[0], p0);
        load3(P, t[1], p1);
        load3(P, t[2], p2);
        cross3(p0, p1, p2, c);
        const double ln = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(c[0], c[0]), __dmul_rn(c[1], c[1])), __dmul_rn(c[2], c[2])));
        if (ln == 0.0) continue;
        const double area = __dmul_rn(0.5, ln);
        double u[4];
        u[0] = __ddiv_rn(c[0], ln);
        u[1] = __ddiv_rn(c[1], ln);
        u[2] = __ddiv_rn(c[2], ln);
        u[3] = -__dadd_rn(__dadd_rn(__dmul_rn(u[0], p0[0]), __dmul_rn(u[1], p0[1])), __dmul_rn(u[2], p0[2]));
        int k = 0;
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = a; b < 4; ++b) acc[k] = __dadd_rn(acc[k], __dmul_rn(area, __dmul_rn(u[a], u[b]))), ++k;
    }
#pragma unroll
    for (int k = 0; k < 10; ++k) Q[10 * v + k] = acc[k];
}

// one edge per thread; min-blocks 1 lets ptxas keep the fp64 solve and flip test in registers (it spills under the default bound)
__global__ void __launch_bounds__(MS_THREADS, 1) edge_cost_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, const float* __restrict__ P,
                                                               const double* __restrict__ Q, const int* __restrict__ T, const u64* __restrict__ ck,
                                                               const int* __restrict__ vstart, const int* __restrict__ vend, const uint8_t* __restrict__ frozen,
                                                               const int* __restrict__ deg, u64* __restrict__ ekey, float* __restrict__ xbar, u64* m1) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E) return;
    const u64 ed = edges[e];
    const int a = static_cast<int>(ed >> 32), b = static_cast<int>(static_cast<unsigned>(ed));
    u64 key = KEY_NONE;
    if (!frozen[a] && !frozen[b]) {
        const int sa = vstart[a], na = vend[a] - sa, sb = vstart[b], nb = vend[b] - sb;
        int c = -1, d = -1, link = 0;
        for (int i = 0; i < na; ++i) {
            int oa, ia;
            corner(ck, T, a, sa + i, &oa, &ia);
            if (oa == b) c = ia;
            if (ia == b) d = oa;
            for (int j = 0; j < nb; ++j) {
                int ob, ib;
                corner(ck, T, b, sb + j, &ob, &ib);
                link += oa == ob;
            }
        }
        bool ok = link == 2 && c >= 0 && d >= 0 && c != d && deg[a] + deg[b] >= 7 && deg[c] >= 4 && deg[d] >= 4;
        if (ok) {
            double q[10];
#pragma unroll
            for (int k = 0; k < 10; ++k) q[k] = __dadd_rn(Q[10LL * a + k], Q[10LL * b + k]);
            const float pa[3] = {P[3LL * a], P[3LL * a + 1], P[3LL * a + 2]}, pb[3] = {P[3LL * b], P[3LL * b + 1], P[3LL * b + 2]};
            float x[3];
            const double cost = placement(q, pa, pb, x);
            ok = star_ok(P, T, ck, sa, na, a, b, x) && star_ok(P, T, ck, sb, nb, b, a, x);
            if (ok) {
                key = (static_cast<u64>(__float_as_uint(__double2float_rn(cost))) << 32) | static_cast<u64>(e);
                xbar[3 * e] = x[0];
                xbar[3 * e + 1] = x[1];
                xbar[3 * e + 2] = x[2];
                atomicMin(m1 + a, key);
                atomicMin(m1 + b, key);
            }
        }
    }
    ekey[e] = key;
}

// the largest key collapsed this round: the k-th smallest accepted key when trimming (sorted != nullptr), else every accepted key
__global__ void set_thr_kernel(DecHdr* hdr, const u64* sorted, long long k) { hdr->thr = sorted ? sorted[k - 1] : KEY_NONE - 1; }

__global__ void __launch_bounds__(MS_THREADS) collapse_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, const u64* __restrict__ ekey,
                                                              const int* __restrict__ aflag, const float* __restrict__ xbar, float* __restrict__ P, double* __restrict__ Q,
                                                              int* __restrict__ rep) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E || !aflag[e] || ekey[e] > hdr->thr) return;
    const u64 ed = edges[e];
    const long long a = static_cast<long long>(ed >> 32), b = static_cast<long long>(static_cast<unsigned>(ed));
    P[3 * a] = xbar[3 * e];
    P[3 * a + 1] = xbar[3 * e + 1];
    P[3 * a + 2] = xbar[3 * e + 2];
#pragma unroll
    for (int k = 0; k < 10; ++k) Q[10 * a + k] = __dadd_rn(Q[10 * a + k], Q[10 * b + k]);
    rep[b] = static_cast<int>(a);
}

__global__ void __launch_bounds__(MS_THREADS) iota_copy_kernel(const float* __restrict__ verts, long long V, float* __restrict__ P, int* __restrict__ rep) {
    const long long v = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (v >= V) return;
    P[3 * v] = verts[3 * v];
    P[3 * v + 1] = verts[3 * v + 1];
    P[3 * v + 2] = verts[3 * v + 2];
    rep[v] = static_cast<int>(v);
}

// ------------------------------------------------------------------------------------------------------------ workspaces
struct CcWs {
    int* bad;
    int* gbox;
    int* T;
    u64* key[2];
    int* val[2];
    int *parent, *cnt, *bmin, *bmax, *fkeep, *fpos, *vref, *vpos;
    void* cub;
    size_t cub_bytes, total;
};

CcWs cc_layout(void* ws, long long V, long long F) {
    Carve c{static_cast<uint8_t*>(ws)};
    CcWs w;
    w.bad = c.take<int>(1);
    w.gbox = c.take<int>(6);
    w.T = c.take<int>(3 * F);
    w.key[0] = c.take<u64>(3 * F);
    w.key[1] = c.take<u64>(3 * F);
    w.val[0] = c.take<int>(3 * F);
    w.val[1] = c.take<int>(3 * F);
    w.parent = c.take<int>(F);
    w.cnt = c.take<int>(F);
    w.bmin = c.take<int>(3 * F);
    w.bmax = c.take<int>(3 * F);
    w.fkeep = c.take<int>(F);
    w.fpos = c.take<int>(F);
    w.vref = c.take<int>(V);
    w.vpos = c.take<int>(V);
    w.cub_bytes = cub_reserve(3 * F);
    w.cub = c.take<uint8_t>(static_cast<long long>(w.cub_bytes));
    w.total = c.off;
    return w;
}

struct DecWs {
    DecHdr* hdr;
    float* P;
    double* Q;
    int *rep, *vstart, *vend, *deg;
    uint8_t* frozen;
    u64 *m1, *m2;
    int* T[2];
    u64* ck[2];
    u64* hk[2];
    u64* ekey;
    float* xbar;
    int *aflag, *fkeep, *fpos, *vref, *vpos;
    void* cub;
    size_t cub_bytes, total;
};

DecWs dec_layout(void* ws, long long V, long long F) {
    Carve c{static_cast<uint8_t*>(ws)};
    DecWs w;
    w.hdr = c.take<DecHdr>(1);
    w.P = c.take<float>(3 * V);
    w.Q = c.take<double>(10 * V);
    w.rep = c.take<int>(V);
    w.vstart = c.take<int>(V);
    w.vend = c.take<int>(V);
    w.deg = c.take<int>(V);
    w.frozen = c.take<uint8_t>(V);
    w.m1 = c.take<u64>(V);
    w.m2 = c.take<u64>(V);
    w.vref = c.take<int>(V);
    w.vpos = c.take<int>(V);
    w.T[0] = c.take<int>(3 * F);
    w.T[1] = c.take<int>(3 * F);
    w.ck[0] = c.take<u64>(3 * F);
    w.ck[1] = c.take<u64>(3 * F);
    w.hk[0] = c.take<u64>(3 * F);
    w.hk[1] = c.take<u64>(3 * F);
    w.ekey = c.take<u64>(3 * F);
    w.xbar = c.take<float>(9 * F);
    w.aflag = c.take<int>(3 * F);
    w.fkeep = c.take<int>(F);
    w.fpos = c.take<int>(F);
    w.cub_bytes = cub_reserve(3 * F);
    w.cub = c.take<uint8_t>(static_cast<long long>(w.cub_bytes));
    w.total = c.off;
    return w;
}

// the largest CUB scratch either operation asks for at these sizes (host-side queries, no launch)
int cub_need(long long V, long long F, size_t* need) {
    size_t b = 0, m = 0;
    const long long n3 = 3 * F;
    cub::DoubleBuffer<u64> dk(nullptr, nullptr);
    cub::DoubleBuffer<int> dv(nullptr, nullptr);
    TPX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, dk, dv, n3, 0, 64));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b, dk, n3, 0, 64));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceSelect::Unique(nullptr, b, static_cast<const u64*>(nullptr), static_cast<u64*>(nullptr), static_cast<long long*>(nullptr), n3));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceSelect::Flagged(nullptr, b, static_cast<const u64*>(nullptr), static_cast<const int*>(nullptr), static_cast<u64*>(nullptr),
                                        static_cast<long long*>(nullptr), n3));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const int*>(nullptr), static_cast<int*>(nullptr), F > V ? F : V));
    m = b > m ? b : m;
    *need = m;
    return TPX_OK;
}

int mesh_check(const char* what, const float* verts, long long V, const long long* faces, long long F, void* ws, size_t ws_bytes, size_t need, long long Vf,
               long long Ff) {
    const int ra = mesh_args(what, verts, V, faces, F, ws, ws_bytes, need);
    if (ra != TPX_OK) return ra;
    size_t cub_bytes;
    const int rc = cub_need(Vf, Ff, &cub_bytes);
    if (rc != TPX_OK) return rc;
    TPX_CHECK(cub_bytes <= cub_reserve(3 * Ff), TPX_ERR_STATE, "%s: sort scratch of %zu bytes exceeds the %zu reserved", what, cub_bytes, cub_reserve(3 * Ff));
    return TPX_OK;
}

// ------------------------------------------------------------------------------------------------------------ clean-up: weld
// clean_mesh's merge_close_vertices / remove_duplicate_faces / remove_null_faces (DESIGN.md §1 "clean-up contract").  The greedy
// merge is resolved in rounds over cells of side h >= r: a referenced vertex decides once every earlier vertex within r has decided.
constexpr int WELD_BATCH = 8;               // rounds launched between two readbacks of the undecided counts
constexpr int CELL_BITS = 21;               // per axis; cells are widened so that no axis needs more
constexpr u64 CELL_NONE = ~0ull;

struct WeldHdr {
    double r2;                  // (merge fraction x box diagonal)^2; no merge unless > 0
    double lo[3];               // box corner the cells start at
    double inv_h;               // 1 / cell side
    int merge;
    int nC;                     // occupied cells
    int bad;                    // faces with an index outside [0, V)
    int und[WELD_BATCH];        // undecided vertices after each round of the batch
};

// box of the referenced vertices (order-preserving ints; warp-reduced first)
__global__ void __launch_bounds__(MS_THREADS) ref_box_kernel(const float* __restrict__ P, const int* __restrict__ vref, long long V, int* __restrict__ gbox) {
    const long long v = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    if (v < V && vref[v]) {
#pragma unroll
        for (int d = 0; d < 3; ++d) lo[d] = hi[d] = ord_f32(P[3 * v + d]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo[d] = min(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
            hi[d] = max(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
        }
    }
    if ((threadIdx.x & 31) == 0 && lo[0] != INT_MAX) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            atomicMin(gbox + d, lo[d]);
            atomicMax(gbox + 3 + d, hi[d]);
        }
    }
}

// r = frac x diagonal (the component filter's box_diag); cells of side max(r, extent / 2^20) widened by 2^-10, so that two points
// within r always lie in the same or adjacent cells whatever the rounding of the cell coordinates
__global__ void weld_params_kernel(const int* gbox, double frac, WeldHdr* hdr) {
    hdr->merge = 0;
    if (gbox[0] > gbox[3] || !(frac > 0.0)) return;
    const double r = __dmul_rn(frac, box_diag(gbox, gbox + 3));
    double ext = 0.0;
    for (int d = 0; d < 3; ++d) {
        hdr->lo[d] = static_cast<double>(unord_f32(gbox[d]));
        ext = fmax(ext, static_cast<double>(unord_f32(gbox[3 + d])) - hdr->lo[d]);
    }
    if (!(r > 0.0) || !isfinite(r) || !isfinite(ext)) return;
    hdr->r2 = __dmul_rn(r, r);
    hdr->inv_h = 1.0 / (fmax(r, ext * (1.0 / (1 << (CELL_BITS - 1)))) * (1.0 + 1.0 / 1024));
    hdr->merge = hdr->r2 > 0.0;
}

__device__ __forceinline__ long long cell_coord(float x, double lo, double inv_h) {
    const double c = floor((static_cast<double>(x) - lo) * inv_h);
    return c < 0.0 ? 0 : (c > double((1 << CELL_BITS) - 1) ? (1 << CELL_BITS) - 1 : static_cast<long long>(c));
}

// cell key of every referenced vertex (CELL_NONE otherwise, sorted last) and the initial state: -1 undecided, else the vertex's
// representative (itself when nothing merges)
__global__ void __launch_bounds__(MS_THREADS) weld_keys_kernel(const float* __restrict__ P, const int* __restrict__ vref, long long V, const WeldHdr* __restrict__ hdr,
                                                               u64* __restrict__ key, int* __restrict__ val, int* __restrict__ state) {
    const long long v = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (v >= V) return;
    const bool live = hdr->merge && vref[v];
    u64 k = CELL_NONE;
    if (live) {
        k = 0;
#pragma unroll
        for (int d = 0; d < 3; ++d) k = (k << CELL_BITS) | static_cast<u64>(cell_coord(P[3 * v + d], hdr->lo[d], hdr->inv_h));
    }
    key[v] = k;
    val[v] = static_cast<int>(v);
    state[v] = live ? -1 : static_cast<int>(v);
}

// first flags of the sorted cell keys (the sentinel run is no cell), and the vertices' positions in sorted order
__global__ void __launch_bounds__(MS_THREADS) cell_flags_kernel(const u64* __restrict__ sk, const int* __restrict__ sv, const float* __restrict__ P, long long V,
                                                                int* __restrict__ flag, float* __restrict__ Ps) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= V) return;
    flag[i] = sk[i] != CELL_NONE && (i == 0 || sk[i] != sk[i - 1]);
    if (sk[i] == CELL_NONE) return;
    const long long v = sv[i];
    Ps[3 * i] = P[3 * v];
    Ps[3 * i + 1] = P[3 * v + 1];
    Ps[3 * i + 2] = P[3 * v + 2];
}

// per sorted position its cell; per cell its key and [start, end) in sorted order; hdr->nC
__global__ void __launch_bounds__(MS_THREADS) cell_ranges_kernel(const u64* __restrict__ sk, const int* __restrict__ flag, const int* __restrict__ excl, long long V,
                                                                 int* __restrict__ cellof, u64* __restrict__ ukey, int* __restrict__ cstart, int* __restrict__ cend,
                                                                 WeldHdr* hdr) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= V || sk[i] == CELL_NONE) return;
    const int c = excl[i] + flag[i] - 1;
    cellof[i] = c;
    if (flag[i]) {
        cstart[c] = static_cast<int>(i);
        ukey[c] = sk[i];
    }
    if (i == V - 1 || sk[i + 1] != sk[i]) {
        cend[c] = static_cast<int>(i + 1);
        if (i == V - 1 || sk[i + 1] == CELL_NONE) hdr->nC = c + 1;
    }
}

// the 27 neighbour cells of every occupied cell (-1 where empty), by binary search over the sorted cell keys
__global__ void __launch_bounds__(MS_THREADS) cell_nb_kernel(const u64* __restrict__ ukey, const WeldHdr* __restrict__ hdr, int* __restrict__ nb) {
    const long long c = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    const int nC = hdr->nC;
    if (c >= nC) return;
    const u64 k = ukey[c], m = (1ull << CELL_BITS) - 1;
    const long long x = static_cast<long long>(k >> (2 * CELL_BITS)), y = static_cast<long long>((k >> CELL_BITS) & m), z = static_cast<long long>(k & m);
    int j = 0;
    for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dz = -1; dz <= 1; ++dz, ++j) {
                const long long a = x + dx, b = y + dy, e = z + dz;
                int found = -1;
                if (a >= 0 && b >= 0 && e >= 0 && a <= static_cast<long long>(m) && b <= static_cast<long long>(m) && e <= static_cast<long long>(m)) {
                    const u64 q = (static_cast<u64>(a) << (2 * CELL_BITS)) | (static_cast<u64>(b) << CELL_BITS) | static_cast<u64>(e);
                    int lo = 0, hi = nC;
                    while (lo < hi) {
                        const int mid = (lo + hi) >> 1;
                        if (ukey[mid] < q) lo = mid + 1; else hi = mid;
                    }
                    if (lo < nC && ukey[lo] == q) found = lo;
                }
                nb[27 * c + j] = found;
            }
}

// One round.  An undecided vertex v scans each neighbour cell in ascending id below v and stops at the first vertex within r that is
// undecided or a seed; v is captured by the smallest such seed if it precedes every such undecided vertex, becomes a seed if there is
// neither, and waits otherwise.  A state is written once, from -1 to its final value, so a stale read only delays a decision.
__global__ void __launch_bounds__(MS_THREADS) weld_round_kernel(const u64* __restrict__ sk, const int* __restrict__ sv, const float* __restrict__ Ps,
                                                                const int* __restrict__ cellof, const int* __restrict__ nb, const int* __restrict__ cstart,
                                                                const int* __restrict__ cend, long long V, const WeldHdr* __restrict__ hdr, int* state, int* und) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= V || sk[i] == CELL_NONE) return;
    volatile int* s = state;
    const int v = sv[i];
    if (s[v] >= 0) return;
    const double r2 = hdr->r2;
    const double px = Ps[3 * i], py = Ps[3 * i + 1], pz = Ps[3 * i + 2];
    int mseed = INT_MAX, mund = INT_MAX;
    const int* nbc = nb + 27LL * cellof[i];
    for (int j = 0; j < 27; ++j) {
        const int c = nbc[j];
        if (c < 0) continue;
        const int e = cend[c];
        for (int p = cstart[c]; p < e; ++p) {
            const int u = sv[p];
            if (u >= v) break;
            const double dx = __dsub_rn(static_cast<double>(Ps[3LL * p]), px);
            const double dy = __dsub_rn(static_cast<double>(Ps[3LL * p + 1]), py);
            const double dz = __dsub_rn(static_cast<double>(Ps[3LL * p + 2]), pz);
            if (!(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) < r2)) continue;
            const int su = s[u];
            if (su < 0) { mund = min(mund, u); break; }
            if (su == u) { mseed = min(mseed, u); break; }
        }
    }
    if (mseed < mund) s[v] = mseed;
    else if (mund == INT_MAX) s[v] = v;
    else atomicAdd(und, 1);
}

__device__ __forceinline__ void sorted3(const int* t, int* a, int* b, int* c) {
    int x = t[0], y = t[1], z = t[2], w;
    if (x > y) { w = x; x = y; y = w; }
    if (y > z) { w = y; y = z; z = w; }
    if (x > y) { w = x; x = y; y = w; }
    *a = x; *b = y; *c = z;
}

// faces onto the representatives; the (middle, largest) key of the index set (CELL_NONE for a face that now repeats an index)
__global__ void __launch_bounds__(MS_THREADS) weld_faces_kernel(const int* __restrict__ Tin, long long F, const int* __restrict__ state, int* __restrict__ T,
                                                                u64* __restrict__ key, int* __restrict__ val) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    int t[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) T[3 * f + k] = t[k] = state[Tin[3 * f + k]];
    int a, b, c;
    sorted3(t, &a, &b, &c);
    key[f] = a == b || b == c ? CELL_NONE : (static_cast<u64>(b) << 32) | static_cast<u64>(c);
    val[f] = static_cast<int>(f);
}

// the smallest index of each face in (middle, largest) order, for the second, stable, pass of the index-set sort
__global__ void __launch_bounds__(MS_THREADS) weld_key1_kernel(const int* __restrict__ T, const u64* __restrict__ key2, const int* __restrict__ val, long long F,
                                                               unsigned* __restrict__ key1) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= F) return;
    int a, b, c;
    sorted3(T + 3LL * val[i], &a, &b, &c);
    key1[i] = key2[i] == CELL_NONE ? 0xffffffffu : static_cast<unsigned>(a);
}

__device__ __forceinline__ bool null_face(const float* P, const int* t) {
    double p0[3], p1[3], p2[3], n[3];
    load3(P, t[0], p0);
    load3(P, t[1], p1);
    load3(P, t[2], p2);
    cross3(p0, p1, p2, n);
    return n[0] == 0.0 && n[1] == 0.0 && n[2] == 0.0;
}

// over the faces sorted by (index set, face id): a face is kept iff its indices are distinct, it is the first of its index set and
// its doubled-area vector (v1 - v0) x (v2 - v0) is not exactly zero
__global__ void __launch_bounds__(MS_THREADS) weld_keep_kernel(const int* __restrict__ T, const float* __restrict__ P, const unsigned* __restrict__ key1,
                                                               const int* __restrict__ val, long long F, int* __restrict__ fkeep) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= F) return;
    const int f = val[i];
    const int* t = T + 3LL * f;
    bool keep = key1[i] != 0xffffffffu;
    if (keep && i > 0 && key1[i - 1] == key1[i]) {
        int a, b, c, x, y, z;
        sorted3(t, &a, &b, &c);
        sorted3(T + 3LL * val[i - 1], &x, &y, &z);
        keep = !(a == x && b == y && c == z);
    }
    fkeep[f] = keep && !null_face(P, t);
}

// ------------------------------------------------------------------------------------------------------------ clean-up: repair
constexpr u64 AREA_NONE = ~0ull;

struct RepHdr {
    int bad;
    int Vs;                     // surviving vertices (the split copies follow them)
};

// undirected edge id of every sorted half-edge key; per edge its face count; per face its three edge ids
__global__ void __launch_bounds__(MS_THREADS) edge_ids_kernel(const u64* __restrict__ sk, const int* __restrict__ sv, const int* __restrict__ flag,
                                                              const int* __restrict__ excl, const int* __restrict__ T, long long n, int* __restrict__ ecnt,
                                                              int* __restrict__ fe) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= n) return;
    const int e = excl[i] + flag[i] - 1, f = sv[i];
    atomicAdd(ecnt + e, 1);
    const int* t = T + 3LL * f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const unsigned u = static_cast<unsigned>(t[k]), v = static_cast<unsigned>(t[(k + 1) % 3]);
        if (((static_cast<u64>(min(u, v)) << 32) | max(u, v)) == sk[i]) fe[3LL * f + k] = e;
    }
}

__global__ void __launch_bounds__(MS_THREADS) new_key_kernel(const u64* __restrict__ sk, long long n, int* __restrict__ flag) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i < n) flag[i] = i == 0 || sk[i] != sk[i - 1];
}

// a face touching an edge with more than two faces is a candidate, keyed by its doubled area |(v1 - v0) x (v2 - v0)| (fp64 bits)
__global__ void __launch_bounds__(MS_THREADS) nm_candidates_kernel(const float* __restrict__ P, const int* __restrict__ T, const int* __restrict__ fe,
                                                                   const int* __restrict__ ecnt, long long F, u64* __restrict__ akey, int* __restrict__ aval,
                                                                   int* __restrict__ fkeep) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    u64 k = AREA_NONE;
    if (ecnt[fe[3 * f]] > 2 || ecnt[fe[3 * f + 1]] > 2 || ecnt[fe[3 * f + 2]] > 2) {
        double p0[3], p1[3], p2[3], c[3];
        load3(P, T[3 * f], p0);
        load3(P, T[3 * f + 1], p1);
        load3(P, T[3 * f + 2], p2);
        cross3(p0, p1, p2, c);
        k = static_cast<u64>(__double_as_longlong(sqrt(__dadd_rn(__dadd_rn(__dmul_rn(c[0], c[0]), __dmul_rn(c[1], c[1])), __dmul_rn(c[2], c[2])))));
    }
    akey[f] = k;
    aval[f] = static_cast<int>(f);
    fkeep[f] = 1;
}

// the sequential definition over the candidates in (area, face id) order: delete a face iff one of its edges still has more than
// two faces.  One warp: the lanes fetch 32 candidates' edge ids, lane 0 decides them in order.
__global__ void __launch_bounds__(32) nm_remove_kernel(const u64* __restrict__ akey, const int* __restrict__ aval, long long F, const int* __restrict__ fe,
                                                       int* ecnt, int* fkeep) {
    const int lane = threadIdx.x;
    for (long long base = 0; base < F; base += 32) {
        const long long i = base + lane;
        const bool cand = i < F && akey[i] != AREA_NONE;
        int f = -1, e0 = 0, e1 = 0, e2 = 0;
        if (cand) {
            f = aval[i];
            e0 = fe[3LL * f];
            e1 = fe[3LL * f + 1];
            e2 = fe[3LL * f + 2];
        }
        const unsigned live = __ballot_sync(0xffffffffu, cand);
        for (int j = 0; j < 32 && ((live >> j) & 1u); ++j) {
            const int fj = __shfl_sync(0xffffffffu, f, j), a = __shfl_sync(0xffffffffu, e0, j), b = __shfl_sync(0xffffffffu, e1, j),
                      c = __shfl_sync(0xffffffffu, e2, j);
            if (lane == 0 && (ecnt[a] > 2 || ecnt[b] > 2 || ecnt[c] > 2)) {
                fkeep[fj] = 0;
                --ecnt[a];
                --ecnt[b];
                --ecnt[c];
            }
            __syncwarp();
        }
        if (live != 0xffffffffu) return;                                   // candidates are a prefix of the sorted keys
    }
}

// corner keys (vertex << 32 | face) of the kept faces (AREA_NONE for the removed ones), value = half-edge id 3 f + k
__global__ void __launch_bounds__(MS_THREADS) rep_corner_keys_kernel(const int* __restrict__ T, const int* __restrict__ fkeep, long long F, u64* __restrict__ ck,
                                                                     int* __restrict__ cv) {
    const long long h = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (h >= 3 * F) return;
    const long long f = h / 3;
    ck[h] = fkeep[f] ? (static_cast<u64>(static_cast<unsigned>(T[h])) << 32) | static_cast<u64>(f) : AREA_NONE;
    cv[h] = static_cast<int>(h);
}

__global__ void __launch_bounds__(MS_THREADS) inverse_kernel(const int* __restrict__ cv, long long n, int* __restrict__ cpos, int* __restrict__ parent) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= n) return;
    cpos[cv[i]] = static_cast<int>(i);
    parent[i] = static_cast<int>(i);
}

// fan keys: corner (v, f) is joined to the corners of v in the faces sharing the edges (v, w) of f; value = the corner's sorted position
__global__ void __launch_bounds__(MS_THREADS) fan_keys_kernel(const int* __restrict__ T, const int* __restrict__ fkeep, const int* __restrict__ cpos, long long F,
                                                              u64* __restrict__ key, int* __restrict__ val) {
    const long long h = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (h >= 3 * F) return;
    const long long f = h / 3;
    const int k = static_cast<int>(h - 3 * f);
    const u64 v = static_cast<unsigned>(T[h]);
    const bool live = fkeep[f];
    key[2 * h] = live ? (v << 32) | static_cast<unsigned>(T[3 * f + (k + 1) % 3]) : AREA_NONE;
    key[2 * h + 1] = live ? (v << 32) | static_cast<unsigned>(T[3 * f + (k + 2) % 3]) : AREA_NONE;
    val[2 * h] = val[2 * h + 1] = cpos[h];
}

// every live corner's fan root (the corner of the fan's smallest face id), the vertices in use, and the split flags: a fan root that
// is not its vertex's first corner gets a copy
__global__ void __launch_bounds__(MS_THREADS) fan_roots_kernel(const u64* __restrict__ ck, long long n, int* parent, int* __restrict__ split, int* __restrict__ vref) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= n) return;
    split[i] = 0;
    if (ck[i] == AREA_NONE) return;
    volatile int* p = parent;
    int r = static_cast<int>(i);
    while (p[r] != r) r = p[r];
    p[i] = r;
    const bool first = i == 0 || (ck[i - 1] >> 32) != (ck[i] >> 32);
    split[i] = r == i && !first;
    vref[ck[i] >> 32] = 1;
}

__global__ void rep_counts_kernel(const int* vref, const int* vpos, long long V, const int* split, const int* spos, long long n3, const int* fkeep, const int* fpos,
                                  long long F, RepHdr* hdr, long long* counts) {
    const int Vs = V ? vpos[V - 1] + vref[V - 1] : 0;
    const long long nsplit = n3 ? static_cast<long long>(spos[n3 - 1]) + split[n3 - 1] : 0;
    hdr->Vs = Vs;
    counts[0] = hdr->bad ? -1 : Vs + nsplit;
    counts[1] = hdr->bad ? -1 : (F ? static_cast<long long>(fpos[F - 1]) + fkeep[F - 1] : 0);
}

__global__ void __launch_bounds__(MS_THREADS) emit_split_kernel(const float* __restrict__ P, const u64* __restrict__ ck, const int* __restrict__ split,
                                                                const int* __restrict__ spos, long long n, const RepHdr* __restrict__ hdr, float* __restrict__ out) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= n || !split[i]) return;
    const long long v = static_cast<long long>(ck[i] >> 32), o = hdr->Vs + static_cast<long long>(spos[i]);
    out[3 * o] = P[3 * v];
    out[3 * o + 1] = P[3 * v + 1];
    out[3 * o + 2] = P[3 * v + 2];
}

__global__ void __launch_bounds__(MS_THREADS) emit_split_faces_kernel(const int* __restrict__ T, const int* __restrict__ fkeep, const int* __restrict__ fpos,
                                                                      const int* __restrict__ cpos, const int* __restrict__ parent, const u64* __restrict__ ck,
                                                                      const int* __restrict__ spos, const int* __restrict__ vpos, long long F,
                                                                      const RepHdr* __restrict__ hdr, long long* __restrict__ out) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F || !fkeep[f]) return;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int r = parent[cpos[3 * f + k]];
        const bool first = r == 0 || (ck[r - 1] >> 32) != (ck[r] >> 32);
        out[3LL * fpos[f] + k] = first ? vpos[T[3 * f + k]] : hdr->Vs + static_cast<long long>(spos[r]);
    }
}

// ------------------------------------------------------------------------------------------------------------ clean-up workspaces
struct WeldWs {
    WeldHdr* hdr;
    int* gbox;
    int *Tin, *T;
    u64* vkey[2];
    int* vval[2];
    int *state, *flag, *excl, *cellof, *cstart, *cend, *nb;
    u64* ukey;
    float* Ps;
    u64* fkey[2];
    int* fval[2];
    unsigned* k1[2];
    int *fkeep, *fpos, *vref, *vpos;
    void* cub;
    size_t cub_bytes, total;
};

WeldWs weld_layout(void* ws, long long V, long long F) {
    Carve c{static_cast<uint8_t*>(ws)};
    WeldWs w;
    w.hdr = c.take<WeldHdr>(1);
    w.gbox = c.take<int>(6);
    w.Tin = c.take<int>(3 * F);
    w.T = c.take<int>(3 * F);
    w.vkey[0] = c.take<u64>(V);
    w.vkey[1] = c.take<u64>(V);
    w.vval[0] = c.take<int>(V);
    w.vval[1] = c.take<int>(V);
    w.state = c.take<int>(V);
    w.flag = c.take<int>(V);
    w.excl = c.take<int>(V);
    w.cellof = c.take<int>(V);
    w.cstart = c.take<int>(V);
    w.cend = c.take<int>(V);
    w.nb = c.take<int>(27 * V);
    w.ukey = c.take<u64>(V);
    w.Ps = c.take<float>(3 * V);
    w.fkey[0] = c.take<u64>(F);
    w.fkey[1] = c.take<u64>(F);
    w.fval[0] = c.take<int>(F);
    w.fval[1] = c.take<int>(F);
    w.k1[0] = c.take<unsigned>(F);
    w.k1[1] = c.take<unsigned>(F);
    w.fkeep = c.take<int>(F);
    w.fpos = c.take<int>(F);
    w.vref = c.take<int>(V);
    w.vpos = c.take<int>(V);
    w.cub_bytes = cub_reserve(F > V ? F : V);
    w.cub = c.take<uint8_t>(static_cast<long long>(w.cub_bytes));
    w.total = c.off;
    return w;
}

struct RepWs {
    RepHdr* hdr;
    int* T;
    u64* key[2];
    int* val[2];
    int *flag, *excl, *ecnt, *fe;
    u64* akey[2];
    int* aval[2];
    u64* ck[2];
    int* cv[2];
    int *cpos, *parent, *split, *spos, *fkeep, *fpos, *vref, *vpos;
    void* cub;
    size_t cub_bytes, total;
};

RepWs rep_layout(void* ws, long long V, long long F) {
    Carve c{static_cast<uint8_t*>(ws)};
    RepWs w;
    w.hdr = c.take<RepHdr>(1);
    w.T = c.take<int>(3 * F);
    w.key[0] = c.take<u64>(6 * F);
    w.key[1] = c.take<u64>(6 * F);
    w.val[0] = c.take<int>(6 * F);
    w.val[1] = c.take<int>(6 * F);
    w.flag = c.take<int>(3 * F);
    w.excl = c.take<int>(3 * F);
    w.ecnt = c.take<int>(3 * F);
    w.fe = c.take<int>(3 * F);
    w.akey[0] = c.take<u64>(F);
    w.akey[1] = c.take<u64>(F);
    w.aval[0] = c.take<int>(F);
    w.aval[1] = c.take<int>(F);
    w.ck[0] = c.take<u64>(3 * F);
    w.ck[1] = c.take<u64>(3 * F);
    w.cv[0] = c.take<int>(3 * F);
    w.cv[1] = c.take<int>(3 * F);
    w.cpos = c.take<int>(3 * F);
    w.parent = c.take<int>(3 * F);
    w.split = c.take<int>(3 * F);
    w.spos = c.take<int>(3 * F);
    w.fkeep = c.take<int>(F);
    w.fpos = c.take<int>(F);
    w.vref = c.take<int>(V);
    w.vpos = c.take<int>(V);
    w.cub_bytes = cub_reserve(6 * F > V ? 6 * F : V);
    w.cub = c.take<uint8_t>(static_cast<long long>(w.cub_bytes));
    w.total = c.off;
    return w;
}

// the CUB scratch the clean-up calls need for sorts of n_sort pairs and scans of n_scan ints, against what the layout reserved
int clean_cub_check(const char* what, long long n_sort, long long n_scan, size_t reserved) {
    size_t b = 0, m = 0;
    cub::DoubleBuffer<u64> dk(nullptr, nullptr);
    cub::DoubleBuffer<unsigned> du(nullptr, nullptr);
    cub::DoubleBuffer<int> dv(nullptr, nullptr);
    TPX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, dk, dv, n_sort, 0, 64));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, du, dv, n_sort, 0, 32));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const int*>(nullptr), static_cast<int*>(nullptr), n_scan));
    m = b > m ? b : m;
    TPX_CHECK(m <= reserved, TPX_ERR_STATE, "%s: sort scratch of %zu bytes exceeds the %zu reserved", what, m, reserved);
    return TPX_OK;
}

}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" {

// ------------------------------------------------------------------------------------------------------------ component filter
size_t tpx_mesh_components_workspace_bytes(int64_t V, int64_t F) {
    if (V < 0 || F < 0 || V >= MS_INDEX_LIMIT || F >= MS_INDEX_LIMIT) return 0;
    return cc_layout(nullptr, V, F).total;
}

int tpx_mesh_components_count(const float* verts, int64_t V, const int64_t* faces_dev, int64_t F, int64_t min_faces, double min_diameter, void* ws,
                              size_t ws_bytes, int64_t* counts_dev, void* stream) {
    TPX_DEVICE_GUARD();   // first: the argument check below sizes the CUB scratch, a CUDA query
    const long long* faces = reinterpret_cast<const long long*>(faces_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = mesh_check("remove_small_components", verts, V, faces, F, ws, ws_bytes, tpx_mesh_components_workspace_bytes(V, F), V, F);
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr, TPX_ERR_ARG, "remove_small_components: null counts");
    const CcWs w = cc_layout(ws, V, F);
    ProfScope prof(PROF_VAE_MISC, st);
    TPX_CUDA(cudaMemsetAsync(w.bad, 0, sizeof(int), st));
    static const int gbox0[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    TPX_CUDA(cudaMemcpyAsync(w.gbox, gbox0, sizeof(gbox0), cudaMemcpyHostToDevice, st));
    if (V) TPX_CUDA(cudaMemsetAsync(w.vref, 0, V * sizeof(int), st));
    if (F) {
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, w.T, w.bad);
        TPX_LAUNCH_CHECK();
        edge_keys_kernel<<<blocks(3 * F), MS_THREADS, 0, st>>>(w.T, F, w.key[0], w.val[0]);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<u64> dk(w.key[0], w.key[1]);
        cub::DoubleBuffer<int> dv(w.val[0], w.val[1]);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, b, dk, dv, 3 * F, 0, key_bits(V), st));
        cc_init_kernel<<<blocks(F), MS_THREADS, 0, st>>>(F, w.parent, w.cnt, w.bmin, w.bmax);
        TPX_LAUNCH_CHECK();
        cc_union_kernel<<<blocks(3 * F), MS_THREADS, 0, st>>>(dk.Current(), dv.Current(), 3 * F, w.parent);
        TPX_LAUNCH_CHECK();
        cc_stats_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T, verts, F, w.parent, w.cnt, w.bmin, w.bmax, w.gbox);
        TPX_LAUNCH_CHECK();
        cc_keep_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.parent, w.cnt, w.bmin, w.bmax, w.gbox, F, min_faces, min_diameter, w.fkeep);
        TPX_LAUNCH_CHECK();
        ref_kernel<<<blocks(3 * F), MS_THREADS, 0, st>>>(w.T, w.fkeep, F, w.vref);
        TPX_LAUNCH_CHECK();
    }
    int r = scan(w.fkeep, w.fpos, F, w.cub, w.cub_bytes, st);
    if (r == TPX_OK) r = scan(w.vref, w.vpos, V, w.cub, w.cub_bytes, st);
    if (r != TPX_OK) return r;
    counts_kernel<<<1, 1, 0, st>>>(w.vref, w.vpos, V, w.fkeep, w.fpos, F, 0, w.bad, counts);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_mesh_components_emit(const float* verts, int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out, int64_t* faces_out, void* stream) {
    TPX_DEVICE_GUARD();
    TPX_CHECK(ws_bytes >= tpx_mesh_components_workspace_bytes(V, F) && ws != nullptr && (V == 0 || verts != nullptr), TPX_ERR_ARG,
              "remove_small_components: bad emit arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const CcWs w = cc_layout(const_cast<void*>(ws), V, F);
    ProfScope prof(PROF_VAE_MISC, st);
    if (V) {
        emit_verts_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, w.vref, w.vpos, V, verts_out);
        TPX_LAUNCH_CHECK();
    }
    if (F) {
        emit_faces_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T, w.fkeep, w.fpos, nullptr, F, w.vpos, reinterpret_cast<long long*>(faces_out));
        TPX_LAUNCH_CHECK();
    }
    return TPX_OK;
}

// ------------------------------------------------------------------------------------------------------------ decimation
size_t tpx_decimate_workspace_bytes(int64_t V, int64_t F) {
    if (V < 0 || F < 0 || V >= MS_INDEX_LIMIT || F >= MS_INDEX_LIMIT) return 0;
    return dec_layout(nullptr, V, F).total;
}

int tpx_decimate(const float* verts, int64_t V, const int64_t* faces_dev, int64_t F, int64_t target, void* ws, size_t ws_bytes, int64_t* counts_dev,
                 int64_t* trace, int64_t trace_cap, void* stream) {
    TPX_DEVICE_GUARD();   // first: the argument check below sizes the CUB scratch, a CUDA query
    const long long* faces = reinterpret_cast<const long long*>(faces_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = mesh_check("decimate", verts, V, faces, F, ws, ws_bytes, tpx_decimate_workspace_bytes(V, F), V, F);
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr && target >= 0, TPX_ERR_ARG, "decimate: null counts or negative target");
    const DecWs w = dec_layout(ws, V, F);
    ProfScope prof(PROF_VAE_MISC, st);
    TPX_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(DecHdr), st));
    if (V) {
        iota_copy_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, V, w.P, w.rep);
        TPX_LAUNCH_CHECK();
    }
    if (F) {
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, w.T[0], &w.hdr->bad);
        TPX_LAUNCH_CHECK();
    }
    const int bits = key_bits(V);
    long long Fc = F, rounds = 0;
    int buf = 0;
    DecHdr h;
    while (Fc > target) {
        const long long n3 = 3 * Fc;
        int* T = w.T[buf];
        corner_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(T, Fc, w.ck[0]);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<u64> dc(w.ck[0], w.ck[1]);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, dc, n3, 0, bits, st));
        const u64* ck = dc.Current();
        TPX_CUDA(cudaMemsetAsync(w.vstart, 0, V * sizeof(int), st));
        TPX_CUDA(cudaMemsetAsync(w.vend, 0, V * sizeof(int), st));
        csr_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(ck, n3, w.vstart, w.vend);
        TPX_LAUNCH_CHECK();
        if (rounds == 0) {
            quadric_kernel<<<blocks(V), MS_THREADS, 0, st>>>(w.P, T, ck, w.vstart, w.vend, V, w.Q);
            TPX_LAUNCH_CHECK();
        }
        vertex_state_kernel<<<blocks(V), MS_THREADS, 0, st>>>(T, ck, w.vstart, w.vend, V, w.frozen, w.deg);
        TPX_LAUNCH_CHECK();
        // edges: sorted unique half-edge keys, into the buffer the sort did not end in
        edge_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(T, Fc, w.hk[0], nullptr);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<u64> dh(w.hk[0], w.hk[1]);
        b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, dh, n3, 0, bits, st));
        const u64* edges = dh.Alternate();
        b = w.cub_bytes;
        TPX_CUDA(cub::DeviceSelect::Unique(w.cub, b, dh.Current(), dh.Alternate(), &w.hdr->E, n3, st));
        TPX_CUDA(cudaMemsetAsync(w.m1, 0xff, V * sizeof(u64), st));
        TPX_CUDA(cudaMemsetAsync(&w.hdr->n_acc, 0, sizeof(int), st));
        edge_cost_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(edges, w.hdr, w.P, w.Q, T, ck, w.vstart, w.vend, w.frozen, w.deg, w.ekey, w.xbar, w.m1);
        TPX_LAUNCH_CHECK();
        TPX_CUDA(cudaMemcpyAsync(w.m2, w.m1, V * sizeof(u64), cudaMemcpyDeviceToDevice, st));
        edge_min2_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(edges, w.hdr, w.m1, w.m2);
        TPX_LAUNCH_CHECK();
        edge_accept_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(edges, w.hdr, w.ekey, w.m2, w.aflag);
        TPX_LAUNCH_CHECK();
        TPX_CUDA(cudaMemcpyAsync(&h, w.hdr, sizeof(DecHdr), cudaMemcpyDeviceToHost, st));
        TPX_CUDA(cudaStreamSynchronize(st));                              // the one readback of the round
        TPX_CHECK(h.bad == 0, TPX_ERR_ARG, "decimate: %d faces have an index outside [0, %lld) or a repeated index", h.bad, (long long)V);
        TPX_CHECK(h.E < (1LL << 32), TPX_ERR_SHAPE, "decimate: %lld edges: edge ids must fit in 32 bits", h.E);
        if (h.n_acc == 0) break;
        long long k = h.n_acc;
        if (Fc - 2 * k < target) {                                        // last round: the smallest keys only
            k = (Fc - target + 1) / 2;
            u64* sel = w.ck[dc.selector ^ 1];                             // the corner keys' spare buffer and the half-edges' sorted buffer
            b = w.cub_bytes;
            TPX_CUDA(cub::DeviceSelect::Flagged(w.cub, b, w.ekey, w.aflag, sel, &w.hdr->n_sel, h.E, st));
            cub::DoubleBuffer<u64> ds(sel, dh.Current());
            b = w.cub_bytes;
            TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, ds, static_cast<long long>(h.n_acc), 0, 64, st));
            set_thr_kernel<<<1, 1, 0, st>>>(w.hdr, ds.Current(), k);
        } else {
            set_thr_kernel<<<1, 1, 0, st>>>(w.hdr, nullptr, 0);
        }
        TPX_LAUNCH_CHECK();
        collapse_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(edges, w.hdr, w.ekey, w.aflag, w.xbar, w.P, w.Q, w.rep);
        TPX_LAUNCH_CHECK();
        remap_kernel<<<blocks(Fc), MS_THREADS, 0, st>>>(T, Fc, w.rep, w.fkeep);
        TPX_LAUNCH_CHECK();
        const int r = scan(w.fkeep, w.fpos, Fc, w.cub, w.cub_bytes, st);
        if (r != TPX_OK) return r;
        compact_faces_kernel<<<blocks(Fc), MS_THREADS, 0, st>>>(T, Fc, w.fkeep, w.fpos, w.T[buf ^ 1], w.hdr, buf ^ 1);
        TPX_LAUNCH_CHECK();
        buf ^= 1;
        Fc -= 2 * k;
        if (trace && rounds < trace_cap) trace[rounds] = Fc;
        ++rounds;
    }
    if (rounds == 0 && F > 0) {                                           // no round ran: the input faces still need their check
        TPX_CUDA(cudaMemcpyAsync(&h, w.hdr, sizeof(DecHdr), cudaMemcpyDeviceToHost, st));
        TPX_CUDA(cudaStreamSynchronize(st));
        TPX_CHECK(h.bad == 0, TPX_ERR_ARG, "decimate: %d faces have an index outside [0, %lld) or a repeated index", h.bad, (long long)V);
    }
    if (rounds == 0) {
        static const int zero = 0;
        TPX_CUDA(cudaMemcpyAsync(&w.hdr->buf, &zero, sizeof(int), cudaMemcpyHostToDevice, st));
        TPX_CUDA(cudaMemcpyAsync(&w.hdr->F, &F, sizeof(long long), cudaMemcpyHostToDevice, st));
        TPX_CUDA(cudaStreamSynchronize(st));                              // the host values above live on this stack frame
    }
    if (V) TPX_CUDA(cudaMemsetAsync(w.vref, 0, V * sizeof(int), st));
    if (Fc) {
        ref_kernel<<<blocks(3 * Fc), MS_THREADS, 0, st>>>(w.T[buf], nullptr, Fc, w.vref);
        TPX_LAUNCH_CHECK();
    }
    const int r = scan(w.vref, w.vpos, V, w.cub, w.cub_bytes, st);
    if (r != TPX_OK) return r;
    counts_kernel<<<1, 1, 0, st>>>(w.vref, w.vpos, V, nullptr, nullptr, 0, Fc, nullptr, counts);
    TPX_LAUNCH_CHECK();
    TPX_CUDA(cudaMemcpyAsync(counts + 2, &rounds, sizeof(long long), cudaMemcpyHostToDevice, st));
    TPX_CUDA(cudaStreamSynchronize(st));
    return TPX_OK;
}

int tpx_decimate_emit(int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out, int64_t* faces_out, void* stream) {
    TPX_DEVICE_GUARD();
    TPX_CHECK(ws_bytes >= tpx_decimate_workspace_bytes(V, F) && ws != nullptr, TPX_ERR_ARG, "decimate: bad emit arguments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const DecWs w = dec_layout(const_cast<void*>(ws), V, F);
    DecHdr h;
    TPX_CUDA(cudaMemcpyAsync(&h, w.hdr, sizeof(DecHdr), cudaMemcpyDeviceToHost, st));
    TPX_CUDA(cudaStreamSynchronize(st));
    ProfScope prof(PROF_VAE_MISC, st);
    if (V) {
        emit_verts_kernel<<<blocks(V), MS_THREADS, 0, st>>>(w.P, w.vref, w.vpos, V, verts_out);
        TPX_LAUNCH_CHECK();
    }
    if (h.F) {
        emit_faces_kernel<<<blocks(h.F), MS_THREADS, 0, st>>>(w.T[h.buf], nullptr, nullptr, nullptr, h.F, w.vpos, reinterpret_cast<long long*>(faces_out));
        TPX_LAUNCH_CHECK();
    }
    return TPX_OK;
}


// ------------------------------------------------------------------------------------------------------------ clean-up
size_t tpx_mesh_weld_workspace_bytes(int64_t V, int64_t F) {
    if (V < 0 || F < 0 || V >= MS_INDEX_LIMIT || F >= MS_INDEX_LIMIT) return 0;
    return weld_layout(nullptr, V, F).total;
}

int tpx_mesh_weld_count(const float* verts, int64_t V, const int64_t* faces_dev, int64_t F, double merge_distance, void* ws, size_t ws_bytes, int64_t* counts_dev,
                        void* stream) {
    const long long* faces = reinterpret_cast<const long long*>(faces_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = mesh_args("clean_mesh", verts, V, faces, F, ws, ws_bytes, tpx_mesh_weld_workspace_bytes(V, F));
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr && merge_distance >= 0.0 && merge_distance < 1e300, TPX_ERR_ARG, "clean_mesh: null counts or merge distance %g", merge_distance);
    TPX_DEVICE_GUARD();
    const WeldWs w = weld_layout(ws, V, F);
    const long long n = F > V ? F : V;
    rc = clean_cub_check("clean_mesh", n, n, w.cub_bytes);
    if (rc != TPX_OK) return rc;
    ProfScope prof(PROF_VAE_MISC, st);
    TPX_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(WeldHdr), st));
    static const int gbox0[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    TPX_CUDA(cudaMemcpyAsync(w.gbox, gbox0, sizeof(gbox0), cudaMemcpyHostToDevice, st));
    if (V) TPX_CUDA(cudaMemsetAsync(w.vref, 0, V * sizeof(int), st));
    if (F) {
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, w.Tin, &w.hdr->bad, true);
        TPX_LAUNCH_CHECK();
        ref_kernel<<<blocks(3 * F), MS_THREADS, 0, st>>>(w.Tin, nullptr, F, w.vref);
        TPX_LAUNCH_CHECK();
    }
    const bool merge = V > 0 && merge_distance > 0.0;
    if (merge) {
        ref_box_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, w.vref, V, w.gbox);
        TPX_LAUNCH_CHECK();
        weld_params_kernel<<<1, 1, 0, st>>>(w.gbox, merge_distance, w.hdr);
        TPX_LAUNCH_CHECK();
    }
    if (V) {
        weld_keys_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, w.vref, V, w.hdr, w.vkey[0], w.vval[0], w.state);
        TPX_LAUNCH_CHECK();
    }
    long long rounds = 0;
    if (merge) {
        const u64* sk;
        const int* sv;
        rc = sort_pairs(w.vkey[0], w.vkey[1], w.vval[0], w.vval[1], V, 64, w.cub, w.cub_bytes, st, &sk, &sv);
        if (rc != TPX_OK) return rc;
        cell_flags_kernel<<<blocks(V), MS_THREADS, 0, st>>>(sk, sv, verts, V, w.flag, w.Ps);
        TPX_LAUNCH_CHECK();
        rc = scan(w.flag, w.excl, V, w.cub, w.cub_bytes, st);
        if (rc != TPX_OK) return rc;
        cell_ranges_kernel<<<blocks(V), MS_THREADS, 0, st>>>(sk, w.flag, w.excl, V, w.cellof, w.ukey, w.cstart, w.cend, w.hdr);
        TPX_LAUNCH_CHECK();
        cell_nb_kernel<<<blocks(V), MS_THREADS, 0, st>>>(w.ukey, w.hdr, w.nb);
        TPX_LAUNCH_CHECK();
        // every round decides at least the smallest undecided vertex, so the loop ends; the host reads the counts once per batch
        for (;;) {
            TPX_CUDA(cudaMemsetAsync(w.hdr->und, 0, sizeof(w.hdr->und), st));
            for (int b = 0; b < WELD_BATCH; ++b) {
                weld_round_kernel<<<blocks(V), MS_THREADS, 0, st>>>(sk, sv, w.Ps, w.cellof, w.nb, w.cstart, w.cend, V, w.hdr, w.state, w.hdr->und + b);
                TPX_LAUNCH_CHECK();
            }
            int und[WELD_BATCH];
            TPX_CUDA(cudaMemcpyAsync(und, w.hdr->und, sizeof(und), cudaMemcpyDeviceToHost, st));
            TPX_CUDA(cudaStreamSynchronize(st));
            int b = 0;
            while (b < WELD_BATCH && und[b] != 0) ++b;
            if (b < WELD_BATCH) {
                rounds += b + 1;
                break;
            }
            rounds += WELD_BATCH;
        }
    }
    if (F) {
        weld_faces_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.Tin, F, w.state, w.T, w.fkey[0], w.fval[0]);
        TPX_LAUNCH_CHECK();
        const u64* sk;
        const int* sv;
        rc = sort_pairs(w.fkey[0], w.fkey[1], w.fval[0], w.fval[1], F, 64, w.cub, w.cub_bytes, st, &sk, &sv);
        if (rc != TPX_OK) return rc;
        weld_key1_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T, sk, sv, F, w.k1[0]);
        TPX_LAUNCH_CHECK();
        int* sv_alt = sv == w.fval[0] ? w.fval[1] : w.fval[0];
        cub::DoubleBuffer<unsigned> dk(w.k1[0], w.k1[1]);
        cub::DoubleBuffer<int> dv(const_cast<int*>(sv), sv_alt);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortPairs(w.cub, b, dk, dv, F, 0, 32, st));   // stable: (index set, face id) order
        weld_keep_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T, verts, dk.Current(), dv.Current(), F, w.fkeep);
        TPX_LAUNCH_CHECK();
        TPX_CUDA(cudaMemsetAsync(w.vref, 0, V * sizeof(int), st));
        ref_kernel<<<blocks(3 * F), MS_THREADS, 0, st>>>(w.T, w.fkeep, F, w.vref);
        TPX_LAUNCH_CHECK();
    }
    rc = scan(w.fkeep, w.fpos, F, w.cub, w.cub_bytes, st);
    if (rc == TPX_OK) rc = scan(w.vref, w.vpos, V, w.cub, w.cub_bytes, st);
    if (rc != TPX_OK) return rc;
    counts_kernel<<<1, 1, 0, st>>>(w.vref, w.vpos, V, w.fkeep, w.fpos, F, 0, &w.hdr->bad, counts);
    TPX_LAUNCH_CHECK();
    TPX_CUDA(cudaMemcpyAsync(counts + 2, &rounds, sizeof(long long), cudaMemcpyHostToDevice, st));
    TPX_CUDA(cudaStreamSynchronize(st));                                  // `rounds` lives on this stack frame
    return TPX_OK;
}

int tpx_mesh_weld_emit(const float* verts, int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out, int64_t* faces_out, void* stream) {
    TPX_CHECK(ws_bytes >= tpx_mesh_weld_workspace_bytes(V, F) && ws != nullptr && (V == 0 || verts != nullptr), TPX_ERR_ARG, "clean_mesh: bad emit arguments");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const WeldWs w = weld_layout(const_cast<void*>(ws), V, F);
    ProfScope prof(PROF_VAE_MISC, st);
    if (V) {
        emit_verts_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, w.vref, w.vpos, V, verts_out);
        TPX_LAUNCH_CHECK();
    }
    if (F) {
        emit_faces_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T, w.fkeep, w.fpos, nullptr, F, w.vpos, reinterpret_cast<long long*>(faces_out));
        TPX_LAUNCH_CHECK();
    }
    return TPX_OK;
}

size_t tpx_mesh_repair_workspace_bytes(int64_t V, int64_t F) {
    if (V < 0 || F < 0 || V >= MS_INDEX_LIMIT || F >= MS_INDEX_LIMIT / 2) return 0;
    return rep_layout(nullptr, V, F).total;
}

int tpx_mesh_repair_count(const float* verts, int64_t V, const int64_t* faces_dev, int64_t F, void* ws, size_t ws_bytes, int64_t* counts_dev, void* stream) {
    const long long* faces = reinterpret_cast<const long long*>(faces_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TPX_CHECK(F < MS_INDEX_LIMIT / 2, TPX_ERR_SHAPE, "repair: %lld faces: must be below 2^30", (long long)F);
    int rc = mesh_args("repair", verts, V, faces, F, ws, ws_bytes, tpx_mesh_repair_workspace_bytes(V, F));
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr, TPX_ERR_ARG, "repair: null counts");
    TPX_DEVICE_GUARD();
    const RepWs w = rep_layout(ws, V, F);
    rc = clean_cub_check("repair", 6 * F > V ? 6 * F : V, 3 * F > V ? 3 * F : V, w.cub_bytes);
    if (rc != TPX_OK) return rc;
    ProfScope prof(PROF_VAE_MISC, st);
    TPX_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(RepHdr), st));
    if (V) TPX_CUDA(cudaMemsetAsync(w.vref, 0, V * sizeof(int), st));
    const long long n3 = 3 * F;
    if (F) {
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, w.T, &w.hdr->bad);
        TPX_LAUNCH_CHECK();
        // 5. non-manifold edges: edge ids and face counts, candidates by (doubled area, face id), the sequential removal
        edge_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.T, F, w.key[0], w.val[0]);
        TPX_LAUNCH_CHECK();
        const u64* sk;
        const int* sv;
        rc = sort_pairs(w.key[0], w.key[1], w.val[0], w.val[1], n3, key_bits(V), w.cub, w.cub_bytes, st, &sk, &sv);
        if (rc != TPX_OK) return rc;
        new_key_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(sk, n3, w.flag);
        TPX_LAUNCH_CHECK();
        rc = scan(w.flag, w.excl, n3, w.cub, w.cub_bytes, st);
        if (rc != TPX_OK) return rc;
        TPX_CUDA(cudaMemsetAsync(w.ecnt, 0, n3 * sizeof(int), st));
        edge_ids_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(sk, sv, w.flag, w.excl, w.T, n3, w.ecnt, w.fe);
        TPX_LAUNCH_CHECK();
        nm_candidates_kernel<<<blocks(F), MS_THREADS, 0, st>>>(verts, w.T, w.fe, w.ecnt, F, w.akey[0], w.aval[0], w.fkeep);
        TPX_LAUNCH_CHECK();
        const u64* ak;
        const int* av;
        rc = sort_pairs(w.akey[0], w.akey[1], w.aval[0], w.aval[1], F, 64, w.cub, w.cub_bytes, st, &ak, &av);
        if (rc != TPX_OK) return rc;
        nm_remove_kernel<<<1, 32, 0, st>>>(ak, av, F, w.fe, w.ecnt, w.fkeep);
        TPX_LAUNCH_CHECK();
        // 6. non-manifold vertices: corners sorted by (vertex, face) into ck[0], fans as unions of corners over shared edges
        rep_corner_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.T, w.fkeep, F, w.ck[0], w.cv[0]);
        TPX_LAUNCH_CHECK();
        const u64* cks;
        const int* cvs;
        rc = sort_pairs(w.ck[0], w.ck[1], w.cv[0], w.cv[1], n3, 64, w.cub, w.cub_bytes, st, &cks, &cvs);
        if (rc != TPX_OK) return rc;
        if (cks != w.ck[0]) TPX_CUDA(cudaMemcpyAsync(w.ck[0], cks, n3 * sizeof(u64), cudaMemcpyDeviceToDevice, st));
        inverse_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(cvs, n3, w.cpos, w.parent);
        TPX_LAUNCH_CHECK();
        fan_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.T, w.fkeep, w.cpos, F, w.key[0], w.val[0]);
        TPX_LAUNCH_CHECK();
        rc = sort_pairs(w.key[0], w.key[1], w.val[0], w.val[1], 2 * n3, 64, w.cub, w.cub_bytes, st, &sk, &sv);
        if (rc != TPX_OK) return rc;
        cc_union_kernel<<<blocks(2 * n3), MS_THREADS, 0, st>>>(sk, sv, 2 * n3, w.parent);
        TPX_LAUNCH_CHECK();
        fan_roots_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.ck[0], n3, w.parent, w.split, w.vref);
        TPX_LAUNCH_CHECK();
    }
    rc = scan(w.split, w.spos, n3, w.cub, w.cub_bytes, st);
    if (rc == TPX_OK) rc = scan(w.vref, w.vpos, V, w.cub, w.cub_bytes, st);
    if (rc == TPX_OK) rc = scan(w.fkeep, w.fpos, F, w.cub, w.cub_bytes, st);
    if (rc != TPX_OK) return rc;
    rep_counts_kernel<<<1, 1, 0, st>>>(w.vref, w.vpos, V, w.split, w.spos, n3, w.fkeep, w.fpos, F, w.hdr, counts);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_mesh_repair_emit(const float* verts, int64_t V, int64_t F, const void* ws, size_t ws_bytes, float* verts_out, int64_t* faces_out, void* stream) {
    TPX_CHECK(ws_bytes >= tpx_mesh_repair_workspace_bytes(V, F) && ws != nullptr && (V == 0 || verts != nullptr), TPX_ERR_ARG, "repair: bad emit arguments");
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const RepWs w = rep_layout(const_cast<void*>(ws), V, F);
    ProfScope prof(PROF_VAE_MISC, st);
    if (V) {
        emit_verts_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, w.vref, w.vpos, V, verts_out);
        TPX_LAUNCH_CHECK();
    }
    if (F) {
        emit_split_kernel<<<blocks(3 * F), MS_THREADS, 0, st>>>(verts, w.ck[0], w.split, w.spos, 3 * F, w.hdr, verts_out);
        TPX_LAUNCH_CHECK();
        emit_split_faces_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T, w.fkeep, w.fpos, w.cpos, w.parent, w.ck[0], w.spos, w.vpos, F, w.hdr,
                                                                  reinterpret_cast<long long*>(faces_out));
        TPX_LAUNCH_CHECK();
    }
    return TPX_OK;
}

}  // extern "C"
