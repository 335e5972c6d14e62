// Isotropic remeshing (DESIGN.md §1 f-7, "Isotropic remeshing contract"): the GPU stand-in for pymeshlab's
// meshing_isotropic_explicit_remeshing that decimate_mesh(..., remesh=True) runs after the quadric decimation (utils/meshutils.py:101-105,
// inference.py:128-129).  The host drives the iterations (mesh.remesh); per iteration:
//   * split (tpx_remesh_split_count / _emit, the mesh grows): long edges flagged over the sorted unique edge list, new vertex ids
//     from a scan in edge order, child counts per face from a scan in face order, the crease list rewritten and re-sorted;
//   * relax (tpx_remesh_relax, in place): collapse rounds (decimation's two-ring minimum acceptance), valence flip rounds (minimum over
//     the candidates touching the quad), one Jacobi tangential smoothing pass, projection onto the input through a uniform grid
//     (tpx_remesh_begin builds it) searched in growing shells.  The host reads one header back per round.
// Every round rebuilds the corner CSR, the frozen state and the edge list with the kernels decimation uses (mesh_common.cuh).  Every
// output position comes from a sort or a scan and every atomic is a min or a count, so results are identical across calls and
// streams.  Compiled with -fmad=false; the fp64 arithmetic is spelled with _rn intrinsics in the order of the numpy test oracle (remesh.py).
#include "mesh_common.cuh"

namespace tpx {

namespace {
constexpr int GRID_AXIS = 160;                     // cells per axis at most GRID_AXIS + 1
constexpr long long GRID_CELLS = (GRID_AXIS + 1LL) * (GRID_AXIS + 1LL) * (GRID_AXIS + 1LL);
constexpr double GRID_SLACK = 1.001;               // cell side over the largest face extent: a face's box spans at most 2 cells per axis

__device__ __forceinline__ double dot3(const double* a, const double* b) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

// squared fp64 distance of two fp32 points, (dx² + dy²) + dz²
__device__ __forceinline__ double dist2(const float* a, const float* b) {
    const double dx = __dsub_rn(static_cast<double>(a[0]), static_cast<double>(b[0]));
    const double dy = __dsub_rn(static_cast<double>(a[1]), static_cast<double>(b[1]));
    const double dz = __dsub_rn(static_cast<double>(a[2]), static_cast<double>(b[2]));
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__device__ __forceinline__ float midf(float a, float b) {
    return __double2float_rn(__dmul_rn(__dadd_rn(static_cast<double>(a), static_cast<double>(b)), 0.5));
}

// n1·n2 < cos(feature) · (|n1| |n2|): the two faces meet at more than the feature angle
__device__ __forceinline__ bool crease_pair(const double* n1, const double* n2, double cosf) {
    return dot3(n1, n2) < __dmul_rn(cosf, __dmul_rn(sqrt(dot3(n1, n1)), sqrt(dot3(n2, n2))));
}

__device__ __forceinline__ long long find_key(const u64* a, long long n, u64 key) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long m = (lo + hi) >> 1;
        if (a[m] < key) lo = m + 1;
        else hi = m;
    }
    return lo < n && a[lo] == key ? lo : -1;
}

__device__ __forceinline__ u64 ekey_of(int a, int b) {
    return (static_cast<u64>(static_cast<unsigned>(min(a, b))) << 32) | static_cast<unsigned>(max(a, b));
}

// ------------------------------------------------------------------------------------------------------------ features
// an edge with exactly two faces (a run of two equal sorted half-edge keys) is a crease iff its faces meet beyond the feature angle
__global__ void __launch_bounds__(MS_THREADS) crease_init_kernel(const u64* __restrict__ key, const int* __restrict__ fid, long long n, const float* __restrict__ P,
                                                                 const int* __restrict__ T, double cosf, int* __restrict__ flag) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= n) return;
    int f = 0;
    if ((i == 0 || key[i - 1] != key[i]) && i + 1 < n && key[i + 1] == key[i] && (i + 2 >= n || key[i + 2] != key[i])) {
        double p[3][3], n1[3], n2[3];
        for (int s = 0; s < 2; ++s) {
            const int* t = T + 3LL * fid[i + s];
#pragma unroll
            for (int k = 0; k < 3; ++k) load3(P, t[k], p[k]);
            cross3(p[0], p[1], p[2], s ? n2 : n1);
        }
        f = crease_pair(n1, n2, cosf);
    }
    flag[i] = f;
}

__global__ void __launch_bounds__(MS_THREADS) feature_kernel(const uint8_t* __restrict__ frozen, long long V, uint8_t* __restrict__ feat) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i < V) feat[i] = frozen[i];
}

__global__ void __launch_bounds__(MS_THREADS) crease_ends_kernel(const u64* __restrict__ creases, long long nC, uint8_t* __restrict__ feat) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= nC) return;
    feat[creases[i] >> 32] = 1;
    feat[static_cast<unsigned>(creases[i])] = 1;
}

// ------------------------------------------------------------------------------------------------------------ split
__global__ void __launch_bounds__(MS_THREADS) split_flag_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, long long cap, const float* __restrict__ P,
                                                                double hi2, int* __restrict__ flag) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= cap) return;
    int f = 0;
    if (e < hdr->E) {
        const u64 ed = edges[e];
        f = dist2(P + 3 * (ed >> 32), P + 3LL * static_cast<unsigned>(ed)) > hi2;
    }
    flag[e] = f;
}

// the split vertex of each edge (t[k], t[k+1]) of face f, or -1
__device__ __forceinline__ int face_splits(const int* t, const u64* edges, long long E, const int* flag, const int* pos, long long V, int* s) {
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const long long e = find_key(edges, E, ekey_of(t[k], t[k == 2 ? 0 : k + 1]));
        s[k] = flag[e] ? static_cast<int>(V + pos[e]) : -1;
        cnt += s[k] >= 0;
    }
    return cnt;
}

__global__ void __launch_bounds__(MS_THREADS) split_count_kernel(const int* __restrict__ T, long long F, const u64* __restrict__ edges, const DecHdr* __restrict__ hdr,
                                                                 const int* __restrict__ flag, const int* __restrict__ pos, long long V, int* __restrict__ kids) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    int s[3];
    kids[f] = 1 + face_splits(T + 3 * f, edges, hdr->E, flag, pos, V, s);
}

// 1 or 2 per crease: a split crease leaves its two halves
__global__ void __launch_bounds__(MS_THREADS) crease_split_count_kernel(const u64* __restrict__ creases, long long nC, const u64* __restrict__ edges,
                                                                        const DecHdr* __restrict__ hdr, const int* __restrict__ flag, int* __restrict__ cnt) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= nC) return;
    cnt[i] = 1 + flag[find_key(edges, hdr->E, creases[i])];
}

__global__ void split_counts_kernel(const DecHdr* hdr, const int* flag, const int* pos, long long V, const int* kids, const int* kpos, long long F, const int* ccnt,
                                    const int* cpos, long long nC, long long* counts) {
    const long long E = hdr->E;
    const bool bad = hdr->bad != 0;
    counts[0] = bad ? -1 : V + (E ? static_cast<long long>(pos[E - 1]) + flag[E - 1] : 0);
    counts[1] = bad ? -1 : (F ? static_cast<long long>(kpos[F - 1]) + kids[F - 1] : 0);
    counts[2] = bad ? -1 : (nC ? static_cast<long long>(cpos[nC - 1]) + ccnt[nC - 1] : 0);
}

__global__ void __launch_bounds__(MS_THREADS) split_verts_kernel(const float* __restrict__ P, long long V, const u64* __restrict__ edges, const DecHdr* __restrict__ hdr,
                                                                 long long cap, const int* __restrict__ flag, const int* __restrict__ pos, float* __restrict__ out) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i < V) {
        out[3 * i] = P[3 * i];
        out[3 * i + 1] = P[3 * i + 1];
        out[3 * i + 2] = P[3 * i + 2];
    }
    if (i >= cap || i >= hdr->E || !flag[i]) return;
    const u64 ed = edges[i];
    const float* a = P + 3 * (ed >> 32);
    const float* b = P + 3LL * static_cast<unsigned>(ed);
    const long long o = V + pos[i];
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * o + d] = midf(a[d], b[d]);
}

__device__ __forceinline__ void put(long long* out, long long o, int a, int b, int c) {
    out[3 * o] = a;
    out[3 * o + 1] = b;
    out[3 * o + 2] = c;
}

// children of face f at kpos[f]..: the face rotated to its canonical pattern, then the fixed child order of the contract
__global__ void __launch_bounds__(MS_THREADS) split_faces_kernel(const int* __restrict__ T, long long F, const u64* __restrict__ edges, const DecHdr* __restrict__ hdr,
                                                                 const int* __restrict__ flag, const int* __restrict__ pos, long long V, const float* __restrict__ Pn,
                                                                 const int* __restrict__ kpos, long long* __restrict__ out) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    const int* t = T + 3 * f;
    int s[3];
    const int cnt = face_splits(t, edges, hdr->E, flag, pos, V, s);
    int r = 0;
    if (cnt == 1) r = s[0] >= 0 ? 0 : (s[1] >= 0 ? 1 : 2);
    if (cnt == 2) r = ((s[0] < 0 ? 0 : (s[1] < 0 ? 1 : 2)) + 1) % 3;
    const int v0 = t[r], v1 = t[(r + 1) % 3], v2 = t[(r + 2) % 3], m0 = s[r], m1 = s[(r + 1) % 3], m2 = s[(r + 2) % 3];
    const long long o = kpos[f];
    if (cnt == 0) {
        put(out, o, v0, v1, v2);
    } else if (cnt == 1) {
        put(out, o, v0, m0, v2);
        put(out, o + 1, m0, v1, v2);
    } else if (cnt == 2) {
        const double da = dist2(Pn + 3LL * m0, Pn + 3LL * v2), db = dist2(Pn + 3LL * v0, Pn + 3LL * m1);
        if (da < db) {
            put(out, o, v0, m0, v2);
            put(out, o + 2, m0, m1, v2);
        } else {
            put(out, o, v0, m0, m1);
            put(out, o + 2, v0, m1, v2);
        }
        put(out, o + 1, m0, v1, m1);
    } else {
        put(out, o, v0, m0, m2);
        put(out, o + 1, m0, v1, m1);
        put(out, o + 2, m2, m1, v2);
        put(out, o + 3, m0, m1, m2);
    }
}

__global__ void __launch_bounds__(MS_THREADS) split_creases_kernel(const u64* __restrict__ creases, long long nC, const u64* __restrict__ edges, const DecHdr* __restrict__ hdr,
                                                                   const int* __restrict__ flag, const int* __restrict__ pos, long long V, const int* __restrict__ cpos,
                                                                   u64* __restrict__ out) {
    const long long i = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (i >= nC) return;
    const u64 c = creases[i];
    const long long e = find_key(edges, hdr->E, c);
    const long long o = cpos[i];
    if (!flag[e]) {
        out[o] = c;
        return;
    }
    const u64 m = static_cast<u64>(V + pos[e]);
    out[o] = (c >> 32) << 32 | m;
    out[o + 1] = (c & 0xFFFFFFFFull) << 32 | m;
}

// ------------------------------------------------------------------------------------------------------------ collapse
__global__ void __launch_bounds__(MS_THREADS, 1) collapse_cost_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, const float* __restrict__ P,
                                                                    const int* __restrict__ T, const u64* __restrict__ ck, const int* __restrict__ vstart,
                                                                    const int* __restrict__ vend, const uint8_t* __restrict__ feat, const int* __restrict__ deg,
                                                                    double lo2, double hi2, u64* __restrict__ ekey, float* __restrict__ xbar, u64* m1) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E) return;
    const u64 ed = edges[e];
    const int a = static_cast<int>(ed >> 32), b = static_cast<int>(static_cast<unsigned>(ed));
    const double len2 = dist2(P + 3LL * a, P + 3LL * b);
    u64 key = KEY_NONE;
    if (len2 < lo2 && !(feat[a] && feat[b])) {
        const int s = feat[a] ? a : (feat[b] ? b : a), r = s == a ? b : a;
        float x[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) x[d] = feat[s] ? P[3LL * s + d] : midf(P[3LL * a + d], P[3LL * b + d]);
        const int sr = vstart[r], nr = vend[r] - sr, ss = vstart[s], ns = vend[s] - ss;
        int c = -1, d = -1, link = 0;
        bool ok = true;
        for (int i = 0; i < nr; ++i) {
            int o, in;
            corner(ck, T, r, sr + i, &o, &in);
            if (o == s) c = in;
            if (in == s) d = o;
            bool common = false;
            for (int j = 0; j < ns; ++j) {
                int os, is;
                corner(ck, T, s, ss + j, &os, &is);
                common = common || os == o || is == o;
            }
            link += common;
            if (o != s && !(dist2(P + 3LL * o, x) < hi2)) ok = false;
        }
        for (int j = 0; j < ns; ++j) {
            int os, is;
            corner(ck, T, s, ss + j, &os, &is);
            if (os != r && !(dist2(P + 3LL * os, x) < hi2)) ok = false;
            if (is != r && !(dist2(P + 3LL * is, x) < hi2)) ok = false;
        }
        ok = ok && link == 2 && c >= 0 && d >= 0 && c != d && deg[a] + deg[b] >= 7 && deg[c] >= 4 && deg[d] >= 4;
        ok = ok && star_ok(P, T, ck, sr, nr, r, s, x) && star_ok(P, T, ck, ss, ns, s, r, x);
        if (ok) {
            key = (static_cast<u64>(__float_as_uint(__double2float_rn(len2))) << 32) | static_cast<u64>(e);
            xbar[3 * e] = x[0];
            xbar[3 * e + 1] = x[1];
            xbar[3 * e + 2] = x[2];
            atomicMin(m1 + a, key);
            atomicMin(m1 + b, key);
        }
    }
    ekey[e] = key;
}

__global__ void __launch_bounds__(MS_THREADS) collapse_apply_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, const int* __restrict__ aflag,
                                                                    const float* __restrict__ xbar, const uint8_t* __restrict__ feat, float* __restrict__ P,
                                                                    int* __restrict__ rep) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E || !aflag[e]) return;
    const u64 ed = edges[e];
    const int a = static_cast<int>(ed >> 32), b = static_cast<int>(static_cast<unsigned>(ed));
    const int s = feat[a] ? a : (feat[b] ? b : a), r = s == a ? b : a;
    P[3LL * s] = xbar[3 * e];
    P[3LL * s + 1] = xbar[3 * e + 1];
    P[3LL * s + 2] = xbar[3 * e + 2];
    rep[r] = s;
}

// ------------------------------------------------------------------------------------------------------------ flip
struct Quad {
    int x, y, c, d, f1, f2;
};

// the quad of edge (a, b) seen from its smaller non-frozen end x: faces f1 = (x, y, c) and f2 = (x, d, y); false when both ends are frozen
__device__ __forceinline__ bool quad_of(int a, int b, const uint8_t* frozen, const u64* ck, const int* T, const int* vstart, const int* vend, Quad* q) {
    if (frozen[a] && frozen[b]) return false;
    q->x = !frozen[a] ? a : b;
    q->y = q->x == a ? b : a;
    q->c = q->d = q->f1 = q->f2 = -1;
    const int s = vstart[q->x], n = vend[q->x] - s;
    for (int i = 0; i < n; ++i) {
        int o, in;
        const int f = corner(ck, T, q->x, s + i, &o, &in);
        if (o == q->y && q->f1 < 0) { q->c = in; q->f1 = f; }
        if (in == q->y && q->f2 < 0) { q->d = o; q->f2 = f; }
    }
    return q->f1 >= 0 && q->f2 >= 0;
}

__device__ __forceinline__ bool nonzero3(const double* n) { return n[0] != 0.0 || n[1] != 0.0 || n[2] != 0.0; }

__global__ void __launch_bounds__(MS_THREADS, 1) flip_cost_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, const float* __restrict__ P,
                                                                const int* __restrict__ T, const u64* __restrict__ ck, const int* __restrict__ vstart,
                                                                const int* __restrict__ vend, const uint8_t* __restrict__ frozen, const int* __restrict__ deg,
                                                                const u64* __restrict__ creases, long long nC, double cosf, u64* __restrict__ ekey, u64* m1) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E) return;
    const u64 ed = edges[e];
    const int a = static_cast<int>(ed >> 32), b = static_cast<int>(static_cast<unsigned>(ed));
    u64 key = KEY_NONE;
    Quad q;
    if (find_key(creases, nC, ed) < 0 && quad_of(a, b, frozen, ck, T, vstart, vend, &q) && q.c != q.d && find_key(edges, hdr->E, ekey_of(q.c, q.d)) < 0) {
        const int ex = deg[q.x] - (frozen[q.x] ? 4 : 6), ey = deg[q.y] - (frozen[q.y] ? 4 : 6);
        const int ec = deg[q.c] - (frozen[q.c] ? 4 : 6), edd = deg[q.d] - (frozen[q.d] ? 4 : 6);
        const int gain = (2 * ex - 1) + (2 * ey - 1) - (2 * ec + 1) - (2 * edd + 1);
        if (gain > 0) {
            double px[3], py[3], pc[3], pd[3], o1[3], o2[3], n1[3], n2[3];
            load3(P, q.x, px);
            load3(P, q.y, py);
            load3(P, q.c, pc);
            load3(P, q.d, pd);
            cross3(px, py, pc, o1);
            cross3(px, pd, py, o2);
            cross3(px, pd, pc, n1);
            cross3(pd, py, pc, n2);
            const bool ok = nonzero3(n1) && nonzero3(n2) && dot3(n1, o1) > 0.0 && dot3(n1, o2) > 0.0 && dot3(n2, o1) > 0.0 && dot3(n2, o2) > 0.0 &&
                            !crease_pair(n1, n2, cosf);
            if (ok) {
                key = (static_cast<u64>(0xFFFFFFFFu - static_cast<unsigned>(gain)) << 32) | static_cast<u64>(e);
                atomicMin(m1 + q.x, key);
                atomicMin(m1 + q.y, key);
                atomicMin(m1 + q.c, key);
                atomicMin(m1 + q.d, key);
            }
        }
    }
    ekey[e] = key;
}

__global__ void __launch_bounds__(MS_THREADS) flip_accept_kernel(const u64* __restrict__ edges, DecHdr* hdr, const int* __restrict__ T, const u64* __restrict__ ck,
                                                                 const int* __restrict__ vstart, const int* __restrict__ vend, const uint8_t* __restrict__ frozen,
                                                                 const u64* __restrict__ ekey, const u64* __restrict__ m1, int* __restrict__ aflag) {
    __shared__ int s_warp[MS_THREADS / 32];
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    int acc = 0;
    if (e < hdr->E) {
        const u64 key = ekey[e];
        if (key != KEY_NONE) {
            const u64 ed = edges[e];
            Quad q;
            quad_of(static_cast<int>(ed >> 32), static_cast<int>(static_cast<unsigned>(ed)), frozen, ck, T, vstart, vend, &q);
            acc = m1[q.x] == key && m1[q.y] == key && m1[q.c] == key && m1[q.d] == key;
        }
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

// accepted quads share no vertex, so a thread reads and writes only faces of its own quad
__global__ void __launch_bounds__(MS_THREADS) flip_apply_kernel(const u64* __restrict__ edges, const DecHdr* __restrict__ hdr, int* T, const u64* __restrict__ ck,
                                                                const int* __restrict__ vstart, const int* __restrict__ vend, const uint8_t* __restrict__ frozen,
                                                                const int* __restrict__ aflag) {
    const long long e = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (e >= hdr->E || !aflag[e]) return;
    const u64 ed = edges[e];
    Quad q;
    quad_of(static_cast<int>(ed >> 32), static_cast<int>(static_cast<unsigned>(ed)), frozen, ck, T, vstart, vend, &q);
    int* t1 = T + 3LL * q.f1;
    int* t2 = T + 3LL * q.f2;
    t1[0] = q.x; t1[1] = q.d; t1[2] = q.c;
    t2[0] = q.d; t2[1] = q.y; t2[2] = q.c;
}

// ------------------------------------------------------------------------------------------------------------ smoothing
__global__ void __launch_bounds__(MS_THREADS) smooth_kernel(const float* __restrict__ P, const int* __restrict__ T, const u64* __restrict__ ck, const int* __restrict__ vstart,
                                                            const int* __restrict__ vend, const uint8_t* __restrict__ feat, long long V, float* __restrict__ out) {
    const long long vv = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (vv >= V) return;
    const int v = static_cast<int>(vv);
    float q[3] = {P[3LL * v], P[3LL * v + 1], P[3LL * v + 2]};
    if (!feat[v]) {
        const int s = vstart[v], n = vend[v] - s;
        double c[3] = {0.0, 0.0, 0.0}, nn[3] = {0.0, 0.0, 0.0};
        int last = -1;
        for (int k = 0; k < n; ++k) {                                  // neighbours in ascending id (a closed fan lists each once as out)
            int next = INT_MAX;
            for (int i = 0; i < n; ++i) {
                int o, in;
                corner(ck, T, v, s + i, &o, &in);
                if (o > last && o < next) next = o;
            }
#pragma unroll
            for (int d = 0; d < 3; ++d) c[d] = __dadd_rn(c[d], static_cast<double>(P[3LL * next + d]));
            last = next;
        }
        for (int i = 0; i < n; ++i) {                                  // faces in ascending id
            const int* t = T + 3LL * static_cast<unsigned>(ck[s + i]);
            double p0[3], p1[3], p2[3], cr[3];
            load3(P, t[0], p0);
            load3(P, t[1], p1);
            load3(P, t[2], p2);
            cross3(p0, p1, p2, cr);
#pragma unroll
            for (int d = 0; d < 3; ++d) nn[d] = __dadd_rn(nn[d], cr[d]);
        }
        const double ln = sqrt(dot3(nn, nn));
        if (ln != 0.0) {
            double p[3], dd[3];
            load3(P, v, p);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                c[d] = __ddiv_rn(c[d], static_cast<double>(n));
                nn[d] = __ddiv_rn(nn[d], ln);
                dd[d] = __dsub_rn(c[d], p[d]);
            }
            const double t = dot3(nn, dd);
            float x[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) x[d] = __double2float_rn(__dadd_rn(p[d], __dsub_rn(dd[d], __dmul_rn(nn[d], t))));
            if (star_ok(P, T, ck, s, n, v, -1, x)) {
                q[0] = x[0];
                q[1] = x[1];
                q[2] = x[2];
            }
        }
    }
    out[3LL * v] = q[0];
    out[3LL * v + 1] = q[1];
    out[3LL * v + 2] = q[2];
}

// ------------------------------------------------------------------------------------------------------------ projection
struct GridHdr {
    double lo[3];
    double h;
    int n[3];
    int bad;              // a face box over more than 2 cells on an axis (cannot happen with the slack; checked anyway)
    int gbox[6];          // box of the input's referenced vertices, order-preserving ints
    int mext;             // largest face box side, fp32 bits (non-negative)
};

struct GridWs {
    GridHdr* hdr;
    int* T;                     // the input faces, int32
    int *cstart, *cend;
    u64* key[2];
    void* cub;
    size_t cub_bytes, total;
};

GridWs grid_layout(void* g, long long F) {
    Carve c{static_cast<uint8_t*>(g)};
    GridWs w;
    w.hdr = c.take<GridHdr>(1);
    w.T = c.take<int>(3 * F);
    w.cstart = c.take<int>(GRID_CELLS + 1);
    w.cend = c.take<int>(GRID_CELLS + 1);
    w.key[0] = c.take<u64>(8 * F);
    w.key[1] = c.take<u64>(8 * F);
    w.cub_bytes = cub_reserve(8 * F);
    w.cub = c.take<uint8_t>(static_cast<long long>(w.cub_bytes));
    w.total = c.off;
    return w;
}

__global__ void __launch_bounds__(MS_THREADS) grid_box_kernel(const float* __restrict__ P, const int* __restrict__ T, long long F, GridHdr* g) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    int lo[3] = {INT_MAX, INT_MAX, INT_MAX}, hi[3] = {INT_MIN, INT_MIN, INT_MIN};
    float ext = 0.0f;
    if (f < F) {
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            float a = P[3LL * T[3 * f] + d], b = a;
#pragma unroll
            for (int k = 1; k < 3; ++k) {
                const float x = P[3LL * T[3 * f + k] + d];
                a = fminf(a, x);
                b = fmaxf(b, x);
            }
            lo[d] = ord_f32(a);
            hi[d] = ord_f32(b);
            ext = fmaxf(ext, b - a);
        }
    }
    int m = __float_as_int(ext);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            lo[d] = min(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
            hi[d] = max(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&g->mext, m);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            atomicMin(g->gbox + d, lo[d]);
            atomicMax(g->gbox + 3 + d, hi[d]);
        }
    }
}

__global__ void grid_params_kernel(GridHdr* g) {
    double ext[3], m = 0.0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        g->lo[d] = unord_f32(g->gbox[d]);
        ext[d] = __dsub_rn(static_cast<double>(unord_f32(g->gbox[3 + d])), g->lo[d]);
        m = fmax(m, ext[d]);
    }
    double h = fmax(__dmul_rn(static_cast<double>(__int_as_float(g->mext)), GRID_SLACK), m / GRID_AXIS);
    if (!(h > 0.0) || !isfinite(h)) h = 1.0;
    g->h = h;
#pragma unroll
    for (int d = 0; d < 3; ++d) g->n[d] = min(static_cast<int>(floor(ext[d] / h)) + 1, GRID_AXIS + 1);
}

__device__ __forceinline__ int cell_of(const GridHdr* g, int d, double x) {
    const double u = floor(__ddiv_rn(__dsub_rn(x, g->lo[d]), g->h));
    return u < 0.0 ? 0 : (u >= g->n[d] - 1 ? g->n[d] - 1 : static_cast<int>(u));
}

// up to 8 (cell << 32 | face) keys per face, padded with a key in the spare cell GRID_CELLS
__global__ void __launch_bounds__(MS_THREADS) grid_keys_kernel(const float* __restrict__ P, const int* __restrict__ T, long long F, GridHdr* g, u64* __restrict__ key) {
    const long long f = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (f >= F) return;
    int i0[3], i1[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float a = P[3LL * T[3 * f] + d], b = a;
#pragma unroll
        for (int k = 1; k < 3; ++k) {
            const float x = P[3LL * T[3 * f + k] + d];
            a = fminf(a, x);
            b = fmaxf(b, x);
        }
        i0[d] = cell_of(g, d, a);
        i1[d] = cell_of(g, d, b);
        if (i1[d] - i0[d] > 1) {
            atomicAdd(&g->bad, 1);
            i1[d] = i0[d] + 1;
        }
    }
    int k = 0;
    for (int x = i0[0]; x <= i1[0]; ++x)
        for (int y = i0[1]; y <= i1[1]; ++y)
            for (int z = i0[2]; z <= i1[2]; ++z)
                key[8 * f + k++] = (static_cast<u64>((static_cast<long long>(x) * g->n[1] + y) * g->n[2] + z) << 32) | static_cast<u64>(f);
    for (; k < 8; ++k) key[8 * f + k] = (static_cast<u64>(GRID_CELLS) << 32) | static_cast<u64>(f);
}

// Ericson's closest point of p on triangle (a, b, c); the region tests in the numpy oracle's order
__device__ void closest_point(const double* p, const double* a, const double* b, const double* c, double* q) {
    double ab[3], ac[3], ap[3], bp[3], cp[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        ab[d] = __dsub_rn(b[d], a[d]);
        ac[d] = __dsub_rn(c[d], a[d]);
        ap[d] = __dsub_rn(p[d], a[d]);
        bp[d] = __dsub_rn(p[d], b[d]);
        cp[d] = __dsub_rn(p[d], c[d]);
    }
    const double d1 = dot3(ab, ap), d2 = dot3(ac, ap), d3 = dot3(ab, bp), d4 = dot3(ac, bp), d5 = dot3(ab, cp), d6 = dot3(ac, cp);
    const double vc = __dsub_rn(__dmul_rn(d1, d4), __dmul_rn(d3, d2));
    const double vb = __dsub_rn(__dmul_rn(d5, d2), __dmul_rn(d1, d6));
    const double va = __dsub_rn(__dmul_rn(d3, d6), __dmul_rn(d5, d4));
    if (d1 <= 0.0 && d2 <= 0.0) { q[0] = a[0]; q[1] = a[1]; q[2] = a[2]; return; }
    if (d3 >= 0.0 && d4 <= d3) { q[0] = b[0]; q[1] = b[1]; q[2] = b[2]; return; }
    if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
        const double t = __ddiv_rn(d1, __dsub_rn(d1, d3));
#pragma unroll
        for (int d = 0; d < 3; ++d) q[d] = __dadd_rn(a[d], __dmul_rn(ab[d], t));
        return;
    }
    if (d6 >= 0.0 && d5 <= d6) { q[0] = c[0]; q[1] = c[1]; q[2] = c[2]; return; }
    if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
        const double t = __ddiv_rn(d2, __dsub_rn(d2, d6));
#pragma unroll
        for (int d = 0; d < 3; ++d) q[d] = __dadd_rn(a[d], __dmul_rn(ac[d], t));
        return;
    }
    const double e43 = __dsub_rn(d4, d3), e56 = __dsub_rn(d5, d6);
    if (va <= 0.0 && e43 >= 0.0 && e56 >= 0.0) {
        const double t = __ddiv_rn(e43, __dadd_rn(e43, e56));
#pragma unroll
        for (int d = 0; d < 3; ++d) q[d] = __dadd_rn(b[d], __dmul_rn(__dsub_rn(c[d], b[d]), t));
        return;
    }
    const double s = __dadd_rn(__dadd_rn(va, vb), vc);
    if (!(s > 0.0)) { q[0] = a[0]; q[1] = a[1]; q[2] = a[2]; return; }
    const double v = __ddiv_rn(vb, s), w = __ddiv_rn(vc, s);
#pragma unroll
    for (int d = 0; d < 3; ++d) q[d] = __dadd_rn(__dadd_rn(a[d], __dmul_rn(ab[d], v)), __dmul_rn(ac[d], w));
}

// the faces registered in one cell against p: keeps the smallest squared distance, then the smallest face id
__device__ __forceinline__ void visit_cell(long long cell, const double* p, const float* P0, const int* T0, const int* cstart, const int* cend, const u64* items,
                                           double* best, int* bf, double* bq) {
    for (int i = cstart[cell]; i < cend[cell]; ++i) {
        const int f = static_cast<int>(static_cast<unsigned>(items[i]));
        const int* t = T0 + 3LL * f;
        double a[3], b[3], c[3], cr[3], q[3];
        load3(P0, t[0], a);
        load3(P0, t[1], b);
        load3(P0, t[2], c);
        cross3(a, b, c, cr);
        if (!nonzero3(cr)) continue;
        closest_point(p, a, b, c, q);
        const double dx = __dsub_rn(q[0], p[0]), dy = __dsub_rn(q[1], p[1]), dz = __dsub_rn(q[2], p[2]);
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (d2 < *best || (d2 == *best && f < *bf)) {
            *best = d2;
            *bf = f;
            bq[0] = q[0];
            bq[1] = q[1];
            bq[2] = q[2];
        }
    }
}

// closest point of the input to each point i (every i, or those with feat[i] == 0): smallest squared distance, then smallest face id.
// Shell k is every in-grid cell at Chebyshev distance exactly k from the point's cell: whole z ranges in the columns on the shell's
// rim, only z = ci ± k in the columns inside it.  The walk stops when the distance to the cells beyond shell k exceeds the best found,
// or when the shell covers the grid.  out may alias P (each thread reads and writes only its own point); a point with no face keeps
// its position (face -1).
__global__ void __launch_bounds__(MS_THREADS, 1) project_kernel(const float* P, float* out, long long n_pts, const uint8_t* __restrict__ feat,
                                                              const float* __restrict__ P0, const int* __restrict__ T0, const GridHdr* __restrict__ g,
                                                              const int* __restrict__ cstart, const int* __restrict__ cend, const u64* __restrict__ items,
                                                              long long* __restrict__ face_out) {
    const long long vv = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (vv >= n_pts || (feat && feat[vv])) return;
    double p[3];
    load3(P, static_cast<int>(vv), p);
    int ci[3], n[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        ci[d] = cell_of(g, d, p[d]);
        n[d] = g->n[d];
    }
    const double h = g->h;
    double best = INFINITY, bq[3] = {p[0], p[1], p[2]};
    int bf = INT_MAX;
    for (int k = 0;; ++k) {
        for (int x = max(ci[0] - k, 0); x <= min(ci[0] + k, n[0] - 1); ++x)
            for (int y = max(ci[1] - k, 0); y <= min(ci[1] + k, n[1] - 1); ++y) {
                const long long col = (static_cast<long long>(x) * n[1] + y) * n[2];
                if (abs(x - ci[0]) == k || abs(y - ci[1]) == k) {               // rim column (k = 0 included): all of it
                    for (int z = max(ci[2] - k, 0); z <= min(ci[2] + k, n[2] - 1); ++z)
                        visit_cell(col + z, p, P0, T0, cstart, cend, items, &best, &bf, bq);
                } else {                                                       // inside column: its bottom and top cells, if in the grid
                    if (ci[2] - k >= 0) visit_cell(col + ci[2] - k, p, P0, T0, cstart, cend, items, &best, &bf, bq);
                    if (ci[2] + k <= n[2] - 1) visit_cell(col + ci[2] + k, p, P0, T0, cstart, cend, items, &best, &bf, bq);
                }
            }
        double lb = INFINITY;                                          // distance to the cells not visited yet
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            if (ci[d] - k > 0) lb = fmin(lb, p[d] - (g->lo[d] + (ci[d] - k) * h));
            if (ci[d] + k < n[d] - 1) lb = fmin(lb, (g->lo[d] + (ci[d] + k + 1) * h) - p[d]);
        }
        if (lb == INFINITY) break;
        lb -= 1e-6 * h;
        if (lb > 0.0 && lb * lb > best) break;
    }
    if (face_out) face_out[vv] = bf == INT_MAX ? -1 : bf;
#pragma unroll
    for (int d = 0; d < 3; ++d) out[3 * vv + d] = __double2float_rn(bq[d]);
}

// ------------------------------------------------------------------------------------------------------------ workspace / driver
struct RmWs {
    DecHdr* hdr;
    int* T[2];
    u64* ck[2];
    u64* hk[2];                 // 6F: half-edge keys, then the rewritten crease list
    u64* edges;
    u64* ekey;
    float* xbar;
    int *aflag, *eflag, *epos, *ccnt, *cpos, *fkeep, *fpos;
    int *vstart, *vend, *deg, *rep;
    uint8_t *frozen, *feat;
    u64 *m1, *m2;
    float* P2;
    void* cub;
    size_t cub_bytes, total;
};

RmWs rm_layout(void* ws, long long V, long long F) {
    Carve c{static_cast<uint8_t*>(ws)};
    RmWs w;
    w.hdr = c.take<DecHdr>(1);
    w.T[0] = c.take<int>(3 * F);
    w.T[1] = c.take<int>(3 * F);
    w.ck[0] = c.take<u64>(3 * F);
    w.ck[1] = c.take<u64>(3 * F);
    w.hk[0] = c.take<u64>(6 * F);
    w.hk[1] = c.take<u64>(6 * F);
    w.edges = c.take<u64>(3 * F);
    w.ekey = c.take<u64>(3 * F);
    w.xbar = c.take<float>(9 * F);
    w.aflag = c.take<int>(3 * F);
    w.eflag = c.take<int>(3 * F);
    w.epos = c.take<int>(3 * F);
    w.ccnt = c.take<int>(3 * F);
    w.cpos = c.take<int>(3 * F);
    w.fkeep = c.take<int>(F);
    w.fpos = c.take<int>(F);
    w.vstart = c.take<int>(V);
    w.vend = c.take<int>(V);
    w.deg = c.take<int>(V);
    w.rep = c.take<int>(V);
    w.frozen = c.take<uint8_t>(V);
    w.feat = c.take<uint8_t>(V);
    w.m1 = c.take<u64>(V);
    w.m2 = c.take<u64>(V);
    w.P2 = c.take<float>(3 * V);
    w.cub_bytes = cub_reserve(6 * F);
    w.cub = c.take<uint8_t>(static_cast<long long>(w.cub_bytes));
    w.total = c.off;
    return w;
}

// the CUB scratch of every call below at these sizes, against the reservation
int rm_cub_check(const char* what, long long F, long long F0, size_t reserved, size_t grid_reserved) {
    size_t b = 0, m = 0;
    cub::DoubleBuffer<u64> dk(nullptr, nullptr);
    cub::DoubleBuffer<int> dv(nullptr, nullptr);
    TPX_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b, dk, 6 * F, 0, 64));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, b, dk, dv, 3 * F, 0, 64));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceSelect::Unique(nullptr, b, static_cast<const u64*>(nullptr), static_cast<u64*>(nullptr), static_cast<long long*>(nullptr), 3 * F));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceSelect::Flagged(nullptr, b, static_cast<const u64*>(nullptr), static_cast<const int*>(nullptr), static_cast<u64*>(nullptr),
                                        static_cast<long long*>(nullptr), 3 * F));
    m = b > m ? b : m;
    TPX_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const int*>(nullptr), static_cast<int*>(nullptr), 3 * F));
    m = b > m ? b : m;
    TPX_CHECK(m <= reserved, TPX_ERR_STATE, "%s: sort scratch of %zu bytes exceeds the %zu reserved", what, m, reserved);
    if (F0 >= 0) {
        TPX_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b, dk, 8 * F0, 0, 64));
        TPX_CHECK(b <= grid_reserved, TPX_ERR_STATE, "%s: grid sort scratch of %zu bytes exceeds the %zu reserved", what, b, grid_reserved);
    }
    return TPX_OK;
}

// corner CSR, frozen flags and degrees, the sorted unique edges (count in hdr->E) and the feature flags of the live faces
int topology(const RmWs& w, const int* T, long long F, long long V, const u64* creases, long long nC, cudaStream_t st, const u64** ck_out) {
    const long long n3 = 3 * F;
    const int bits = key_bits(V);
    corner_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(T, F, w.ck[0]);
    TPX_LAUNCH_CHECK();
    cub::DoubleBuffer<u64> dc(w.ck[0], w.ck[1]);
    size_t b = w.cub_bytes;
    TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, dc, n3, 0, bits, st));
    const u64* ck = dc.Current();
    TPX_CUDA(cudaMemsetAsync(w.vstart, 0, V * sizeof(int), st));
    TPX_CUDA(cudaMemsetAsync(w.vend, 0, V * sizeof(int), st));
    csr_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(ck, n3, w.vstart, w.vend);
    TPX_LAUNCH_CHECK();
    vertex_state_kernel<<<blocks(V), MS_THREADS, 0, st>>>(T, ck, w.vstart, w.vend, V, w.frozen, w.deg);
    TPX_LAUNCH_CHECK();
    edge_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(T, F, w.hk[0], nullptr);
    TPX_LAUNCH_CHECK();
    cub::DoubleBuffer<u64> dh(w.hk[0], w.hk[1]);
    b = w.cub_bytes;
    TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, dh, n3, 0, bits, st));
    b = w.cub_bytes;
    TPX_CUDA(cub::DeviceSelect::Unique(w.cub, b, dh.Current(), w.edges, &w.hdr->E, n3, st));
    feature_kernel<<<blocks(V), MS_THREADS, 0, st>>>(w.frozen, V, w.feat);
    TPX_LAUNCH_CHECK();
    if (nC) {
        crease_ends_kernel<<<blocks(nC), MS_THREADS, 0, st>>>(creases, nC, w.feat);
        TPX_LAUNCH_CHECK();
    }
    *ck_out = ck;
    return TPX_OK;
}

int read_hdr(const RmWs& w, DecHdr* h, cudaStream_t st) {
    TPX_CUDA(cudaMemcpyAsync(h, w.hdr, sizeof(DecHdr), cudaMemcpyDeviceToHost, st));
    TPX_CUDA(cudaStreamSynchronize(st));
    return TPX_OK;
}

__global__ void __launch_bounds__(MS_THREADS) faces_out_kernel(const int* __restrict__ T, long long F, long long* __restrict__ out) {
    const long long h = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (h < 3 * F) out[h] = T[h];
}

__global__ void __launch_bounds__(MS_THREADS) iota_kernel(int* rep, long long V) {
    const long long v = blockIdx.x * static_cast<long long>(MS_THREADS) + threadIdx.x;
    if (v < V) rep[v] = static_cast<int>(v);
}

__global__ void begin_counts_kernel(const DecHdr* hdr, const long long* nC, const GridHdr* g, long long* counts) {
    counts[0] = hdr->bad != 0 || g->bad != 0 ? -1 : *nC;
}

// a collapse removes exactly the two faces on its edge (its removed end is not frozen, so the edge has two faces), so the host keeps
// the face count without a readback; the count the last compaction wrote (hdr->F) must agree with it
int face_count_check(const DecHdr& h, long long Fc, long long collapse_rounds) {
    TPX_CHECK(collapse_rounds == 0 || h.F == Fc, TPX_ERR_STATE, "remesh relax: %lld faces after compaction, %lld expected", h.F, Fc);
    return TPX_OK;
}

int crease_arg(const void* creases, long long nC, long long F) {
    TPX_CHECK(nC >= 0 && nC <= 3 * F && (creases != nullptr || nC == 0), TPX_ERR_ARG, "remesh: %lld creases for %lld faces", nC, F);
    return TPX_OK;
}
}  // namespace

}  // namespace tpx

using namespace tpx;

extern "C" {

size_t tpx_remesh_workspace_bytes(int64_t V, int64_t F) {
    if (V < 0 || F < 0 || V >= MS_INDEX_LIMIT || F >= MS_INDEX_LIMIT / 2) return 0;
    return rm_layout(nullptr, V, F).total;
}

size_t tpx_remesh_grid_bytes(int64_t F) {
    if (F < 0 || F >= MS_INDEX_LIMIT / 8) return 0;
    return grid_layout(nullptr, F).total;
}

int tpx_remesh_begin(const float* verts, int64_t V, const int64_t* faces_dev, int64_t F, double cos_feature, void* grid, size_t grid_bytes, void* ws,
                     size_t ws_bytes, int64_t* creases_out, int64_t* counts_dev, void* stream) {
    const long long* faces = reinterpret_cast<const long long*>(faces_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = mesh_args("remesh", verts, V, faces, F, ws, ws_bytes, tpx_remesh_workspace_bytes(V, F));
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr && (creases_out != nullptr || F == 0) && grid != nullptr && (reinterpret_cast<uintptr_t>(grid) & 255) == 0, TPX_ERR_ARG,
              "remesh: null counts, creases or grid, or an unaligned grid");
    TPX_CHECK(grid_bytes >= tpx_remesh_grid_bytes(F) && tpx_remesh_grid_bytes(F) > 0, TPX_ERR_ARG, "remesh: grid of %zu bytes, %zu needed", grid_bytes,
              tpx_remesh_grid_bytes(F));
    TPX_CHECK(cos_feature >= -1.0 && cos_feature <= 1.0, TPX_ERR_ARG, "remesh: cos(feature angle) %g outside [-1, 1]", cos_feature);
    TPX_DEVICE_GUARD();
    const RmWs w = rm_layout(ws, V, F);
    const GridWs g = grid_layout(grid, F);
    rc = rm_cub_check("remesh", F, F, w.cub_bytes, g.cub_bytes);
    if (rc != TPX_OK) return rc;
    ProfScope prof(PROF_VAE_MISC, st);
    TPX_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(DecHdr), st));
    TPX_CUDA(cudaMemsetAsync(g.hdr, 0, sizeof(GridHdr), st));
    static const int gbox0[6] = {INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN};
    TPX_CUDA(cudaMemcpyAsync(g.hdr->gbox, gbox0, sizeof(gbox0), cudaMemcpyHostToDevice, st));
    TPX_CUDA(cudaMemsetAsync(&w.hdr->n_sel, 0, sizeof(long long), st));
    TPX_CUDA(cudaMemsetAsync(g.cstart, 0, (GRID_CELLS + 1) * sizeof(int), st));
    TPX_CUDA(cudaMemsetAsync(g.cend, 0, (GRID_CELLS + 1) * sizeof(int), st));
    if (F) {
        const long long n3 = 3 * F;
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, g.T, &w.hdr->bad);
        TPX_LAUNCH_CHECK();
        // creases: half-edge keys with their faces, sorted; runs of exactly two tested
        edge_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(g.T, F, w.hk[0], w.aflag);
        TPX_LAUNCH_CHECK();
        const u64* sk;
        const int* sv;
        rc = sort_pairs(w.hk[0], w.hk[1], w.aflag, w.epos, n3, key_bits(V), w.cub, w.cub_bytes, st, &sk, &sv);
        if (rc != TPX_OK) return rc;
        crease_init_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(sk, sv, n3, verts, g.T, cos_feature, w.eflag);
        TPX_LAUNCH_CHECK();
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceSelect::Flagged(w.cub, b, sk, w.eflag, reinterpret_cast<u64*>(creases_out), &w.hdr->n_sel, n3, st));
        // projection grid over the input
        grid_box_kernel<<<blocks(F), MS_THREADS, 0, st>>>(verts, g.T, F, g.hdr);
        TPX_LAUNCH_CHECK();
        grid_params_kernel<<<1, 1, 0, st>>>(g.hdr);
        TPX_LAUNCH_CHECK();
        grid_keys_kernel<<<blocks(F), MS_THREADS, 0, st>>>(verts, g.T, F, g.hdr, g.key[0]);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<u64> dg(g.key[0], g.key[1]);
        b = g.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortKeys(g.cub, b, dg, 8 * F, 0, 64, st));
        if (dg.selector) TPX_CUDA(cudaMemcpyAsync(g.key[0], g.key[1], 8 * F * sizeof(u64), cudaMemcpyDeviceToDevice, st));
        csr_kernel<<<blocks(8 * F), MS_THREADS, 0, st>>>(g.key[0], 8 * F, g.cstart, g.cend);
        TPX_LAUNCH_CHECK();
    }
    begin_counts_kernel<<<1, 1, 0, st>>>(w.hdr, &w.hdr->n_sel, g.hdr, counts);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_remesh_closest(const float* pts, int64_t n, const float* verts0, int64_t V0, int64_t F0, const void* grid, size_t grid_bytes, float* out,
                       int64_t* face_out_dev, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TPX_CHECK(n >= 0 && (n == 0 || (pts != nullptr && out != nullptr && face_out_dev != nullptr)) && V0 >= 0 && F0 >= 0 && (verts0 != nullptr || V0 == 0) &&
                  (V0 > 0 || F0 == 0) && grid != nullptr && tpx_remesh_grid_bytes(F0) > 0 && grid_bytes >= tpx_remesh_grid_bytes(F0),
              TPX_ERR_ARG, "remesh closest: bad points, input mesh or grid");
    TPX_DEVICE_GUARD();
    const GridWs g = grid_layout(const_cast<void*>(grid), F0);
    ProfScope prof(PROF_VAE_MISC, st);
    if (n && F0) {
        project_kernel<<<blocks(n), MS_THREADS, 0, st>>>(pts, out, n, nullptr, verts0, g.T, g.hdr, g.cstart, g.cend, g.key[0],
                                                          reinterpret_cast<long long*>(face_out_dev));
        TPX_LAUNCH_CHECK();
    } else if (n) {
        TPX_CUDA(cudaMemcpyAsync(out, pts, 3 * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
        TPX_CUDA(cudaMemsetAsync(face_out_dev, 0xff, n * sizeof(int64_t), st));
    }
    return TPX_OK;
}

int tpx_remesh_split_count(const float* verts, int64_t V, const int64_t* faces_dev, int64_t F, const int64_t* creases_dev, int64_t nC, double target_len,
                           void* ws, size_t ws_bytes, int64_t* counts_dev, void* stream) {
    const long long* faces = reinterpret_cast<const long long*>(faces_dev);
    const u64* creases = reinterpret_cast<const u64*>(creases_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = mesh_args("remesh split", verts, V, faces, F, ws, ws_bytes, tpx_remesh_workspace_bytes(V, F));
    if (rc == TPX_OK) rc = crease_arg(creases_dev, nC, F);
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr && target_len > 0.0 && isfinite(target_len), TPX_ERR_ARG, "remesh split: null counts or target length %g", target_len);
    TPX_DEVICE_GUARD();
    const RmWs w = rm_layout(ws, V, F);
    rc = rm_cub_check("remesh split", F, -1, w.cub_bytes, 0);
    if (rc != TPX_OK) return rc;
    ProfScope prof(PROF_VAE_MISC, st);
    const double hi = target_len * (4.0 / 3.0), hi2 = hi * hi;
    const long long n3 = 3 * F;
    TPX_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(DecHdr), st));
    if (F) {
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, w.T[0], &w.hdr->bad);
        TPX_LAUNCH_CHECK();
        edge_keys_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.T[0], F, w.hk[0], nullptr);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<u64> dh(w.hk[0], w.hk[1]);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, dh, n3, 0, key_bits(V), st));
        b = w.cub_bytes;
        TPX_CUDA(cub::DeviceSelect::Unique(w.cub, b, dh.Current(), w.edges, &w.hdr->E, n3, st));
        split_flag_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, n3, verts, hi2, w.eflag);
        TPX_LAUNCH_CHECK();
        rc = scan(w.eflag, w.epos, n3, w.cub, w.cub_bytes, st);
        if (rc != TPX_OK) return rc;
        split_count_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T[0], F, w.edges, w.hdr, w.eflag, w.epos, V, w.fkeep);
        TPX_LAUNCH_CHECK();
        rc = scan(w.fkeep, w.fpos, F, w.cub, w.cub_bytes, st);
        if (rc != TPX_OK) return rc;
        if (nC) {
            crease_split_count_kernel<<<blocks(nC), MS_THREADS, 0, st>>>(creases, nC, w.edges, w.hdr, w.eflag, w.ccnt);
            TPX_LAUNCH_CHECK();
            rc = scan(w.ccnt, w.cpos, nC, w.cub, w.cub_bytes, st);
            if (rc != TPX_OK) return rc;
        }
    }
    split_counts_kernel<<<1, 1, 0, st>>>(w.hdr, w.eflag, w.epos, V, w.fkeep, w.fpos, F, w.ccnt, w.cpos, nC, counts);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_remesh_split_emit(const float* verts, int64_t V, int64_t F, const int64_t* creases_dev, int64_t nC, int64_t nC_out, const void* ws, size_t ws_bytes,
                          float* verts_out, int64_t* faces_out, int64_t* creases_out, void* stream) {
    const u64* creases = reinterpret_cast<const u64*>(creases_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TPX_CHECK(ws != nullptr && ws_bytes >= tpx_remesh_workspace_bytes(V, F) && tpx_remesh_workspace_bytes(V, F) > 0 && (V == 0 || (verts && verts_out)) &&
                  (F == 0 || faces_out) && nC_out >= nC && nC_out <= 2 * nC && (nC_out == 0 || creases_out),
              TPX_ERR_ARG, "remesh split: bad emit arguments");
    int rc = crease_arg(creases_dev, nC, F);
    if (rc != TPX_OK) return rc;
    TPX_DEVICE_GUARD();
    const RmWs w = rm_layout(const_cast<void*>(ws), V, F);
    ProfScope prof(PROF_VAE_MISC, st);
    const long long n3 = 3 * F;
    if (V || F) {
        split_verts_kernel<<<blocks(V > n3 ? V : n3), MS_THREADS, 0, st>>>(verts, V, w.edges, w.hdr, F ? n3 : 0, w.eflag, w.epos, verts_out);
        TPX_LAUNCH_CHECK();
    }
    if (F) {
        split_faces_kernel<<<blocks(F), MS_THREADS, 0, st>>>(w.T[0], F, w.edges, w.hdr, w.eflag, w.epos, V, verts_out, w.fpos, reinterpret_cast<long long*>(faces_out));
        TPX_LAUNCH_CHECK();
    }
    if (nC) {
        split_creases_kernel<<<blocks(nC), MS_THREADS, 0, st>>>(creases, nC, w.edges, w.hdr, w.eflag, w.epos, V, w.cpos, w.hk[0]);
        TPX_LAUNCH_CHECK();
        cub::DoubleBuffer<u64> dc(w.hk[0], w.hk[1]);
        size_t b = w.cub_bytes;
        TPX_CUDA(cub::DeviceRadixSort::SortKeys(w.cub, b, dc, nC_out, 0, 64, st));
        TPX_CUDA(cudaMemcpyAsync(creases_out, dc.Current(), nC_out * sizeof(u64), cudaMemcpyDeviceToDevice, st));
    }
    return TPX_OK;
}

int tpx_remesh_relax(float* verts, int64_t V, int64_t* faces_dev, int64_t F, const int64_t* creases_dev, int64_t nC, const float* verts0, int64_t V0,
                     int64_t F0, const void* grid, size_t grid_bytes, double target_len, double cos_feature, void* ws, size_t ws_bytes,
                     int64_t* counts_dev, void* stream) {
    long long* faces = reinterpret_cast<long long*>(faces_dev);
    const u64* creases = reinterpret_cast<const u64*>(creases_dev);
    long long* counts = reinterpret_cast<long long*>(counts_dev);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = mesh_args("remesh relax", verts, V, faces, F, ws, ws_bytes, tpx_remesh_workspace_bytes(V, F));
    if (rc == TPX_OK) rc = crease_arg(creases_dev, nC, F);
    if (rc != TPX_OK) return rc;
    TPX_CHECK(counts != nullptr && target_len > 0.0 && isfinite(target_len) && cos_feature >= -1.0 && cos_feature <= 1.0, TPX_ERR_ARG,
              "remesh relax: null counts, target length %g or cos(feature angle) %g", target_len, cos_feature);
    TPX_CHECK(V0 >= 0 && F0 >= 0 && (verts0 != nullptr || V0 == 0) && (V0 > 0 || F0 == 0) && grid != nullptr &&
                  grid_bytes >= tpx_remesh_grid_bytes(F0) && tpx_remesh_grid_bytes(F0) > 0,
              TPX_ERR_ARG, "remesh relax: bad input mesh or grid");
    TPX_DEVICE_GUARD();
    const RmWs w = rm_layout(ws, V, F);
    const GridWs g = grid_layout(const_cast<void*>(grid), F0);
    rc = rm_cub_check("remesh relax", F, -1, w.cub_bytes, 0);
    if (rc != TPX_OK) return rc;
    ProfScope prof(PROF_VAE_MISC, st);
    const double lo = target_len * 0.8, hi = target_len * (4.0 / 3.0), lo2 = lo * lo, hi2 = hi * hi;
    TPX_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(DecHdr), st));
    if (V) {
        iota_kernel<<<blocks(V), MS_THREADS, 0, st>>>(w.rep, V);
        TPX_LAUNCH_CHECK();
    }
    long long Fc = F, rounds[2] = {0, 0};
    int buf = 0;
    DecHdr h;
    if (F) {
        faces_in_kernel<<<blocks(F), MS_THREADS, 0, st>>>(faces, F, V, w.T[0], &w.hdr->bad);
        TPX_LAUNCH_CHECK();
        rc = read_hdr(w, &h, st);
        if (rc != TPX_OK) return rc;
        TPX_CHECK(h.bad == 0, TPX_ERR_ARG, "remesh relax: %d faces have an index outside [0, %lld) or a repeated index", h.bad, (long long)V);
    }
    const u64* ck = nullptr;
    // collapse rounds
    while (Fc > 0) {
        const long long n3 = 3 * Fc;
        int* T = w.T[buf];
        rc = topology(w, T, Fc, V, creases, nC, st, &ck);
        if (rc != TPX_OK) return rc;
        TPX_CUDA(cudaMemsetAsync(w.m1, 0xff, V * sizeof(u64), st));
        TPX_CUDA(cudaMemsetAsync(&w.hdr->n_acc, 0, sizeof(int), st));
        collapse_cost_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, verts, T, ck, w.vstart, w.vend, w.feat, w.deg, lo2, hi2, w.ekey, w.xbar, w.m1);
        TPX_LAUNCH_CHECK();
        TPX_CUDA(cudaMemcpyAsync(w.m2, w.m1, V * sizeof(u64), cudaMemcpyDeviceToDevice, st));
        edge_min2_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, w.m1, w.m2);
        TPX_LAUNCH_CHECK();
        edge_accept_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, w.ekey, w.m2, w.aflag);
        TPX_LAUNCH_CHECK();
        rc = read_hdr(w, &h, st);                                         // the one readback of the round
        if (rc != TPX_OK) return rc;
        rc = face_count_check(h, Fc, rounds[0]);
        if (rc != TPX_OK) return rc;
        if (h.n_acc == 0) break;
        collapse_apply_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, w.aflag, w.xbar, w.feat, verts, w.rep);
        TPX_LAUNCH_CHECK();
        remap_kernel<<<blocks(Fc), MS_THREADS, 0, st>>>(T, Fc, w.rep, w.fkeep);
        TPX_LAUNCH_CHECK();
        rc = scan(w.fkeep, w.fpos, Fc, w.cub, w.cub_bytes, st);
        if (rc != TPX_OK) return rc;
        compact_faces_kernel<<<blocks(Fc), MS_THREADS, 0, st>>>(T, Fc, w.fkeep, w.fpos, w.T[buf ^ 1], w.hdr, buf ^ 1);
        TPX_LAUNCH_CHECK();
        buf ^= 1;
        Fc -= 2LL * h.n_acc;                                              // the two faces on each collapsed edge; checked against hdr->F
        ++rounds[0];
    }
    if (rounds[0] > 0 && Fc == 0) {                                       // the loop ended without reading the last compaction back
        rc = read_hdr(w, &h, st);
        if (rc == TPX_OK) rc = face_count_check(h, Fc, rounds[0]);
        if (rc != TPX_OK) return rc;
    }
    // flip rounds
    while (Fc > 0) {
        const long long n3 = 3 * Fc;
        int* T = w.T[buf];
        rc = topology(w, T, Fc, V, creases, nC, st, &ck);
        if (rc != TPX_OK) return rc;
        TPX_CUDA(cudaMemsetAsync(w.m1, 0xff, V * sizeof(u64), st));
        TPX_CUDA(cudaMemsetAsync(&w.hdr->n_acc, 0, sizeof(int), st));
        flip_cost_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, verts, T, ck, w.vstart, w.vend, w.frozen, w.deg, creases, nC, cos_feature, w.ekey, w.m1);
        TPX_LAUNCH_CHECK();
        flip_accept_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, T, ck, w.vstart, w.vend, w.frozen, w.ekey, w.m1, w.aflag);
        TPX_LAUNCH_CHECK();
        rc = read_hdr(w, &h, st);
        if (rc != TPX_OK) return rc;
        rc = face_count_check(h, Fc, rounds[0]);
        if (rc != TPX_OK) return rc;
        if (h.n_acc == 0) break;
        flip_apply_kernel<<<blocks(n3), MS_THREADS, 0, st>>>(w.edges, w.hdr, T, ck, w.vstart, w.vend, w.frozen, w.aflag);
        TPX_LAUNCH_CHECK();
        ++rounds[1];
    }
    // smoothing (Jacobi: every move from the old positions) and projection of the non-feature vertices onto the input
    if (Fc > 0) {
        rc = topology(w, w.T[buf], Fc, V, creases, nC, st, &ck);
        if (rc != TPX_OK) return rc;
        smooth_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, w.T[buf], ck, w.vstart, w.vend, w.feat, V, w.P2);
        TPX_LAUNCH_CHECK();
        TPX_CUDA(cudaMemcpyAsync(verts, w.P2, 3 * V * sizeof(float), cudaMemcpyDeviceToDevice, st));
        if (F0) {
            project_kernel<<<blocks(V), MS_THREADS, 0, st>>>(verts, verts, V, w.feat, verts0, g.T, g.hdr, g.cstart, g.cend, g.key[0], nullptr);
            TPX_LAUNCH_CHECK();
        }
        faces_out_kernel<<<blocks(3 * Fc), MS_THREADS, 0, st>>>(w.T[buf], Fc, faces);
        TPX_LAUNCH_CHECK();
    }
    const long long out[3] = {Fc, rounds[0], rounds[1]};
    TPX_CUDA(cudaMemcpyAsync(counts, out, sizeof(out), cudaMemcpyHostToDevice, st));
    TPX_CUDA(cudaStreamSynchronize(st));                                  // `out` lives on this stack frame
    return TPX_OK;
}

}  // extern "C"
