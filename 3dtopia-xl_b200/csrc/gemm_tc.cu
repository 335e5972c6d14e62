// Host launcher for the wgmma GEMM: tensor-map construction (cached), tile-shape dispatch, and the linear-GEMM entry points.
#include "gemm_tc.cuh"

#include <map>
#include <mutex>
#include <tuple>

namespace tpx {

// ---- tensor maps ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

static CUtensorMapSwizzle swizzle_for(int bk) {
    return bk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

using MapKey = std::tuple<const void*, long long, long long, long long, int, int, int>;   // last: rank (2 / 5) * 16 + element bytes
static std::map<MapKey, CUtensorMap> g_maps;
static std::mutex g_maps_mu;

// 2-D: row-major [rows, K] matrix of fp16 (esz 2) or fp32 (esz 4) elements, box = [box_rows, bk], swizzle = box row bytes (128/64/32)
static int map_2d(const void* ptr, long long rows, long long K, long long ld, int box_rows, int bk, CUtensorMap* out, int esz = 2, bool swizzled = true) {
    MapKey key{ptr, rows, K, ld, box_rows, bk, 2 * 16 + esz + (swizzled ? 0 : 8)};
    std::lock_guard<std::mutex> lk(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return TPX_OK; }
    EncodeTiledFn enc = encode_fn();
    TPX_CHECK(enc != nullptr, TPX_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no driver?)");
    TPX_CHECK((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (ld * esz) % 16 == 0, TPX_ERR_ARG,
              "TMA operand must be 16-B aligned (ptr %p, row stride %lld elements of %d bytes)", ptr, ld, esz);
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
    cuuint64_t gstr[1] = {static_cast<cuuint64_t>(ld) * esz};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(bk), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, esz == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swizzled ? swizzle_for(bk * esz / 2) : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TPX_CHECK(r == CUDA_SUCCESS, TPX_ERR_CUDA, "cuTensorMapEncodeTiled(2d) failed: %d (rows %lld K %lld ld %lld box %d x %d)", (int)r, rows, K, ld, box_rows, bk);
    if (g_maps.size() > 4096) g_maps.clear();
    g_maps[key] = m;
    *out = m;
    return TPX_OK;
}

// 5-D: channels-last volume [P, S, S, S, C] fp16; box = 128 voxel rows x bk channels
static int map_conv(const void* ptr, long long P, int S, int C, int bk, CUtensorMap* out) {
    MapKey key{ptr, P, S, C, 0, bk, 5 * 16 + 2};
    std::lock_guard<std::mutex> lk(g_maps_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) { *out = it->second; return TPX_OK; }
    EncodeTiledFn enc = encode_fn();
    TPX_CHECK(enc != nullptr, TPX_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no driver?)");
    TPX_CHECK(S == 4 || S == 8, TPX_ERR_SHAPE, "conv volume edge must be 4 or 8, got %d", S);
    cuuint64_t gdim[5] = {(cuuint64_t)C, (cuuint64_t)S, (cuuint64_t)S, (cuuint64_t)S, (cuuint64_t)P};
    cuuint64_t gstr[4] = {(cuuint64_t)C * 2, (cuuint64_t)S * C * 2, (cuuint64_t)S * S * C * 2, (cuuint64_t)S * S * S * C * 2};
    cuuint32_t box[5] = {(cuuint32_t)bk, (cuuint32_t)S, (cuuint32_t)S, (cuuint32_t)(S == 4 ? 4 : 2), (cuuint32_t)(S == 4 ? 2 : 1)};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUtensorMap m;
    CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle_for(bk), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TPX_CHECK(r == CUDA_SUCCESS, TPX_ERR_CUDA, "cuTensorMapEncodeTiled(5d) failed: %d (P %lld S %d C %d bk %d)", (int)r, P, S, C, bk);
    if (g_maps.size() > 4096) g_maps.clear();
    g_maps[key] = m;
    *out = m;
    return TPX_OK;
}

// General fp16 tensor map (rank <= 5, dims / strides innermost first, strides in bytes for dims 1..rank-1); not cached.
int make_tensor_map_nd(const void* ptr, int rank, const long long* dims, const long long* strides_bytes, const int* box, int swizzle_bytes,
                       CUtensorMap* out, int l2_promotion_bytes) {
    EncodeTiledFn enc = encode_fn();
    TPX_CHECK(enc != nullptr, TPX_ERR_CUDA, "cuTensorMapEncodeTiled unavailable (no driver?)");
    TPX_CHECK(rank >= 1 && rank <= 5 && (reinterpret_cast<uintptr_t>(ptr) & 15) == 0, TPX_ERR_ARG, "tensor map: rank %d / unaligned base", rank);
    cuuint64_t gdim[5];
    cuuint64_t gstr[4];
    cuuint32_t bx[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdim[i] = static_cast<cuuint64_t>(dims[i]);
        bx[i] = static_cast<cuuint32_t>(box[i]);
        estr[i] = 1;
        if (i > 0) {
            TPX_CHECK(strides_bytes[i - 1] % 16 == 0, TPX_ERR_ARG, "tensor map: stride %lld of dim %d is not a multiple of 16 bytes", strides_bytes[i - 1], i);
            gstr[i - 1] = static_cast<cuuint64_t>(strides_bytes[i - 1]);
        }
    }
    const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                  : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                        : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(ptr), gdim, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                     l2_promotion_bytes >= 256  ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                     : l2_promotion_bytes >= 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B
                     : l2_promotion_bytes >= 64  ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
                                                 : CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    TPX_CHECK(r == CUDA_SUCCESS, TPX_ERR_CUDA, "cuTensorMapEncodeTiled(rank %d) failed: %d", rank, static_cast<int>(r));
    return TPX_OK;
}

int make_tensor_map_2d(const void* ptr, long long rows, long long cols, long long ld, int box_rows, int box_cols, CUtensorMap* out) {
    return map_2d(ptr, rows, cols, ld, box_rows, box_cols, out);
}

// The geometry the 24-column head-split bulk stores need at tile width bn (EPI_HEADS with heads_tma requested).
static bool heads_bulk_ok(const GemmProblem& p, const GemmArgs& a, int bn) {
    return p.epi == EPI_HEADS && a.heads_tma != 0 && p.a_mode == AMODE_LINEAR && gemm_wn(bn, p.a_mode) % 24 == 0 && p.N % bn == 0 && a.Dh % 24 == 0 &&
           a.split_cols % 24 == 0 && a.Nseq % 32 == 0 && a.Nseq > 0 && p.M % a.Nseq == 0 && a.DhP % 8 == 0 && (a.vt_which_plus1 == 0 || a.vt_ld % 8 == 0);
}

// Automatic tile width of a linear GEMM: minimise rounds x width over the ping-pong widths {128, 144}, rounds = ceil(tiles / SMs), so
// the last round leaves few SMs idle; 144 (two 72-wide heads, divides 1152 / 3456 / 4608) only where its epilogue is a bulk one (gated
// residual; head split in 24-column groups).  Ties go to 144 (fewer tiles: less operand re-read).
int gemm_pick_bn(const GemmProblem& p) {
    const long sms = gemm_num_sms();
    const long tm = (p.M + 127) / 128;
    int best = 128;
    long best_cost = -1;
    for (int bn : {128, 144}) {
        if (bn == 144 && !gemm_tma_epilogue(p.epi, bn) && !heads_bulk_ok(p, p.args, bn)) continue;
        const long tiles = tm * ((p.N + bn - 1) / bn);
        const long cost = ((tiles + sms - 1) / sms) * bn;
        if (best_cost < 0 || cost <= best_cost) { best = bn; best_cost = cost; }
    }
    return best;
}

// Output tensor maps of the bulk-store epilogues (tc / td / te default to copies of the A map when unused).  Validates the geometry the
// 24-column head-split stores need and clears a.heads_tma when it does not hold (the kernel then takes the per-thread path).
static int make_output_maps(const GemmProblem& p, GemmArgs& a, const CUtensorMap& ta, CUtensorMap& tc, CUtensorMap& td, CUtensorMap& te) {
    int rc = TPX_OK;
    tc = ta; td = ta; te = ta;
    if (p.epi == EPI_HEADS && a.heads_tma != 0) {
        const bool ok = heads_bulk_ok(p, a, p.BN);
        a.heads_tma = ok ? 1 : 0;
        if (ok) {
            const long long rows = static_cast<long long>(p.M / a.Nseq) * a.H * a.Nseq, rows_t = static_cast<long long>(p.M / a.Nseq) * a.H * a.DhP;
            __half* outs[3] = {a.out0, a.out1, a.out2};
            CUtensorMap* maps[3] = {&tc, &td, &te};
            const int nwhich = p.N / a.split_cols;
            for (int w = 0; w < nwhich && w < 3; ++w) {
                TPX_CHECK(outs[w] != nullptr, TPX_ERR_ARG, "gemm: head-split output %d is null", w);
                if (w + 1 == a.vt_which_plus1) rc = map_2d(outs[w], rows_t, a.vt_ld, a.vt_ld, 24, 32, maps[w], 2, false);
                else rc = map_2d(outs[w], rows, a.DhP, a.DhP, 32, 24, maps[w], 2, false);
                if (rc != TPX_OK) return rc;
            }
        }
    } else {
        a.heads_tma = 0;
    }
    const int wn = gemm_wn(p.BN, p.a_mode);
    if (gemm_tma_epilogue(p.epi, wn)) {
        // fp16 [M, N] in 64-column x 32-row boxes, or the fp32 residual in 32 x 32 boxes (+ 16 x 32 for the last 16 columns of a 144 tile)
        if (p.epi == EPI_GATED) {
            TPX_CHECK(a.xres != nullptr && a.gate != nullptr, TPX_ERR_ARG, "gemm: gated epilogue without residual / gate");
            rc = map_2d(a.xres, p.M, p.N, a.ldx, 32, 32, &tc, 4);
            if (rc == TPX_OK && wn % 32 != 0) rc = map_2d(a.xres, p.M, p.N, a.ldx, 32, 16, &td, 4);
        } else if (a.convt_store != 0) {
            // out0 already points at the (a,b,c) corner of the [P, 8, 8, 8, N] volume: the stride-2 sub-lattice as a 5-D tensor
            TPX_CHECK(a.out0 != nullptr && p.M % 64 == 0 && p.epi == EPI_STORE, TPX_ERR_ARG, "gemm: transposed-conv store needs EPI_STORE and M = P * 64");
            const long long C = p.N, dims[5] = {C, 4, 4, 4, p.M / 64};
            const long long strides[4] = {2 * C * 2, 16 * C * 2, 128 * C * 2, 512 * C * 2};
            const int box[5] = {64, 4, 4, 2, 1};
            rc = make_tensor_map_nd(a.out0, 5, dims, strides, box, 128, &tc, 256);
        } else {
            TPX_CHECK(a.out0 != nullptr && a.ldo >= p.N, TPX_ERR_ARG, "gemm: output pointer / row stride (%d < N %d)", a.ldo, p.N);
            rc = map_2d(a.out0, p.M, p.N, a.ldo, 32, 64, &tc, 2);
        }
    }
    return rc;
}

// Every instantiated (tile width, k-block, A mode, epilogue); a combination not listed has no kernel.
#define TPX_GEMM_INSTANCES(X) \
    /* DiT (every tile width x every DiT epilogue, so any hidden size that is a multiple of 128 works); 128 / 144: ping-pong schedule */ \
    X(128, 64, AMODE_LINEAR, EPI_STORE) \
    X(128, 64, AMODE_LINEAR, EPI_GELU) \
    X(128, 64, AMODE_LINEAR, EPI_HEADS) \
    X(128, 64, AMODE_LINEAR, EPI_GATED) \
    X(144, 64, AMODE_LINEAR, EPI_STORE) \
    X(144, 64, AMODE_LINEAR, EPI_GELU) \
    X(144, 64, AMODE_LINEAR, EPI_HEADS) \
    X(144, 64, AMODE_LINEAR, EPI_GATED) \
    X(192, 64, AMODE_LINEAR, EPI_STORE) \
    X(192, 64, AMODE_LINEAR, EPI_GELU) \
    X(192, 64, AMODE_LINEAR, EPI_HEADS) \
    X(192, 64, AMODE_LINEAR, EPI_GATED) \
    X(256, 64, AMODE_LINEAR, EPI_STORE) \
    X(256, 64, AMODE_LINEAR, EPI_GELU) \
    X(256, 64, AMODE_LINEAR, EPI_HEADS) \
    X(256, 64, AMODE_LINEAR, EPI_GATED) \
    /* VAE */ \
    X(256, 64, AMODE_CONV3, EPI_STORE) \
    X(256, 64, AMODE_CONV3, EPI_RESID_SCALE) \
    X(256, 64, AMODE_LINEAR, EPI_RESID_SCALE) \
    X(32, 64, AMODE_CONV3, EPI_STORE) \
    X(32, 64, AMODE_LINEAR, EPI_STORE) \
    X(32, 32, AMODE_CONV3, EPI_STORE) \
    X(32, 32, AMODE_CONV3, EPI_RESID_SCALE) \
    X(16, 32, AMODE_CONV3, EPI_NCDHW) \
    /* VAE encoder: conv1 of the 32 -> 256 block at 4^3 and its K = 32 shortcut; conv_out (2 of 16 rows) + quant_conv */ \
    X(256, 32, AMODE_CONV3, EPI_STORE) \
    X(256, 32, AMODE_LINEAR, EPI_STORE) \
    X(16, 64, AMODE_CONV3, EPI_MOMENTS)

static bool gemm_has_kernel(int bn, int bk, int amode, int epi) {
#define TPX_HAS(BN_, BK_, AM_, EP_) \
    if (bn == BN_ && bk == BK_ && amode == AM_ && epi == EP_) return true;
    TPX_GEMM_INSTANCES(TPX_HAS)
#undef TPX_HAS
    return false;
}

// k-block depth: 32-channel conv operands load 64-B rows; a linear K of 32 does too where a BK = 32 kernel exists for its tile and
// epilogue (the VAE encoder's 1x1 shortcut), and otherwise runs the BK = 64 kernel, the TMA zero-filling columns 32..63 of each row.
static int gemm_bk(const GemmProblem& p) {
    if (p.a_mode == AMODE_CONV3) return p.conv_C == 32 ? 32 : 64;
    return p.K == 32 && gemm_has_kernel(p.BN, 32, p.a_mode, p.epi) ? 32 : 64;
}

template <int BN, int BK, int AMODE, int EPI>
static int launch_one(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& td, const CUtensorMap& te, const GemmArgs& a,
                      cudaStream_t stream) {
    using Cfg = GemmCfg<BN, BK, AMODE>;
    GemmArgs ka = a;
    ka.tiles_n = (a.N + BN - 1) / BN;
    ka.num_tiles = ((a.M + 127) / 128) * ka.tiles_n;
    auto kern = gemm_tc_kernel<BN, BK, AMODE, EPI>;
    static bool attr_set = false;
    if (!attr_set) {
        TPX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_set = true;
    }
    const int grid = ka.num_tiles < gemm_num_sms() ? ka.num_tiles : gemm_num_sms();
    TPX_CUDA(launch_pdl(kern, dim3(grid), dim3(Cfg::THREADS), Cfg::SMEM_BYTES, stream, ta, tb, tc, td, te, ka));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int launch_gemm(const GemmProblem& p, cudaStream_t stream) {
    TPX_CHECK(p.M > 0 && p.N > 0 && p.K > 0, TPX_ERR_SHAPE, "gemm: empty problem %d x %d x %d", p.M, p.N, p.K);
    TPX_CHECK(p.N % 8 == 0 && p.K % 8 == 0, TPX_ERR_SHAPE, "gemm: N (%d) and K (%d) must be multiples of 8", p.N, p.K);
    const int bk = gemm_bk(p);
    TPX_CHECK(gemm_has_kernel(p.BN, bk, p.a_mode, p.epi), TPX_ERR_SHAPE, "gemm: no kernel instantiated for BN=%d BK=%d amode=%d epi=%d", p.BN, bk,
              p.a_mode, p.epi);
    ProfScope prof(p.a_mode == AMODE_CONV3 ? PROF_CONV_GEMM : PROF_GEMM, stream);
    GemmArgs a = p.args;
    a.M = p.M;
    a.N = p.N;
    a.num_kb = (p.K + bk - 1) / bk;
    a.conv_S = p.conv_S;
    a.chunks_per_tap = p.a_mode == AMODE_CONV3 ? p.conv_C / bk : 1;
    CUtensorMap ta, tb;
    int rc;
    if (p.a_mode == AMODE_LINEAR) {
        rc = map_2d(p.A, p.M, p.K, p.lda, 128, bk, &ta);
    } else {
        TPX_CHECK(p.conv_C % bk == 0 && p.K == 27 * p.conv_C, TPX_ERR_SHAPE, "conv gemm: K (%d) must be 27*C (%d)", p.K, p.conv_C);
        const int s3 = p.conv_S * p.conv_S * p.conv_S;
        TPX_CHECK(p.M % s3 == 0, TPX_ERR_SHAPE, "conv gemm: M (%d) must be P*S^3", p.M);
        rc = map_conv(p.A, p.M / s3, p.conv_S, p.conv_C, bk, &ta);
    }
    if (rc != TPX_OK) return rc;
    rc = map_2d(p.W, p.N, p.K, p.K, p.BN, bk, &tb);
    if (rc != TPX_OK) return rc;
    CUtensorMap tc, td, te;
    rc = make_output_maps(p, a, ta, tc, td, te);
    if (rc != TPX_OK) return rc;

#define TPX_CASE(BN_, BK_, AM_, EP_) \
    if (p.BN == BN_ && bk == BK_ && p.a_mode == AM_ && p.epi == EP_) return launch_one<BN_, BK_, AM_, EP_>(ta, tb, tc, td, te, a, stream);
    TPX_GEMM_INSTANCES(TPX_CASE)
#undef TPX_CASE
    set_error("gemm: no kernel instantiated for BN=%d BK=%d amode=%d epi=%d", p.BN, bk, p.a_mode, p.epi);   // unreachable: checked above
    return TPX_ERR_SHAPE;
}

// The problem of a linear GEMM, with the checks launch_gemm makes before it touches anything: a bad shape or tile width fails here,
// before any launch (the head-split entry clears its outputs only after this).
static int linear_problem(const __half* A, int lda, const __half* W, int M, int N, int K, int epi, const GemmArgs& args, int tile_n, GemmProblem& p) {
    p = GemmProblem{};
    p.A = A; p.a_mode = AMODE_LINEAR; p.lda = lda; p.W = W; p.M = M; p.N = N; p.K = K;
    p.epi = epi; p.args = args;
    TPX_CHECK(tile_n >= 0, TPX_ERR_ARG, "gemm: tile width %d (0 = automatic, or one of the instantiated widths)", tile_n);
    TPX_CHECK(M > 0 && N > 0 && K > 0, TPX_ERR_SHAPE, "gemm: empty problem %d x %d x %d", M, N, K);
    TPX_CHECK(N % 8 == 0 && K % 8 == 0, TPX_ERR_SHAPE, "gemm: N (%d) and K (%d) must be multiples of 8", N, K);
    p.BN = tile_n > 0 ? tile_n : gemm_pick_bn(p);
    const int bk = gemm_bk(p);
    TPX_CHECK(gemm_has_kernel(p.BN, bk, p.a_mode, p.epi), TPX_ERR_SHAPE, "gemm: no kernel instantiated for BN=%d BK=%d amode=%d epi=%d", p.BN, bk,
              p.a_mode, p.epi);
    return TPX_OK;
}

int gemm_linear(const __half* A, int lda, const __half* W, int M, int N, int K, int epi, const GemmArgs& args, int tile_n, cudaStream_t st) {
    GemmProblem p;
    const int rc = linear_problem(A, lda, W, M, N, K, epi, args, tile_n, p);
    if (rc != TPX_OK) return rc;
    return launch_gemm(p, st);
}

}  // namespace tpx

using namespace tpx;

extern "C" {

int tpx_linear(const void* A, int lda, const void* W, const void* bias, void* out, int ldo, int M, int N, int K, int act, float post_scale, int tile_n,
               void* stream) {
    TPX_CHECK(A != nullptr && W != nullptr && out != nullptr, TPX_ERR_ARG, "linear: null argument");
    TPX_DEVICE_GUARD();
    GemmArgs a{};
    a.bias = static_cast<const __half*>(bias); a.post_scale = post_scale; a.out0 = static_cast<__half*>(out); a.ldo = ldo;
    return gemm_linear(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), M, N, K, act ? EPI_GELU : EPI_STORE, a, tile_n,
                       static_cast<cudaStream_t>(stream));
}

int tpx_linear_gated(const void* A, int lda, const void* W, const void* bias, const void* gate, int gate_bstride, int gate_batches, int rows_per_batch,
                     float* xres, int ldx, int M, int N, int K, int tile_n, void* stream) {
    TPX_CHECK(A != nullptr && W != nullptr && gate != nullptr && xres != nullptr, TPX_ERR_ARG, "linear_gated: null argument");
    TPX_CHECK(gate_batches > 0 && rows_per_batch > 0, TPX_ERR_ARG, "linear_gated: bad gate batching");
    TPX_DEVICE_GUARD();
    GemmArgs a{};
    a.bias = static_cast<const __half*>(bias); a.post_scale = 1.0f; a.xres = xres; a.ldx = ldx;
    a.gate = static_cast<const __half*>(gate); a.gate_bstride = gate_bstride; a.rows_per_batch = rows_per_batch; a.gate_batches = gate_batches;
    return gemm_linear(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), M, N, K, EPI_GATED, a, tile_n, static_cast<cudaStream_t>(stream));
}

int tpx_linear_heads(const void* A, int lda, const void* W, const void* bias, void* out0, void* out1, void* out2, int M, int N, int K, int split_cols,
                     int H, int Dh, int DhP, int n_seq_tokens, float post_scale, int tile_n, int transposed_which, int transposed_ld, void* stream) {
    TPX_CHECK(A != nullptr && W != nullptr && out0 != nullptr, TPX_ERR_ARG, "linear_heads: null argument");
    TPX_CHECK(Dh % 8 == 0 && DhP % 8 == 0 && DhP >= Dh && split_cols == H * Dh && N % split_cols == 0, TPX_ERR_SHAPE, "linear_heads: bad head geometry");
    TPX_DEVICE_GUARD();
    GemmArgs a{};
    a.bias = static_cast<const __half*>(bias); a.post_scale = post_scale;
    a.out0 = static_cast<__half*>(out0); a.out1 = static_cast<__half*>(out1); a.out2 = static_cast<__half*>(out2);
    a.split_cols = split_cols; a.Dh = Dh; a.DhP = DhP; a.H = H; a.Nseq = n_seq_tokens;
    a.vt_which_plus1 = transposed_which >= 0 ? transposed_which + 1 : 0;
    a.vt_ld = transposed_ld;
    TPX_CHECK(n_seq_tokens > 0 && M % n_seq_tokens == 0, TPX_ERR_SHAPE, "linear_heads: M (%d) must be a whole number of %d-token sequences", M,
              n_seq_tokens);
    TPX_CHECK(transposed_which < 0 || transposed_ld >= n_seq_tokens, TPX_ERR_SHAPE, "linear_heads: transposed row length %d < %d tokens", transposed_ld,
              n_seq_tokens);
    const bool bulk = Dh % 24 == 0 && n_seq_tokens % 32 == 0;
    a.heads_tma = bulk ? 1 : 0;
    GemmProblem p;
    const int rc = linear_problem(static_cast<const __half*>(A), lda, static_cast<const __half*>(W), M, N, K, EPI_HEADS, a, tile_n, p);
    if (rc != TPX_OK) return rc;
    if (bulk) {
        // bulk-store epilogue: it writes the Dh real columns of the n_seq tokens only, so the padding is cleared here (the DiT forward
        // clears its workspace once per call instead).  The per-thread epilogue writes the padding itself.
        void* outs[3] = {out0, out1, out2};
        const size_t per = static_cast<size_t>(M / n_seq_tokens) * H * n_seq_tokens * DhP * 2;
        for (int w = 0; w < N / split_cols && w < 3; ++w) {
            TPX_CHECK(outs[w] != nullptr, TPX_ERR_ARG, "linear_heads: output %d is null", w);
            const size_t bytes = w == transposed_which ? static_cast<size_t>(M / n_seq_tokens) * H * DhP * transposed_ld * 2 : per;
            TPX_CUDA(cudaMemsetAsync(outs[w], 0, bytes, static_cast<cudaStream_t>(stream)));
        }
    }
    return launch_gemm(p, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
