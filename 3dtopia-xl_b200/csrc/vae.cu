// VAE decoder handle: repacked fp16 parameters keyed by the reference's state_dict names and the decode schedule.
//   reference: models/vae3d_dib.py:437-440 (VAE.decode), :369-387 (Decoder.forward), :220-226 (MidBlock),
//              :259-267 (UpBlock), :128-145 (ResnetBlock), :34-48 (VolumeAttention)
// Activations are channels-last fp16 [P, S^3, C]; every primitive is independent (GroupNorm statistics are
// per primitive), so the whole decoder is a batch of P tiny volumes.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "kernels.cuh"

using namespace tpx;

struct VaeRes {
    int cin, cout;
    __half *n1g, *n1b, *W1, *b1, *n2g, *n2b, *W2, *b2, *Wsc, *bsc;  // Wsc null when cin == cout
};

struct tpx_vae {
    int C0, C1, Cout, heads;
    __half* store = nullptr;
    size_t store_halves = 0;
    __half *w_pq, *b_pq, *Win, *bin;
    VaeRes res[6];                           // mid0, mid1, up0.0, up0.1, up1.0, up1.1
    __half *ang, *anb, *Wqkv, *Wap, *bap;    // mid attention
    __half *Wup, *bup;                       // [8*C0, C0], [8*C0]
    __half *nog, *nob, *Wout, *bout;         // norm_out, conv_out (padded to 16 rows)
    std::vector<std::string> required;
    std::vector<uint8_t> seen;
    bool finalized = false;
};

namespace {
const char* kResPrefix[6] = {"decoder.mid_block.nets.0.", "decoder.mid_block.nets.1.", "decoder.up_blocks.0.nets.0.", "decoder.up_blocks.0.nets.1.",
                             "decoder.up_blocks.1.nets.0.", "decoder.up_blocks.1.nets.1."};

struct HCarver {
    __half* base;
    size_t off = 0;
    __half* take(size_t n) {
        __half* p = base == nullptr ? nullptr : base + off;
        off += (n + 63) & ~static_cast<size_t>(63);   // 128-B slots (TMA operands need 16-B alignment)
        return p;
    }
};

void carve(tpx_vae* h, __half* base) {
    HCarver c{base};
    const size_t C0 = h->C0, C1 = h->C1;
    h->w_pq = c.take(8); h->b_pq = c.take(8);
    h->Win = c.take(C0 * 27); h->bin = c.take(C0);
    for (int i = 0; i < 6; ++i) {
        VaeRes& r = h->res[i];
        r.cin = i < 4 ? h->C0 : (i == 4 ? h->C0 : h->C1);
        r.cout = i < 4 ? h->C0 : h->C1;
        r.n1g = c.take(r.cin); r.n1b = c.take(r.cin);
        r.W1 = c.take(static_cast<size_t>(r.cout) * 27 * r.cin); r.b1 = c.take(r.cout);
        r.n2g = c.take(r.cout); r.n2b = c.take(r.cout);
        r.W2 = c.take(static_cast<size_t>(r.cout) * 27 * r.cout); r.b2 = c.take(r.cout);
        if (r.cin != r.cout) { r.Wsc = c.take(static_cast<size_t>(r.cout) * r.cin); r.bsc = c.take(r.cout); }
        else { r.Wsc = nullptr; r.bsc = nullptr; }
    }
    h->ang = c.take(C0); h->anb = c.take(C0);
    h->Wqkv = c.take(3 * C0 * C0); h->Wap = c.take(C0 * C0); h->bap = c.take(C0);
    h->Wup = c.take(8 * C0 * C0); h->bup = c.take(8 * C0);
    h->nog = c.take(C1); h->nob = c.take(C1);
    h->Wout = c.take(16 * 27 * C1); h->bout = c.take(16);
    h->store_halves = c.off;
}

enum SlotKind { SK_PLAIN, SK_CONV3, SK_CONV3_T, SK_CONVT2, SK_BIAS_REP8 };
struct VSlot {
    __half* ptr;
    SlotKind kind;
    std::vector<int64_t> shape;
    int a, b;  // conv dims (Cout, Cin) or (Cin, Cout)
};

bool find_vslot(tpx_vae* h, const std::string& key, VSlot* s) {
    const int64_t C0 = h->C0, C1 = h->C1;
    auto plain = [&](__half* p, std::vector<int64_t> shp) { *s = VSlot{p, SK_PLAIN, shp, 0, 0}; return true; };
    if (key == "post_quant_conv.weight") return plain(h->w_pq, {1, 1, 1, 1, 1});
    if (key == "post_quant_conv.bias") return plain(h->b_pq, {1});
    if (key == "decoder.conv_in.weight") return plain(h->Win, {C0, 1, 3, 3, 3});
    if (key == "decoder.conv_in.bias") return plain(h->bin, {C0});
    if (key == "decoder.norm_out.weight") return plain(h->nog, {C1});
    if (key == "decoder.norm_out.bias") return plain(h->nob, {C1});
    if (key == "decoder.conv_out.weight") { *s = VSlot{h->Wout, SK_CONV3_T, {C1, h->Cout, 3, 3, 3}, h->Cout, static_cast<int>(C1)}; return true; }
    if (key == "decoder.conv_out.bias") return plain(h->bout, {h->Cout});
    if (key == "decoder.up_blocks.0.upsample.weight") { *s = VSlot{h->Wup, SK_CONVT2, {C0, C0, 2, 2, 2}, static_cast<int>(C0), static_cast<int>(C0)}; return true; }
    if (key == "decoder.up_blocks.0.upsample.bias") { *s = VSlot{h->bup, SK_BIAS_REP8, {C0}, static_cast<int>(C0), 0}; return true; }
    const std::string a = "decoder.mid_block.attns.0.";
    if (key == a + "norm.weight") return plain(h->ang, {C0});
    if (key == a + "norm.bias") return plain(h->anb, {C0});
    if (key == a + "attn.qkv.weight") return plain(h->Wqkv, {3 * C0, C0});
    if (key == a + "attn.proj.weight") return plain(h->Wap, {C0, C0});
    if (key == a + "attn.proj.bias") return plain(h->bap, {C0});
    for (int i = 0; i < 6; ++i) {
        const std::string p = kResPrefix[i];
        if (key.rfind(p, 0) != 0) continue;
        VaeRes& r = h->res[i];
        const std::string t = key.substr(p.size());
        if (t == "norm1.weight") return plain(r.n1g, {r.cin});
        if (t == "norm1.bias") return plain(r.n1b, {r.cin});
        if (t == "norm2.weight") return plain(r.n2g, {r.cout});
        if (t == "norm2.bias") return plain(r.n2b, {r.cout});
        if (t == "conv1.weight") { *s = VSlot{r.W1, SK_CONV3, {r.cout, r.cin, 3, 3, 3}, r.cout, r.cin}; return true; }
        if (t == "conv1.bias") return plain(r.b1, {r.cout});
        if (t == "conv2.weight") { *s = VSlot{r.W2, SK_CONV3, {r.cout, r.cout, 3, 3, 3}, r.cout, r.cout}; return true; }
        if (t == "conv2.bias") return plain(r.b2, {r.cout});
        if (r.Wsc != nullptr && t == "shortcut.weight") return plain(r.Wsc, {r.cout, r.cin, 1, 1, 1});
        if (r.Wsc != nullptr && t == "shortcut.bias") return plain(r.bsc, {r.cout});
        return false;
    }
    return false;
}

__global__ void rep8_kernel(const __half* __restrict__ src, __half* __restrict__ dst, int C) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 8 * C) dst[i] = src[i % C];
}

struct VaeWs {
    __half *X, *T1, *T2, *X2, *Q, *K, *V, *U, *G, *sa, *sb, *sc, *sd;
    size_t total;
};
VaeWs carve_vws(const tpx_vae* h, int P, uint8_t* base) {
    VaeWs w;
    size_t off = 0;
    auto take = [&](size_t halves) { uint8_t* p = base == nullptr ? nullptr : base + off; off += (halves * 2 + 1023) & ~static_cast<size_t>(1023); return reinterpret_cast<__half*>(p); };
    const size_t S4 = static_cast<size_t>(P) * 64 * h->C0, S8 = static_cast<size_t>(P) * 512 * h->C0, s8 = static_cast<size_t>(P) * 512 * h->C1;
    w.X = take(S4); w.T1 = take(S4); w.T2 = take(S4); w.X2 = take(S4); w.Q = take(S4); w.K = take(S4); w.V = take(S4);
    w.U = take(S8); w.G = take(S8);
    w.sa = take(s8); w.sb = take(s8); w.sc = take(s8); w.sd = take(s8);
    w.total = off;
    return w;
}

int conv3(const __half* x, const __half* W, const __half* bias, const __half* resid, float alpha, __half* out, float* out32, int n_valid, int P, int S,
          int C, int Cout, int epi, cudaStream_t st) {
    // 8^3 layers with narrow outputs: the input block is staged once per output tile (conv_halo.cu) instead of once per tap
    if (conv3_halo_supported(S, C, Cout, epi)) return launch_conv3_halo(x, W, bias, resid, alpha, out, out32, n_valid, P, C, Cout, epi, st);
    GemmProblem p{};
    p.A = x; p.a_mode = AMODE_CONV3; p.conv_S = S; p.conv_C = C; p.W = W;
    p.M = P * S * S * S; p.N = Cout; p.K = 27 * C; p.BN = Cout; p.epi = epi;
    GemmArgs a{};
    a.bias = bias; a.post_scale = 1.0f; a.out0 = out; a.ldo = Cout; a.resid = resid; a.alpha = alpha; a.out32 = out32; a.n_valid = n_valid;
    a.S3 = S * S * S;
    p.args = a;
    return launch_gemm(p, st);
}

int check_run_args(const tpx_vae* h, const void* z, const void* dst, int P, const void* ws, size_t ws_bytes, const char* what) {
    TPX_CHECK(h != nullptr && z != nullptr && dst != nullptr && ws != nullptr, TPX_ERR_ARG, "%s: null argument", what);
    TPX_CHECK(h->finalized, TPX_ERR_STATE, "%s: weights not finalized (load_state_dict first)", what);
    TPX_CHECK(P > 0, TPX_ERR_SHAPE, "%s: empty batch", what);
    TPX_CHECK(ws_bytes >= tpx_vae_workspace_bytes(h, P), TPX_ERR_ARG, "%s: workspace too small (%zu < %zu)", what, ws_bytes, tpx_vae_workspace_bytes(h, P));
    TPX_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, TPX_ERR_ARG, "%s: workspace must be 256-B aligned", what);
    return TPX_OK;
}

// The decode schedule.  stop < 0 runs it to the end and writes `out`; stop = TPX_VAE_STAGE_* ends after that stage and copies its
// channels-last fp16 activation into `tap` (tpx_vae_debug_stage).  Both run the same launches up to the stop.
int vae_run(tpx_vae* h, const void* z, int z_dtype, void* out, int out_dtype, int P, int stop, void* tap, void* ws, cudaStream_t st) {
    VaeWs w = carve_vws(h, P, static_cast<uint8_t*>(ws));
    const int C0 = h->C0, C1 = h->C1;
    const float skip = sqrtf(0.5f);
    const float eps = 1e-5f;
    int rc;
#define TPX_RC(call) do { rc = (call); if (rc != TPX_OK) return rc; } while (0)
#define TPX_TAP(stage, act, S3, C)                                                                                                   \
    do {                                                                                                                             \
        if (stop == (stage)) {                                                                                                       \
            TPX_CUDA(cudaMemcpyAsync(tap, act, static_cast<size_t>(P) * (S3) * (C) * sizeof(__half), cudaMemcpyDeviceToDevice, st)); \
            return TPX_OK;                                                                                                           \
        }                                                                                                                            \
    } while (0)
    TPX_RC(launch_vae_conv_in(z, z_dtype, h->w_pq, h->b_pq, h->Win, h->bin, P, C0, w.X, st));
    __half *X = w.X, *X2 = w.X2;
    TPX_TAP(TPX_VAE_STAGE_CONV_IN, X, 64, C0);
    auto res4 = [&](const VaeRes& r) -> int {   // ResnetBlock C0->C0 at 4^3
        int rc2;
        if ((rc2 = launch_groupnorm_silu(X, r.n1g, r.n1b, P, 64, C0, 32, eps, 1, w.T1, st)) != TPX_OK) return rc2;
        if ((rc2 = conv3(w.T1, r.W1, r.b1, nullptr, 1.f, w.T2, nullptr, 0, P, 4, C0, C0, EPI_STORE, st)) != TPX_OK) return rc2;
        if ((rc2 = launch_groupnorm_silu(w.T2, r.n2g, r.n2b, P, 64, C0, 32, eps, 1, w.T1, st)) != TPX_OK) return rc2;
        if ((rc2 = conv3(w.T1, r.W2, r.b2, X, skip, X2, nullptr, 0, P, 4, C0, C0, EPI_RESID_SCALE, st)) != TPX_OK) return rc2;
        std::swap(X, X2);
        return TPX_OK;
    };
    TPX_RC(res4(h->res[0]));
    TPX_TAP(TPX_VAE_STAGE_MID_RES0, X, 64, C0);
    {   // VolumeAttention: GN -> qkv -> 64-token attention per primitive -> proj, (x + res) * skip
        TPX_RC(launch_groupnorm_silu(X, h->ang, h->anb, P, 64, C0, 32, eps, 0, w.T1, st));
        GemmProblem p{};
        p.A = w.T1; p.a_mode = AMODE_LINEAR; p.lda = C0; p.W = h->Wqkv; p.M = P * 64; p.N = 3 * C0; p.K = C0; p.BN = 256; p.epi = EPI_HEADS;
        GemmArgs a{};
        a.post_scale = 1.0f; a.out0 = w.Q; a.out1 = w.K; a.out2 = w.V; a.split_cols = C0; a.Dh = 32; a.DhP = 32; a.H = h->heads; a.Nseq = 64;
        p.args = a;
        TPX_RC(launch_gemm(p, st));
        TPX_RC(launch_attention(w.Q, w.K, w.V, w.T2, P, h->heads, 64, 64, 32, 32, 1.0f / sqrtf(32.f), st));
        GemmProblem q{};
        q.A = w.T2; q.a_mode = AMODE_LINEAR; q.lda = C0; q.W = h->Wap; q.M = P * 64; q.N = C0; q.K = C0; q.BN = 256; q.epi = EPI_RESID_SCALE;
        GemmArgs b{};
        b.bias = h->bap; b.post_scale = 1.0f; b.out0 = X2; b.ldo = C0; b.resid = X; b.alpha = skip;
        q.args = b;
        TPX_RC(launch_gemm(q, st));
        std::swap(X, X2);
    }
    TPX_TAP(TPX_VAE_STAGE_MID_ATTN, X, 64, C0);
    TPX_RC(res4(h->res[1]));
    TPX_TAP(TPX_VAE_STAGE_MID_RES1, X, 64, C0);
    TPX_RC(res4(h->res[2]));
    TPX_TAP(TPX_VAE_STAGE_UP0_RES0, X, 64, C0);
    TPX_RC(res4(h->res[3]));
    TPX_TAP(TPX_VAE_STAGE_UP0_RES1, X, 64, C0);
    {   // ConvTranspose3d(k2,s2): 8 independent 1x1 GEMMs, one per output offset (a,b,c); each writes its stride-2 sub-lattice of the
        // 8^3 volume with bulk tensor stores (full 128-B lines; the single N = 8*C0 GEMM with a per-thread scatter epilogue was store-bound)
        for (int abc = 0; abc < 8; ++abc) {
            GemmProblem p{};
            p.A = X; p.a_mode = AMODE_LINEAR; p.lda = C0; p.W = h->Wup + static_cast<size_t>(abc) * C0 * C0; p.M = P * 64; p.N = C0; p.K = C0; p.BN = 256;
            p.epi = EPI_STORE;
            GemmArgs a{};
            a.bias = h->bup + static_cast<size_t>(abc) * C0; a.post_scale = 1.0f; a.ldo = C0; a.convt_store = 1;
            a.out0 = w.U + (static_cast<size_t>((abc >> 2) * 8 + ((abc >> 1) & 1)) * 8 + (abc & 1)) * C0;
            p.args = a;
            TPX_RC(launch_gemm(p, st));
        }
    }
    TPX_TAP(TPX_VAE_STAGE_UPSAMPLE, w.U, 512, C0);
    {   // ResnetBlock C0 -> C1 at 8^3 with 1x1 shortcut
        const VaeRes& r = h->res[4];
        TPX_RC(launch_groupnorm_silu(w.U, r.n1g, r.n1b, P, 512, C0, 32, eps, 1, w.G, st));
        TPX_RC(conv3(w.G, r.W1, r.b1, nullptr, 1.f, w.sa, nullptr, 0, P, 8, C0, C1, EPI_STORE, st));
        TPX_RC(launch_groupnorm_silu(w.sa, r.n2g, r.n2b, P, 512, C1, 32, eps, 1, w.sb, st));
        GemmProblem p{};
        p.A = w.U; p.a_mode = AMODE_LINEAR; p.lda = C0; p.W = r.Wsc; p.M = P * 512; p.N = C1; p.K = C0; p.BN = 32; p.epi = EPI_STORE;
        GemmArgs a{};
        a.bias = r.bsc; a.post_scale = 1.0f; a.out0 = w.sc; a.ldo = C1;
        p.args = a;
        TPX_RC(launch_gemm(p, st));
        TPX_RC(conv3(w.sb, r.W2, r.b2, w.sc, skip, w.sd, nullptr, 0, P, 8, C1, C1, EPI_RESID_SCALE, st));
    }
    TPX_TAP(TPX_VAE_STAGE_UP1_RES0, w.sd, 512, C1);
    {   // ResnetBlock C1 -> C1 at 8^3
        const VaeRes& r = h->res[5];
        TPX_RC(launch_groupnorm_silu(w.sd, r.n1g, r.n1b, P, 512, C1, 32, eps, 1, w.sa, st));
        TPX_RC(conv3(w.sa, r.W1, r.b1, nullptr, 1.f, w.sb, nullptr, 0, P, 8, C1, C1, EPI_STORE, st));
        TPX_RC(launch_groupnorm_silu(w.sb, r.n2g, r.n2b, P, 512, C1, 32, eps, 1, w.sa, st));
        TPX_RC(conv3(w.sa, r.W2, r.b2, w.sd, skip, w.sc, nullptr, 0, P, 8, C1, C1, EPI_RESID_SCALE, st));
    }
    TPX_TAP(TPX_VAE_STAGE_UP1_RES1, w.sc, 512, C1);
    TPX_RC(launch_groupnorm_silu(w.sc, h->nog, h->nob, P, 512, C1, 32, eps, 1, w.sa, st));
    TPX_TAP(TPX_VAE_STAGE_NORM_OUT, w.sa, 512, C1);
    TPX_RC(conv3(w.sa, h->Wout, h->bout, nullptr, 1.f, out_dtype == TPX_DTYPE_F16 ? static_cast<__half*>(out) : nullptr,
                 out_dtype == TPX_DTYPE_F32 ? static_cast<float*>(out) : nullptr, h->Cout, P, 8, C1, 16, EPI_NCDHW, st));
#undef TPX_TAP
#undef TPX_RC
    return TPX_OK;
}
}  // namespace

extern "C" {

int tpx_vae_create(const tpx_vae_config* c, tpx_vae** out) {
    TPX_CHECK(c != nullptr && out != nullptr, TPX_ERR_ARG, "vae_create: null argument");
    TPX_CHECK(c->latent_channels == 1, TPX_ERR_SHAPE, "vae_create: latent_channels %d unsupported (kernel set covers the shipped config: 1)", c->latent_channels);
    TPX_CHECK(c->ch_mid == 256 && c->ch_out == 32 && c->out_channels >= 1 && c->out_channels <= 16, TPX_ERR_SHAPE,
              "vae_create: up_channels (%d,%d)/out %d unsupported (kernel set covers the shipped config: (256,32)/6)", c->ch_mid, c->ch_out, c->out_channels);
    TPX_CHECK(c->attn_heads > 0 && c->ch_mid % c->attn_heads == 0 && (c->ch_mid / c->attn_heads) == 32, TPX_ERR_SHAPE, "vae_create: attention head dim must be 32");
    TPX_DEVICE_GUARD();
    tpx_vae* h = new tpx_vae();
    h->C0 = c->ch_mid; h->C1 = c->ch_out; h->Cout = c->out_channels; h->heads = c->attn_heads;
    carve(h, nullptr);
    cudaError_t e = cudaMalloc(&h->store, h->store_halves * 2);
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "cudaMalloc(vae parameter store)"); }
    e = cudaMemset(h->store, 0, h->store_halves * 2);
    if (e != cudaSuccess) { cudaFree(h->store); delete h; return cuda_fail(e, "cudaMemset(vae parameter store)"); }
    carve(h, h->store);
    auto& r = h->required;
    for (const char* k : {"post_quant_conv.weight", "post_quant_conv.bias", "decoder.conv_in.weight", "decoder.conv_in.bias", "decoder.norm_out.weight",
                          "decoder.norm_out.bias", "decoder.conv_out.weight", "decoder.conv_out.bias", "decoder.up_blocks.0.upsample.weight",
                          "decoder.up_blocks.0.upsample.bias", "decoder.mid_block.attns.0.norm.weight", "decoder.mid_block.attns.0.norm.bias",
                          "decoder.mid_block.attns.0.attn.qkv.weight", "decoder.mid_block.attns.0.attn.proj.weight",
                          "decoder.mid_block.attns.0.attn.proj.bias"})
        r.emplace_back(k);
    for (int i = 0; i < 6; ++i) {
        for (const char* k : {"norm1.weight", "norm1.bias", "conv1.weight", "conv1.bias", "norm2.weight", "norm2.bias", "conv2.weight", "conv2.bias"})
            r.emplace_back(std::string(kResPrefix[i]) + k);
        if (h->res[i].Wsc != nullptr) { r.emplace_back(std::string(kResPrefix[i]) + "shortcut.weight"); r.emplace_back(std::string(kResPrefix[i]) + "shortcut.bias"); }
    }
    h->seen.assign(r.size(), 0);
    *out = h;
    return TPX_OK;
}

void tpx_vae_destroy(tpx_vae* h) {
    if (h == nullptr) return;
    if (h->store != nullptr) cudaFree(h->store);
    delete h;
}

int tpx_vae_set_weight(tpx_vae* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream) {
    TPX_CHECK(h != nullptr && ref_key != nullptr && dev_ptr != nullptr && shape != nullptr, TPX_ERR_ARG, "vae_set_weight: null argument");
    const std::string key(ref_key);
    if (key.rfind("encoder.", 0) == 0 || key.rfind("quant_conv.", 0) == 0) return 1;  // not on the decode path
    VSlot s;
    if (!find_vslot(h, key, &s)) { set_error("vae_set_weight: unexpected key '%s'", ref_key); return TPX_ERR_KEY; }
    bool ok = ndim == static_cast<int>(s.shape.size());
    long long n = 1;
    for (int i = 0; ok && i < ndim; ++i) { ok = shape[i] == s.shape[i]; n *= shape[i]; }
    TPX_CHECK(ok, TPX_ERR_SHAPE, "vae_set_weight: size mismatch for %s", ref_key);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int rc = TPX_OK;
    switch (s.kind) {
        case SK_PLAIN: rc = launch_to_half(dev_ptr, dtype, s.ptr, n, st); break;
        case SK_CONV3: rc = launch_pack_conv3(dev_ptr, dtype, s.ptr, s.a, s.b, 0, st); break;
        case SK_CONV3_T: rc = launch_pack_conv3(dev_ptr, dtype, s.ptr, s.a, s.b, 1, st); break;   // rows >= Cout stay zero
        case SK_CONVT2: rc = launch_pack_convt2(dev_ptr, dtype, s.ptr, s.a, s.b, st); break;
        case SK_BIAS_REP8: {
            rc = launch_to_half(dev_ptr, dtype, s.ptr, n, st);   // first C entries, then replicated for the 8 output offsets
            if (rc == TPX_OK) { rep8_kernel<<<(8 * s.a + 255) / 256, 256, 0, st>>>(s.ptr, s.ptr, s.a); rc = cudaGetLastError() == cudaSuccess ? TPX_OK : TPX_ERR_CUDA; }
            break;
        }
    }
    if (rc != TPX_OK) return rc;
    for (size_t i = 0; i < h->required.size(); ++i)
        if (h->required[i] == key) h->seen[i] = 1;
    h->finalized = false;
    return TPX_OK;
}

int tpx_vae_finalize(tpx_vae* h, void* stream) {
    (void)stream;
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "vae_finalize: null handle");
    for (size_t i = 0; i < h->required.size(); ++i) TPX_CHECK(h->seen[i], TPX_ERR_STATE, "vae_finalize: missing key '%s' in state_dict", h->required[i].c_str());
    h->finalized = true;
    return TPX_OK;
}

size_t tpx_vae_workspace_bytes(const tpx_vae* h, int P) {
    if (h == nullptr || P <= 0) return 0;
    return carve_vws(h, P, nullptr).total;
}

int tpx_vae_decode(tpx_vae* h, const void* z, int z_dtype, void* out, int out_dtype, int P, void* ws, size_t ws_bytes, void* stream) {
    const int rc = check_run_args(h, z, out, P, ws, ws_bytes, "vae_decode");
    if (rc != TPX_OK) return rc;
    TPX_CHECK(out_dtype == TPX_DTYPE_F32 || out_dtype == TPX_DTYPE_F16, TPX_ERR_ARG, "vae_decode: bad output dtype %d", out_dtype);
    return vae_run(h, z, z_dtype, out, out_dtype, P, -1, nullptr, ws, static_cast<cudaStream_t>(stream));
}

int tpx_vae_debug_stage(tpx_vae* h, const void* z, int z_dtype, int P, int stage, void* tap_f16, void* ws, size_t ws_bytes, void* stream) {
    const int rc = check_run_args(h, z, tap_f16, P, ws, ws_bytes, "vae_debug_stage");
    if (rc != TPX_OK) return rc;
    TPX_CHECK(stage >= TPX_VAE_STAGE_CONV_IN && stage <= TPX_VAE_STAGE_NORM_OUT, TPX_ERR_ARG, "vae_debug_stage: bad stage %d", stage);
    return vae_run(h, z, z_dtype, nullptr, TPX_DTYPE_F16, P, stage, tap_f16, ws, static_cast<cudaStream_t>(stream));
}

int tpx_conv3d_k3(const void* x, const void* W, const void* bias, const void* resid, float alpha, void* out, int P, int S, int C, int Cout, void* stream) {
    TPX_CHECK(x != nullptr && W != nullptr && out != nullptr, TPX_ERR_ARG, "conv3d_k3: null argument");
    TPX_DEVICE_GUARD();
    const bool plain = resid == nullptr && alpha == 1.0f;
    return conv3(static_cast<const __half*>(x), static_cast<const __half*>(W), static_cast<const __half*>(bias), static_cast<const __half*>(resid), alpha,
                 static_cast<__half*>(out), nullptr, 0, P, S, C, Cout, plain ? EPI_STORE : EPI_RESID_SCALE, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
