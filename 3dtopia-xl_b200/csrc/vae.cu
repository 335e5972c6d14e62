// VAE decoder and encoder handles: repacked fp16 parameters keyed by the reference's state_dict names, and the decode / encode schedules.
//   reference: models/vae3d_dib.py:437-440 (VAE.decode), :369-387 (Decoder.forward), :220-226 (MidBlock),
//              :259-267 (UpBlock), :128-145 (ResnetBlock), :34-48 (VolumeAttention);
//              :431-435 (VAE.encode), :310-327 (Encoder.forward), :178-184 (DownBlock), :428 (quant_conv)
// Activations are channels-last fp16 [P, S^3, C]; every primitive is independent (GroupNorm statistics are
// per primitive), so the whole decoder is a batch of P tiny volumes.
#include <cmath>

#include "kernels.cuh"

using namespace tpx;

struct VaeRes {
    int cin, cout;
    __half *n1g, *n1b, *W1, *b1, *n2g, *n2b, *W2, *b2, *Wsc, *bsc;  // Wsc null when cin == cout
};
struct VaeAttn {
    __half *ng, *nb, *Wqkv, *Wproj, *bproj;
    int heads;
};

struct tpx_vae {
    int C0, C1, Cout;
    ParamStore params;
    __half *w_pq, *b_pq, *Win, *bin;
    VaeRes res[6];                           // mid0, mid1, up0.0, up0.1, up1.0, up1.1
    VaeAttn attn;                            // mid attention
    __half *Wup, *bup;                       // [8*C0, C0], [8*C0]
    __half *nog, *nob, *Wout, *bout;         // norm_out, conv_out (padded to 16 rows)
};


// Encoder of the released layout (down_channels [32, 256], in_channels 6, latent 1): conv_in 6 -> 32 at 8^3, two 32-channel
// ResnetBlocks, the stride-2 downsample to 4^3, a 32 -> 256 block with its 1x1 shortcut, a 256 block, the mid block (res, attention,
// res), norm_out + SiLU and conv_out 256 -> 2 with quant_conv in its epilogue.
struct tpx_vae_encoder {
    int Cin = 6, C0 = 32, C1 = 256;
    ParamStore params;
    __half *Win, *bin;                       // conv_in [32, 6*27] (the reference's own layout), bias
    VaeRes res[6];                           // down0.0, down0.1 (32, 8^3), down1.0 (32 -> 256), down1.1, mid0, mid1 (256, 4^3)
    __half *Wds, *bds;                       // downsample, repacked for the space-to-depth input: [32, 27*256]
    VaeAttn attn;                            // mid attention
    __half *nog, *nob, *Wout, *bout;         // norm_out, conv_out (padded to 16 rows)
    __half* quant;                           // quant_conv [w00, w01, w10, w11, b0, b1]
};

namespace {
// Parameter slots are 128 B apart (TMA operands need 16-B alignment)
constexpr size_t kSlotAlign = 128;

// ResnetBlock (vae3d_dib.py:128-145) and VolumeAttention (:34-48) keys under `p`, the same in the decoder and the encoder
void res_params(ParamStore& s, const std::string& p, VaeRes& r, int cin, int cout) {
    r.cin = cin;
    r.cout = cout;
    s.weight_bias(p + "norm1", r.n1g, r.n1b, {cin});
    s.weight_bias(p + "conv1", r.W1, r.b1, {cout, cin, 3, 3, 3}, PK_CONV3);
    s.weight_bias(p + "norm2", r.n2g, r.n2b, {cout});
    s.weight_bias(p + "conv2", r.W2, r.b2, {cout, cout, 3, 3, 3}, PK_CONV3);
    r.Wsc = r.bsc = nullptr;
    if (cin != cout) s.weight_bias(p + "shortcut", r.Wsc, r.bsc, {cout, cin, 1, 1, 1});
}

void attn_params(ParamStore& s, const std::string& p, VaeAttn& at, int C, int heads) {
    at.heads = heads;
    s.weight_bias(p + "norm", at.ng, at.nb, {C});
    at.Wqkv = s.param(p + "attn.qkv.weight", {3 * C, C});
    s.weight_bias(p + "attn.proj", at.Wproj, at.bproj, {C, C});
}

void declare_decoder(tpx_vae* h, ParamStore& s, int heads) {
    const int64_t C0 = h->C0, C1 = h->C1;
    s.weight_bias("post_quant_conv", h->w_pq, h->b_pq, {1, 1, 1, 1, 1});
    s.weight_bias("decoder.conv_in", h->Win, h->bin, {C0, 1, 3, 3, 3});
    const char* res[6] = {"mid_block.nets.0.", "mid_block.nets.1.", "up_blocks.0.nets.0.", "up_blocks.0.nets.1.", "up_blocks.1.nets.0.",
                          "up_blocks.1.nets.1."};
    for (int i = 0; i < 6; ++i) res_params(s, std::string("decoder.") + res[i], h->res[i], i < 5 ? h->C0 : h->C1, i < 4 ? h->C0 : h->C1);
    attn_params(s, "decoder.mid_block.attns.0.", h->attn, h->C0, heads);
    h->Wup = s.param("decoder.up_blocks.0.upsample.weight", {C0, C0, 2, 2, 2}, PK_CONVT2);
    h->bup = s.param_at(s.take(8 * C0), "decoder.up_blocks.0.upsample.bias", {C0}, PK_BIAS_REP8);
    s.weight_bias("decoder.norm_out", h->nog, h->nob, {C1});
    h->Wout = s.param_at(s.take(16 * 27 * C1), "decoder.conv_out.weight", {C1, h->Cout, 3, 3, 3}, PK_CONV3_T);   // rows >= Cout stay zero
    h->bout = s.param_at(s.take(16), "decoder.conv_out.bias", {h->Cout});
}

struct VaeWs {
    __half *X, *T1, *T2, *X2, *Q, *K, *V, *U, *G, *sa, *sb, *sc, *sd;
    size_t total;
};
VaeWs carve_vws(const tpx_vae* h, int P, void* base) {
    Carve c{static_cast<uint8_t*>(base), 1024};
    VaeWs w;
    const size_t S4 = static_cast<size_t>(P) * 64 * h->C0, S8 = static_cast<size_t>(P) * 512 * h->C0, s8 = static_cast<size_t>(P) * 512 * h->C1;
    w.X = c.take<__half>(S4); w.T1 = c.take<__half>(S4); w.T2 = c.take<__half>(S4); w.X2 = c.take<__half>(S4); w.Q = c.take<__half>(S4);
    w.K = c.take<__half>(S4); w.V = c.take<__half>(S4);
    w.U = c.take<__half>(S8); w.G = c.take<__half>(S8);
    w.sa = c.take<__half>(s8); w.sb = c.take<__half>(s8); w.sc = c.take<__half>(s8); w.sd = c.take<__half>(s8);
    w.total = c.off;
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

// ---- blocks both schedules run (weights come as structs, scratch as pointers: no handle) ------------------------------------
struct BlockScratch {
    __half *T1, *T2, *Q, *K, *V;   // [P, S^3, C] each
};
constexpr float kSkip = 0.70710678118654752f;   // sqrtf(0.5f): skip_scale (vae3d_dib.py:338, :395)
constexpr float kEps = 1e-5f;

// ResnetBlock C -> C at S^3 (vae3d_dib.py:128-145): GN+SiLU -> conv1 -> GN+SiLU -> conv2 + x, * skip.  X2 receives the result and the two
// pointers are swapped, so X is the block's output on return.  4 launches.
int resnet_block(const VaeRes& r, int S, __half*& X, __half*& X2, const BlockScratch& sc, int P, cudaStream_t st) {
    const int S3 = S * S * S, C = r.cin;
    int rc;
    if ((rc = launch_groupnorm_silu(X, r.n1g, r.n1b, P, S3, C, 32, kEps, 1, sc.T1, st)) != TPX_OK) return rc;
    if ((rc = conv3(sc.T1, r.W1, r.b1, nullptr, 1.f, sc.T2, nullptr, 0, P, S, C, C, EPI_STORE, st)) != TPX_OK) return rc;
    if ((rc = launch_groupnorm_silu(sc.T2, r.n2g, r.n2b, P, S3, C, 32, kEps, 1, sc.T1, st)) != TPX_OK) return rc;
    if ((rc = conv3(sc.T1, r.W2, r.b2, X, kSkip, X2, nullptr, 0, P, S, C, C, EPI_RESID_SCALE, st)) != TPX_OK) return rc;
    std::swap(X, X2);
    return TPX_OK;
}

// VolumeAttention at 4^3 (vae3d_dib.py:34-48): GN -> qkv -> 64-token attention per primitive -> proj, (x + res) * skip.  Result in X
// (swapped as above).  4 launches.
int attention_block(const VaeAttn& at, __half*& X, __half*& X2, const BlockScratch& sc, int P, int C, cudaStream_t st) {
    int rc;
    if ((rc = launch_groupnorm_silu(X, at.ng, at.nb, P, 64, C, 32, kEps, 0, sc.T1, st)) != TPX_OK) return rc;
    GemmProblem p{};
    p.A = sc.T1; p.a_mode = AMODE_LINEAR; p.lda = C; p.W = at.Wqkv; p.M = P * 64; p.N = 3 * C; p.K = C; p.BN = 256; p.epi = EPI_HEADS;
    GemmArgs a{};
    a.post_scale = 1.0f; a.out0 = sc.Q; a.out1 = sc.K; a.out2 = sc.V; a.split_cols = C; a.Dh = 32; a.DhP = 32; a.H = at.heads; a.Nseq = 64;
    p.args = a;
    if ((rc = launch_gemm(p, st)) != TPX_OK) return rc;
    if ((rc = launch_attention(sc.Q, sc.K, sc.V, sc.T2, P, at.heads, 64, 64, 32, 32, 1.0f / sqrtf(32.f), st)) != TPX_OK) return rc;
    GemmProblem q{};
    q.A = sc.T2; q.a_mode = AMODE_LINEAR; q.lda = C; q.W = at.Wproj; q.M = P * 64; q.N = C; q.K = C; q.BN = 256; q.epi = EPI_RESID_SCALE;
    GemmArgs b{};
    b.bias = at.bproj; b.post_scale = 1.0f; b.out0 = X2; b.ldo = C; b.resid = X; b.alpha = kSkip;
    q.args = b;
    if ((rc = launch_gemm(q, st)) != TPX_OK) return rc;
    std::swap(X, X2);
    return TPX_OK;
}

// Argument checks of the decode and encode entry points; ws_bytes_fn is the handle's *_workspace_bytes.
template <class H>
int check_run_args(const H* h, size_t (*ws_bytes_fn)(const H*, int), const void* in, const void* dst, int P, const void* ws, size_t ws_bytes,
                   const char* what) {
    TPX_CHECK(h != nullptr && in != nullptr && dst != nullptr && ws != nullptr, TPX_ERR_ARG, "%s: null argument", what);
    TPX_CHECK(h->params.finalized, TPX_ERR_STATE, "%s: weights not finalized (load_state_dict first)", what);
    TPX_CHECK(P > 0, TPX_ERR_SHAPE, "%s: empty batch", what);
    const size_t need = ws_bytes_fn(h, P);
    TPX_CHECK(ws_bytes >= need, TPX_ERR_ARG, "%s: workspace too small (%zu < %zu)", what, ws_bytes, need);
    TPX_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, TPX_ERR_ARG, "%s: workspace must be 256-B aligned", what);
    return TPX_OK;
}

// The schedules' launch check and debug tap: stop = the stage to end after (< 0: none), whose activation is copied into `tap`
#define TPX_RC(call) do { rc = (call); if (rc != TPX_OK) return rc; } while (0)
#define TPX_TAP(stage, act, S3, C)                                                                                                   \
    do {                                                                                                                             \
        if (stop == (stage)) {                                                                                                       \
            TPX_CUDA(cudaMemcpyAsync(tap, act, static_cast<size_t>(P) * (S3) * (C) * sizeof(__half), cudaMemcpyDeviceToDevice, st)); \
            return TPX_OK;                                                                                                           \
        }                                                                                                                            \
    } while (0)

// The decode schedule.  stop < 0 runs it to the end and writes `out`; stop = TPX_VAE_STAGE_* ends after that stage and copies its
// channels-last fp16 activation into `tap` (tpx_vae_debug_stage).  Both run the same launches up to the stop.
int vae_run(tpx_vae* h, const void* z, int z_dtype, void* out, int out_dtype, int P, int stop, void* tap, void* ws, cudaStream_t st) {
    VaeWs w = carve_vws(h, P, ws);
    const int C0 = h->C0, C1 = h->C1;
    const float skip = kSkip;
    const float eps = kEps;
    int rc;
    TPX_RC(launch_vae_conv_in(z, z_dtype, h->w_pq, h->b_pq, h->Win, h->bin, P, C0, w.X, st));
    __half *X = w.X, *X2 = w.X2;
    const BlockScratch sc{w.T1, w.T2, w.Q, w.K, w.V};
    TPX_TAP(TPX_VAE_STAGE_CONV_IN, X, 64, C0);
    TPX_RC(resnet_block(h->res[0], 4, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_STAGE_MID_RES0, X, 64, C0);
    TPX_RC(attention_block(h->attn, X, X2, sc, P, C0, st));
    TPX_TAP(TPX_VAE_STAGE_MID_ATTN, X, 64, C0);
    TPX_RC(resnet_block(h->res[1], 4, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_STAGE_MID_RES1, X, 64, C0);
    TPX_RC(resnet_block(h->res[2], 4, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_STAGE_UP0_RES0, X, 64, C0);
    TPX_RC(resnet_block(h->res[3], 4, X, X2, sc, P, st));
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
    return TPX_OK;
}

// ---- encoder ----------------------------------------------------------------------------------------------------------------
void declare_encoder(tpx_vae_encoder* h, ParamStore& s, int heads) {
    const int64_t C0 = h->C0, C1 = h->C1;
    s.weight_bias("encoder.conv_in", h->Win, h->bin, {C0, h->Cin, 3, 3, 3});
    const char* res[6] = {"down_blocks.0.nets.0.", "down_blocks.0.nets.1.", "down_blocks.1.nets.0.", "down_blocks.1.nets.1.", "mid_block.nets.0.",
                          "mid_block.nets.1."};
    for (int i = 0; i < 6; ++i) res_params(s, std::string("encoder.") + res[i], h->res[i], i < 3 ? h->C0 : h->C1, i < 2 ? h->C0 : h->C1);
    h->Wds = s.take(C0 * 27 * 8 * C0);
    h->bds = s.take(C0);
    s.weight_bias_at("encoder.down_blocks.0.downsample", h->Wds, h->bds, {C0, C0, 3, 3, 3}, PK_CONV3_S2D);
    attn_params(s, "encoder.mid_block.attns.0.", h->attn, h->C1, heads);
    s.weight_bias("encoder.norm_out", h->nog, h->nob, {C1});
    h->Wout = s.take(16 * 27 * C1);   // rows 2..15 stay zero
    h->bout = s.take(16);
    s.weight_bias_at("encoder.conv_out", h->Wout, h->bout, {2, C1, 3, 3, 3}, PK_CONV3);
    h->quant = s.take(8);
    s.weight_bias_at("quant_conv", h->quant, h->quant + 4, {2, 2, 1, 1, 1});
}

// Scratch: every activation of the encoder is 32 KB per primitive (8^3 x 32 or 4^3 x 256 fp16), so the workspace is eight such buffers.
struct EncWs {
    __half *A, *B, *T1, *T2, *Q, *K, *V, *SC;
    size_t total;
};
EncWs carve_ews(int P, void* base) {
    Carve c{static_cast<uint8_t*>(base), 1024};
    EncWs w;
    const size_t n = static_cast<size_t>(P) * 16384;
    w.A = c.take<__half>(n); w.B = c.take<__half>(n); w.T1 = c.take<__half>(n); w.T2 = c.take<__half>(n);
    w.Q = c.take<__half>(n); w.K = c.take<__half>(n); w.V = c.take<__half>(n); w.SC = c.take<__half>(n);
    w.total = c.off;
    return w;
}

// The encode schedule (Encoder.forward + quant_conv, vae3d_dib.py:310-327, :431-433).  stop < 0 runs it to the end and writes the
// moments; stop = TPX_VAE_ENC_STAGE_* ends after that stage and copies its channels-last fp16 activation into `tap`.
// Launches: conv_in 1, 8^3 block 4 + 4, downsample 2, 32 -> 256 block 5, 256 blocks 4 each, attention 4, norm_out 1, conv_out 1: 34.
int enc_run(tpx_vae_encoder* h, const void* x, int x_dtype, void* out, int out_dtype, int P, int stop, void* tap, void* ws, cudaStream_t st) {
    EncWs w = carve_ews(P, ws);
    const int C0 = h->C0, C1 = h->C1;
    const BlockScratch sc{w.T1, w.T2, w.Q, w.K, w.V};
    int rc;
    __half *X = w.A, *X2 = w.B;
    TPX_RC(launch_vae_enc_conv_in(x, x_dtype, h->Win, h->bin, P, X, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_CONV_IN, X, 512, C0);
    TPX_RC(resnet_block(h->res[0], 8, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_DOWN0_RES0, X, 512, C0);
    TPX_RC(resnet_block(h->res[1], 8, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_DOWN0_RES1, X, 512, C0);
    // Conv3d(k3, s2, p1) 8^3 -> 4^3 as a stride-1 conv over the space-to-depth volume [P, 4^3, 8*32] (launch_pack_conv3_s2d)
    TPX_RC(launch_space_to_depth2(X, w.T1, P, C0, st));
    TPX_RC(conv3(w.T1, h->Wds, h->bds, nullptr, 1.f, X2, nullptr, 0, P, 4, 8 * C0, C0, EPI_STORE, st));
    std::swap(X, X2);
    TPX_TAP(TPX_VAE_ENC_STAGE_DOWNSAMPLE, X, 64, C0);
    {   // ResnetBlock C0 -> C1 at 4^3 with its 1x1 shortcut (a K = 32 GEMM)
        const VaeRes& r = h->res[2];
        TPX_RC(launch_groupnorm_silu(X, r.n1g, r.n1b, P, 64, C0, 32, kEps, 1, w.T1, st));
        TPX_RC(conv3(w.T1, r.W1, r.b1, nullptr, 1.f, w.T2, nullptr, 0, P, 4, C0, C1, EPI_STORE, st));
        TPX_RC(launch_groupnorm_silu(w.T2, r.n2g, r.n2b, P, 64, C1, 32, kEps, 1, w.T1, st));
        GemmProblem p{};
        p.A = X; p.a_mode = AMODE_LINEAR; p.lda = C0; p.W = r.Wsc; p.M = P * 64; p.N = C1; p.K = C0; p.BN = 256; p.epi = EPI_STORE;
        GemmArgs a{};
        a.bias = r.bsc; a.post_scale = 1.0f; a.out0 = w.SC; a.ldo = C1;
        p.args = a;
        TPX_RC(launch_gemm(p, st));
        TPX_RC(conv3(w.T1, r.W2, r.b2, w.SC, kSkip, X2, nullptr, 0, P, 4, C1, C1, EPI_RESID_SCALE, st));
        std::swap(X, X2);
    }
    TPX_TAP(TPX_VAE_ENC_STAGE_DOWN1_RES0, X, 64, C1);
    TPX_RC(resnet_block(h->res[3], 4, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_DOWN1_RES1, X, 64, C1);
    TPX_RC(resnet_block(h->res[4], 4, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_MID_RES0, X, 64, C1);
    TPX_RC(attention_block(h->attn, X, X2, sc, P, C1, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_MID_ATTN, X, 64, C1);
    TPX_RC(resnet_block(h->res[5], 4, X, X2, sc, P, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_MID_RES1, X, 64, C1);
    TPX_RC(launch_groupnorm_silu(X, h->nog, h->nob, P, 64, C1, 32, kEps, 1, w.T1, st));
    TPX_TAP(TPX_VAE_ENC_STAGE_NORM_OUT, w.T1, 64, C1);
    {   // conv_out 256 -> 2 (16-row tile, rows 2..15 zero) with quant_conv in the epilogue, written NCDHW [P, 2, 4, 4, 4]
        GemmProblem p{};
        p.A = w.T1; p.a_mode = AMODE_CONV3; p.conv_S = 4; p.conv_C = C1; p.W = h->Wout;
        p.M = P * 64; p.N = 16; p.K = 27 * C1; p.BN = 16; p.epi = EPI_MOMENTS;
        GemmArgs a{};
        a.bias = h->bout; a.post_scale = 1.0f; a.quant = h->quant; a.S3 = 64;
        a.out0 = out_dtype == TPX_DTYPE_F16 ? static_cast<__half*>(out) : nullptr;
        a.out32 = out_dtype == TPX_DTYPE_F32 ? static_cast<float*>(out) : nullptr;
        p.args = a;
        TPX_RC(launch_gemm(p, st));
    }
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
    h->C0 = c->ch_mid; h->C1 = c->ch_out; h->Cout = c->out_channels;
    h->params.ignored = {"encoder.", "quant_conv."};   // not on the decode path
    const int heads = c->attn_heads;
    const int rc = h->params.create(kSlotAlign, [h, heads](ParamStore& s) { declare_decoder(h, s, heads); });
    if (rc != TPX_OK) { delete h; return rc; }
    *out = h;
    return TPX_OK;
}

void tpx_vae_destroy(tpx_vae* h) { delete h; }

int tpx_vae_set_weight(tpx_vae* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream) {
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "vae_set_weight: null argument");
    return h->params.set("vae_set_weight", ref_key, dev_ptr, dtype, shape, ndim, static_cast<cudaStream_t>(stream));
}

int tpx_vae_finalize(tpx_vae* h, void* stream) {
    (void)stream;
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "vae_finalize: null handle");
    const int rc = h->params.complete("vae_finalize");
    if (rc != TPX_OK) return rc;
    h->params.finalized = true;
    return TPX_OK;
}

size_t tpx_vae_workspace_bytes(const tpx_vae* h, int P) {
    if (h == nullptr || P <= 0) return 0;
    return carve_vws(h, P, nullptr).total;
}

int tpx_vae_decode(tpx_vae* h, const void* z, int z_dtype, void* out, int out_dtype, int P, void* ws, size_t ws_bytes, void* stream) {
    const int rc = check_run_args(h, tpx_vae_workspace_bytes, z, out, P, ws, ws_bytes, "vae_decode");
    if (rc != TPX_OK) return rc;
    TPX_CHECK(out_dtype == TPX_DTYPE_F32 || out_dtype == TPX_DTYPE_F16, TPX_ERR_ARG, "vae_decode: bad output dtype %d", out_dtype);
    return vae_run(h, z, z_dtype, out, out_dtype, P, -1, nullptr, ws, static_cast<cudaStream_t>(stream));
}

int tpx_vae_debug_stage(tpx_vae* h, const void* z, int z_dtype, int P, int stage, void* tap_f16, void* ws, size_t ws_bytes, void* stream) {
    const int rc = check_run_args(h, tpx_vae_workspace_bytes, z, tap_f16, P, ws, ws_bytes, "vae_debug_stage");
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


// ---- encoder -------------------------------------------------------------------------------------------------------------------
int tpx_vae_encoder_create(const tpx_vae_config* c, tpx_vae_encoder** out) {
    TPX_CHECK(c != nullptr && out != nullptr, TPX_ERR_ARG, "vae_encoder_create: null argument");
    TPX_CHECK(c->latent_channels == 1 && c->out_channels == 6, TPX_ERR_SHAPE,
              "vae_encoder_create: latent %d / in_channels %d unsupported (kernel set covers the shipped config: 1 / 6)", c->latent_channels, c->out_channels);
    TPX_CHECK(c->ch_mid == 256 && c->ch_out == 32, TPX_ERR_SHAPE, "vae_encoder_create: down_channels (%d,%d) unsupported (kernel set covers (32,256))",
              c->ch_out, c->ch_mid);
    TPX_CHECK(c->attn_heads > 0 && c->ch_mid % c->attn_heads == 0 && (c->ch_mid / c->attn_heads) == 32, TPX_ERR_SHAPE, "vae_encoder_create: attention head dim must be 32");
    TPX_DEVICE_GUARD();
    tpx_vae_encoder* h = new tpx_vae_encoder();
    h->params.ignored = {"decoder.", "post_quant_conv."};   // not on the encode path
    const int heads = c->attn_heads;
    const int rc = h->params.create(kSlotAlign, [h, heads](ParamStore& s) { declare_encoder(h, s, heads); });
    if (rc != TPX_OK) { delete h; return rc; }
    *out = h;
    return TPX_OK;
}

void tpx_vae_encoder_destroy(tpx_vae_encoder* h) { delete h; }

int tpx_vae_encoder_set_weight(tpx_vae_encoder* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream) {
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "vae_encoder_set_weight: null argument");
    return h->params.set("vae_encoder_set_weight", ref_key, dev_ptr, dtype, shape, ndim, static_cast<cudaStream_t>(stream));
}

int tpx_vae_encoder_finalize(tpx_vae_encoder* h, void* stream) {
    (void)stream;
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "vae_encoder_finalize: null handle");
    const int rc = h->params.complete("vae_encoder_finalize");
    if (rc != TPX_OK) return rc;
    h->params.finalized = true;
    return TPX_OK;
}

size_t tpx_vae_encoder_workspace_bytes(const tpx_vae_encoder* h, int P) {
    if (h == nullptr || P <= 0) return 0;
    return carve_ews(P, nullptr).total;
}

int tpx_vae_encode(tpx_vae_encoder* h, const void* x, int x_dtype, void* moments_out, int out_dtype, int P, void* ws, size_t ws_bytes, void* stream) {
    const int rc = check_run_args(h, tpx_vae_encoder_workspace_bytes, x, moments_out, P, ws, ws_bytes, "vae_encode");
    if (rc != TPX_OK) return rc;
    TPX_CHECK(out_dtype == TPX_DTYPE_F32 || out_dtype == TPX_DTYPE_F16, TPX_ERR_ARG, "vae_encode: bad output dtype %d", out_dtype);
    return enc_run(h, x, x_dtype, moments_out, out_dtype, P, -1, nullptr, ws, static_cast<cudaStream_t>(stream));
}

int tpx_vae_encode_debug_stage(tpx_vae_encoder* h, const void* x, int x_dtype, int P, int stage, void* tap_f16, void* ws, size_t ws_bytes, void* stream) {
    const int rc = check_run_args(h, tpx_vae_encoder_workspace_bytes, x, tap_f16, P, ws, ws_bytes, "vae_encode_debug_stage");
    if (rc != TPX_OK) return rc;
    TPX_CHECK(stage >= TPX_VAE_ENC_STAGE_CONV_IN && stage <= TPX_VAE_ENC_STAGE_NORM_OUT, TPX_ERR_ARG, "vae_encode_debug_stage: bad stage %d", stage);
    return enc_run(h, x, x_dtype, nullptr, TPX_DTYPE_F16, P, stage, tap_f16, ws, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
