// DiT handle: packed fp16 parameter store keyed by the reference's state_dict names, the per-image
// conditioning hoist, and the per-step forward schedule (one stream, ~12 launches per block, no host sync).
//   reference: models/dit_crossattn.py:111-213, models/attention.py, models/utils.py
#include <cstdlib>

#include "kernels.cuh"

using namespace tpx;

struct DitLayer {
    __half *Wq, *bq, *Wkv, *bkv, *Wcp, *bcp, *Wqkv, *bqkv, *Wsp, *bsp, *W1, *b1, *W2, *b2;
};

struct tpx_dit {
    int N, Cin, Cout, Dc, D, L, H, Dm, Dh, DhP, Ltot;
    ParamStore params;
    std::vector<DitLayer> layers;
    __half *Wada, *bada;                  // [L*9D + 2D, D], [L*9D + 2D]
    __half *null16, *Wx, *bx, *Wt0, *bt0, *Wt2, *bt2, *Wfl, *bfl;
    __half *uconst;                       // [L, D] : proj(to_v(null)) per block
    __half *tmp_v;                        // [D]
    bool has_null = false;                // null_cond_embedding given (cond_drop_prob > 0 models only; dit_crossattn.py:143-146)
    // conditioning store
    __half *ck = nullptr, *cv = nullptr, *y16 = nullptr;
    int cond_n = 0, cond_M = 0, cond_MP = 0;
    bool tc_attn = false;                 // wgmma attention (Dh == 72, N % 8 == 0); V kept transposed
    // timestep table (tpx_dit_set_timesteps): modulation rows [K, Ltot] of a sampling schedule's timesteps, in caller memory
    __half* ts_table = nullptr;
    std::vector<long long> ts_values;
};

namespace {
// The parameter store, keyed by the reference's state_dict names.  Optional: null_cond_embedding (only models with cond_drop_prob > 0
// have it) and the attention biases (absent with attn_proj_bias = False; the rest stay zero).
void declare_params(tpx_dit* h, ParamStore& s) {
    const int64_t D = h->D, Dc = h->Dc, Dm = h->Dm;
    const auto prefix = [h](int i) { return i < h->L ? "blocks." + std::to_string(i) + "." : std::string("final_layer."); };
    h->layers.resize(h->L);
    for (int i = 0; i < h->L; ++i) {
        DitLayer& l = h->layers[i];
        const std::string p = prefix(i);
        s.weight_bias(p + "crossattn.to_q", l.Wq, l.bq, {D, D}, PK_PLAIN, false);
        l.Wkv = s.take(2 * D * Dc);       // to_k rows, then to_v rows: one GEMM computes both
        l.bkv = s.take(2 * D);
        s.weight_bias_at(p + "crossattn.to_k", l.Wkv, l.bkv, {D, Dc}, PK_PLAIN, false);
        s.weight_bias_at(p + "crossattn.to_v", l.Wkv + D * Dc, l.bkv + D, {D, Dc}, PK_PLAIN, false);
        s.weight_bias(p + "crossattn.proj", l.Wcp, l.bcp, {D, D}, PK_PLAIN, false);
        s.weight_bias(p + "attn.qkv", l.Wqkv, l.bqkv, {3 * D, D}, PK_PLAIN, false);
        s.weight_bias(p + "attn.proj", l.Wsp, l.bsp, {D, D}, PK_PLAIN, false);
        s.weight_bias(p + "mlp.fc1", l.W1, l.b1, {Dm, D});
        s.weight_bias(p + "mlp.fc2", l.W2, l.b2, {D, Dm});
    }
    // every block's adaLN rows (9D each), then the final layer's 2D: one GEMV computes all modulations of a step
    h->Wada = s.take(static_cast<size_t>(h->Ltot) * D);
    h->bada = s.take(h->Ltot);
    for (int i = 0; i <= h->L; ++i)
        s.weight_bias_at(prefix(i) + "adaLN_modulation.1", h->Wada + static_cast<size_t>(i) * 9 * D * D, h->bada + static_cast<size_t>(i) * 9 * D,
                         {i < h->L ? 9 * D : 2 * D, D});
    h->null16 = s.param("null_cond_embedding", {Dc}, PK_PLAIN, false);
    s.weight_bias("x_embedder", h->Wx, h->bx, {D, h->Cin});
    s.weight_bias("t_embedder.mlp.0", h->Wt0, h->bt0, {D, 256});
    s.weight_bias("t_embedder.mlp.2", h->Wt2, h->bt2, {D, D});
    s.weight_bias("final_layer.linear", h->Wfl, h->bfl, {h->Cout, D});
    h->uconst = s.take(static_cast<size_t>(h->L) * D);
    h->tmp_v = s.take(D);
}

struct DitWs {
    float* xres;
    __half *h16, *q, *k, *v, *ao, *hid, *mod, *ts16, *fin;
    float *th1, *temb;
    size_t total;
};

DitWs carve_ws(const tpx_dit* h, int S, void* base) {
    Carve c{static_cast<uint8_t*>(base)};
    DitWs w;
    const size_t T = static_cast<size_t>(S) * h->N;
    w.xres = c.take<float>(T * h->D);
    w.h16 = c.take<__half>(T * h->D);
    const size_t hb = static_cast<size_t>(S) * h->H * h->N * h->DhP;
    w.q = c.take<__half>(hb);
    w.k = c.take<__half>(hb);
    w.v = c.take<__half>(hb);
    w.ao = c.take<__half>(T * h->D);
    w.hid = c.take<__half>(T * h->Dm);
    w.mod = c.take<__half>(static_cast<size_t>(S) * h->Ltot);
    w.ts16 = c.take<__half>(static_cast<size_t>(S) * h->D);
    w.fin = c.take<__half>(T * h->Cout);
    w.th1 = c.take<float>(static_cast<size_t>(S) * h->D);
    w.temb = c.take<float>(static_cast<size_t>(S) * h->D);
    w.total = c.off;
    return w;
}

// Conditioning store: K and V of every block's cross-attention, then the fp16 conditioning
struct CondWs {
    __half *ck, *cv, *y16;
    int MP;                        // key count padded for the transposed V (TMA row pitch must be a multiple of 16 B)
    size_t total;
};

CondWs carve_cond(const tpx_dit* h, int n_cross, int M, void* base) {
    Carve c{static_cast<uint8_t*>(base)};
    CondWs w;
    w.MP = (M + 7) & ~7;
    const size_t kv = static_cast<size_t>(h->L) * n_cross * h->H * w.MP * h->DhP;
    w.ck = c.take<__half>(kv);
    w.cv = c.take<__half>(kv);
    w.y16 = c.take<__half>(static_cast<size_t>(n_cross) * M * h->Dc);
    w.total = c.off;
    return w;
}

// Timestep table: [K, Ltot] fp16 modulation rows | K int64 timesteps (device copy) | scratch of one chunk of TS_CHUNK timesteps
constexpr int TS_CHUNK = 8;    // = the batched GEMV's maximum batch: the adaLN weights are streamed once per 8 timesteps
constexpr int TS_MAX = 4096;
struct TsWs {
    __half* table;
    long long* t_dev;
    float *th1, *temb;
    __half* ts16;
    size_t total;
};

TsWs carve_ts(const tpx_dit* h, int K, void* base) {
    Carve c{static_cast<uint8_t*>(base)};
    TsWs w;
    w.table = c.take<__half>(static_cast<size_t>(K) * h->Ltot);
    w.t_dev = c.take<long long>(K);
    w.th1 = c.take<float>(static_cast<size_t>(TS_CHUNK) * h->D);
    w.temb = c.take<float>(static_cast<size_t>(TS_CHUNK) * h->D);
    w.ts16 = c.take<__half>(static_cast<size_t>(TS_CHUNK) * h->D);
    w.total = c.off;
    return w;
}

}  // namespace

extern "C" {

int tpx_dit_create(const tpx_dit_config* c, tpx_dit** out) {
    TPX_CHECK(c != nullptr && out != nullptr, TPX_ERR_ARG, "dit_create: null argument");
    TPX_CHECK(c->hidden_size % 128 == 0 && c->hidden_size <= 2048, TPX_ERR_SHAPE, "dit_create: hidden_size %d must be a multiple of 128 (<= 2048)", c->hidden_size);
    TPX_CHECK(c->num_heads > 0 && c->hidden_size % c->num_heads == 0, TPX_ERR_SHAPE, "dit_create: hidden %d not divisible by heads %d", c->hidden_size, c->num_heads);
    const int Dh = c->hidden_size / c->num_heads;
    TPX_CHECK(Dh % 8 == 0 && Dh <= 128, TPX_ERR_SHAPE, "dit_create: head dim %d must be a multiple of 8 and <= 128", Dh);
    TPX_CHECK(c->condition_channels % 8 == 0 && c->mlp_hidden % 8 == 0 && c->out_channels % 8 == 0, TPX_ERR_SHAPE,
              "dit_create: condition/mlp/out channels must be multiples of 8 (%d/%d/%d)", c->condition_channels, c->mlp_hidden, c->out_channels);
    TPX_CHECK(c->depth > 0 && c->seq_length > 0 && c->in_channels > 0, TPX_ERR_SHAPE, "dit_create: non-positive size");
    TPX_CHECK(c->in_channels % 4 == 0, TPX_ERR_SHAPE, "dit_create: in_channels %d must be a multiple of 4", c->in_channels);
    TPX_DEVICE_GUARD();
    tpx_dit* h = new tpx_dit();
    h->N = c->seq_length; h->Cin = c->in_channels; h->Cout = c->out_channels; h->Dc = c->condition_channels;
    h->D = c->hidden_size; h->L = c->depth; h->H = c->num_heads; h->Dm = c->mlp_hidden; h->Dh = Dh;
    h->DhP = Dh <= 16 ? 16 : (Dh <= 32 ? 32 : (Dh <= 64 ? 64 : (Dh <= 80 ? 80 : 128)));
    h->Ltot = h->L * 9 * h->D + 2 * h->D;
    h->tc_attn = (h->Dh == 72 && h->N % 8 == 0);   // the wgmma kernel's 80-wide tiles
    const int rc = h->params.create(16, [h](ParamStore& s) { declare_params(h, s); });
    if (rc != TPX_OK) { delete h; return rc; }
    *out = h;
    return TPX_OK;
}

void tpx_dit_destroy(tpx_dit* h) { delete h; }

int tpx_dit_set_weight(tpx_dit* h, const char* ref_key, const void* dev_ptr, int dtype, const int64_t* shape, int ndim, void* stream) {
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "dit_set_weight: null argument");
    const int rc = h->params.set("dit_set_weight", ref_key, dev_ptr, dtype, shape, ndim, static_cast<cudaStream_t>(stream));
    if (rc != TPX_OK) return rc;
    h->has_null = h->params.seen(h->null16);
    h->ts_values.clear();       // a timestep table derived from the previous weights is stale
    h->ts_table = nullptr;
    return TPX_OK;
}

int tpx_dit_get_weight(tpx_dit* h, const char* ref_key, void* dst_dev, int dtype, void* stream) {
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "dit_get_weight: null argument");
    return h->params.get("dit_get_weight", ref_key, dst_dev, dtype, static_cast<cudaStream_t>(stream));
}

int tpx_dit_finalize(tpx_dit* h, void* stream) {
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "dit_finalize: null handle");
    int rc = h->params.complete("dit_finalize");
    if (rc != TPX_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // per-block constant of cross-attention against an all-null context: h(Wp . h(Wv . null + bv) + bp)
    for (int i = 0; h->has_null && i < h->L; ++i) {
        const DitLayer& l = h->layers[i];
        rc = launch_gemv(GEMV_IN_F16, GEMV_OUT_F16, l.Wkv + static_cast<size_t>(h->D) * h->Dc, l.bkv + h->D, h->null16, nullptr, 1, h->D, h->Dc,
                         h->tmp_v, nullptr, h->D, st);
        if (rc != TPX_OK) return rc;
        rc = launch_gemv(GEMV_IN_F16, GEMV_OUT_F16, l.Wcp, l.bcp, h->tmp_v, nullptr, 1, h->D, h->D, h->uconst + static_cast<size_t>(i) * h->D, nullptr,
                         h->D, st);
        if (rc != TPX_OK) return rc;
    }
    h->params.finalized = true;
    return TPX_OK;
}

size_t tpx_dit_cond_bytes(const tpx_dit* h, int n_cross, int M) {
    if (h == nullptr || n_cross <= 0 || M <= 0) return 0;
    return carve_cond(h, n_cross, M, nullptr).total;
}

size_t tpx_dit_workspace_bytes(const tpx_dit* h, int n_seq) {
    if (h == nullptr || n_seq <= 0) return 0;
    return carve_ws(h, n_seq, nullptr).total;
}

int tpx_dit_set_cond(tpx_dit* h, const float* y, int n_cross, int M, void* cond_ws, size_t cond_bytes, void* stream) {
    TPX_CHECK(h != nullptr && y != nullptr && cond_ws != nullptr, TPX_ERR_ARG, "dit_set_cond: null argument");
    TPX_CHECK(h->params.finalized, TPX_ERR_STATE, "dit_set_cond: weights not finalized (load_state_dict first)");
    TPX_CHECK(n_cross > 0 && M > 0, TPX_ERR_SHAPE, "dit_set_cond: empty conditioning (%d x %d)", n_cross, M);
    TPX_CHECK(cond_bytes >= tpx_dit_cond_bytes(h, n_cross, M), TPX_ERR_ARG, "dit_set_cond: conditioning store too small (%zu < %zu)", cond_bytes,
              tpx_dit_cond_bytes(h, n_cross, M));
    TPX_CHECK((reinterpret_cast<uintptr_t>(cond_ws) & 255) == 0, TPX_ERR_ARG, "dit_set_cond: store must be 256-B aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const CondWs w = carve_cond(h, n_cross, M, cond_ws);
    h->ck = w.ck;
    h->cv = w.cv;
    h->y16 = w.y16;
    h->cond_n = n_cross;
    h->cond_M = M;
    h->cond_MP = w.MP;
    // key columns [M, MP) of the transposed V must be finite
    if (h->tc_attn) TPX_CUDA(cudaMemsetAsync(h->cv, 0, reinterpret_cast<uint8_t*>(h->y16) - reinterpret_cast<uint8_t*>(h->cv), st));
    int rc = launch_to_half(y, TPX_DTYPE_F32, h->y16, static_cast<long long>(n_cross) * M * h->Dc, st);
    if (rc != TPX_OK) return rc;
    const size_t per_layer = static_cast<size_t>(n_cross) * h->H * M * h->DhP;
    const size_t per_layer_v = h->tc_attn ? static_cast<size_t>(n_cross) * h->H * h->cond_MP * h->DhP : per_layer;
    for (int i = 0; i < h->L; ++i) {
        GemmArgs a{};
        a.bias = h->layers[i].bkv;
        a.post_scale = 1.0f;
        a.out0 = h->ck + i * per_layer;
        a.out1 = h->cv + i * per_layer_v;
        a.split_cols = h->D; a.Dh = h->Dh; a.DhP = h->DhP; a.H = h->H; a.Nseq = M;
        if (h->tc_attn) { a.vt_which_plus1 = 2; a.vt_ld = h->cond_MP; }
        rc = gemm_linear(h->y16, h->Dc, h->layers[i].Wkv, n_cross * M, 2 * h->D, h->Dc, EPI_HEADS, a, 0, st);
        if (rc != TPX_OK) return rc;
    }
    return TPX_OK;
}

// One forward.  The modulation vectors of the step come either from `t` (device timesteps: timestep MLP + the adaLN GEMV pass run here and
// fill the workspace's [B, Ltot] table) or, when `t` is null, from `mod_rows` = one precomputed row shared by the whole batch (tpx_dit_forward_step).
// stop_stage < 0 runs the whole schedule and writes `out`; stop_stage = TPX_DIT_STAGE_* returns right after that stage of block stop_block
// (tpx_dit_debug_stage) and leaves the workspace as it stands.  Both run the same launches up to the stop.
static int dit_forward_impl(tpx_dit* h, const float* x, const int64_t* t, const __half* mod_rows, int B, int use_cfg, float cfg_scale, void* out, void* ws,
                            size_t ws_bytes, void* stream, int stop_block = -1, int stop_stage = -1) {
    TPX_CHECK(h != nullptr && x != nullptr && (t != nullptr || mod_rows != nullptr) && (out != nullptr || stop_stage >= 0) && ws != nullptr, TPX_ERR_ARG,
              "dit_forward: null argument");
    TPX_CHECK(h->params.finalized, TPX_ERR_STATE, "dit_forward: weights not finalized");
    TPX_CHECK(B >= 1 && B <= 8, TPX_ERR_SHAPE, "dit_forward: batch %d must be in [1,8]", B);
    TPX_CHECK(use_cfg >= 0 && use_cfg <= 2, TPX_ERR_ARG, "dit_forward: use_cfg %d", use_cfg);
    TPX_CHECK(use_cfg == 0 || h->has_null, TPX_ERR_STATE, "dit_forward: classifier-free guidance needs null_cond_embedding (model built with cond_drop_prob = 0)");
    const int S = use_cfg ? 2 * B : B;       // sequences in the batch
    const int Sc = use_cfg == 1 ? B : S;     // leading sequences with real cross-attention
    TPX_CHECK(h->ck != nullptr && h->cond_n == Sc, TPX_ERR_STATE, "dit_forward: conditioning holds %d sequences, this call needs %d (call set_cond)",
              h->cond_n, Sc);
    TPX_CHECK(ws_bytes >= tpx_dit_workspace_bytes(h, S), TPX_ERR_ARG, "dit_forward: workspace too small (%zu < %zu)", ws_bytes,
              tpx_dit_workspace_bytes(h, S));
    TPX_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, TPX_ERR_ARG, "dit_forward: workspace must be 256-B aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const DitWs w = carve_ws(h, S, ws);
    const int N = h->N, D = h->D, Ltot = h->Ltot, M = h->cond_M;
    const float qscale = 1.0f / sqrtf(static_cast<float>(h->Dh));
    int rc;
    static const bool dbg_sync = getenv("TPX_DEBUG_SYNC") != nullptr && getenv("TPX_DEBUG_SYNC")[0] == '1';
    int op_index = 0;
#define TPX_RC(call)                                                                                              \
    do {                                                                                                          \
        rc = (call);                                                                                              \
        if (rc != TPX_OK) return rc;                                                                              \
        if (dbg_sync) {                                                                                           \
            fprintf(stderr, "[tpx] op %d: %s\n", op_index, #call);                                               \
            fflush(stderr);                                                                                       \
            TPX_CUDA(cudaStreamSynchronize(st));                                                                  \
        }                                                                                                         \
        ++op_index;                                                                                               \
    } while (0)

    // The head-split GEMM epilogues write only the Dh real columns of each 80-wide head row (24-column bulk stores); the padding
    // columns / rows of q, k, v(T) must be zero, so the three buffers (contiguous in the workspace) are cleared once per forward.
    TPX_CUDA(cudaMemsetAsync(w.q, 0, reinterpret_cast<uint8_t*>(w.ao) - reinterpret_cast<uint8_t*>(w.q), st));
    // timestep embedding (fp32) -> silu -> fp16, then every adaLN modulation of the network in one GEMV pass — unless the row of this
    // step was hoisted out of the sampling loop (tpx_dit_set_timesteps): then the whole batch reads that one row (batch stride 0)
    const __half* mod_base = w.mod;
    int mod_bs = Ltot;
    if (t != nullptr) {
        TPX_RC(launch_gemv(GEMV_IN_TIMESTEP, GEMV_OUT_F32_SILU, h->Wt0, h->bt0, nullptr, reinterpret_cast<const long long*>(t), B, D, 256, w.th1, nullptr, D, st));
        TPX_RC(launch_gemv(GEMV_IN_F32, GEMV_OUT_F32_AND_SILU16, h->Wt2, h->bt2, w.th1, nullptr, B, D, D, w.temb, w.ts16, D, st));
        TPX_RC(launch_gemv(GEMV_IN_F16, GEMV_OUT_F16, h->Wada, h->bada, w.ts16, nullptr, B, Ltot, D, w.mod, nullptr, Ltot, st));
    } else {
        mod_base = mod_rows;
        mod_bs = 0;
    }
    // token embedding, fp32, written to both CFG halves
    TPX_RC(launch_x_embed(x, h->Wx, h->bx, B * N, h->Cin, D, w.xres, use_cfg ? static_cast<long long>(B) * N * D : 0, st));
    if (stop_stage == TPX_DIT_STAGE_EMBED) return TPX_OK;

    const size_t per_layer_kv = static_cast<size_t>(h->cond_n) * h->H * M * h->DhP;
    const size_t per_layer_v = h->tc_attn ? static_cast<size_t>(h->cond_n) * h->H * h->cond_MP * h->DhP : per_layer_kv;
    for (int i = 0; i < h->L; ++i) {
        const DitLayer& l = h->layers[i];
        const __half* mod = mod_base + static_cast<size_t>(i) * 9 * D;   // (shift,scale,gate) x (mca,msa,mlp)
        // ---- cross-attention branch (sequences [0,Sc)) ----
        TPX_RC(launch_ln_modulate(w.xres, Sc * N, D, 1e-6f, mod + 0 * D, mod + 1 * D, mod_bs, N, B, w.h16, nullptr, nullptr, 0, st));
        {
            GemmArgs a{};
            a.bias = l.bq; a.post_scale = qscale; a.out0 = w.q;
            a.split_cols = D; a.Dh = h->Dh; a.DhP = h->DhP; a.H = h->H; a.Nseq = N; a.heads_tma = 1;
            TPX_RC(gemm_linear(w.h16, D, l.Wq, Sc * N, D, D, EPI_HEADS, a, D % 144 == 0 && h->Dh % 24 == 0 && N % 32 == 0 ? 144 : 0, st));
        }
        if (h->tc_attn) TPX_RC(launch_attention_tc(w.q, h->ck + i * per_layer_kv, h->cv + i * per_layer_v, w.ao, Sc, h->H, N, M, h->cond_MP, h->Dh, qscale, st));
        else TPX_RC(launch_attention(w.q, h->ck + i * per_layer_kv, h->cv + i * per_layer_kv, w.ao, Sc, h->H, N, M, h->Dh, h->DhP, qscale, st));
        {
            GemmArgs a{};
            a.bias = l.bcp; a.post_scale = 1.0f; a.xres = w.xres; a.ldx = D;
            a.gate = mod + 2 * D; a.gate_bstride = mod_bs; a.rows_per_batch = N; a.gate_batches = B;
            TPX_RC(gemm_linear(w.ao, D, l.Wcp, Sc * N, D, D, EPI_GATED, a, 0, st));
        }
        if (i == stop_block && stop_stage == TPX_DIT_STAGE_CROSS) return TPX_OK;
        // ---- self-attention branch (all sequences); the collapsed cross-attention of the null half is added here ----
        TPX_RC(launch_ln_modulate(w.xres, S * N, D, 1e-6f, mod + 3 * D, mod + 4 * D, mod_bs, N, B, w.h16, Sc < S ? mod + 2 * D : nullptr,
                                  h->uconst + static_cast<size_t>(i) * D, Sc * N, st));
        {
            GemmArgs a{};
            a.bias = l.bqkv; a.post_scale = 1.0f; a.out0 = w.q; a.out1 = w.k; a.out2 = w.v;
            a.split_cols = D; a.Dh = h->Dh; a.DhP = h->DhP; a.H = h->H; a.Nseq = N; a.heads_tma = 1;
            if (h->tc_attn) { a.vt_which_plus1 = 3; a.vt_ld = N; }
            TPX_RC(gemm_linear(w.h16, D, l.Wqkv, S * N, 3 * D, D, EPI_HEADS, a, 0, st));
        }
        if (h->tc_attn) TPX_RC(launch_attention_tc(w.q, w.k, w.v, w.ao, S, h->H, N, N, N, h->Dh, qscale, st));
        else TPX_RC(launch_attention(w.q, w.k, w.v, w.ao, S, h->H, N, N, h->Dh, h->DhP, qscale, st));
        {
            GemmArgs a{};
            a.bias = l.bsp; a.post_scale = 1.0f; a.xres = w.xres; a.ldx = D;
            a.gate = mod + 5 * D; a.gate_bstride = mod_bs; a.rows_per_batch = N; a.gate_batches = B;
            TPX_RC(gemm_linear(w.ao, D, l.Wsp, S * N, D, D, EPI_GATED, a, 0, st));
        }
        if (i == stop_block && stop_stage == TPX_DIT_STAGE_SELF) return TPX_OK;
        // ---- MLP branch ----
        TPX_RC(launch_ln_modulate(w.xres, S * N, D, 1e-6f, mod + 6 * D, mod + 7 * D, mod_bs, N, B, w.h16, nullptr, nullptr, 0, st));
        {
            GemmArgs a{};
            a.bias = l.b1; a.post_scale = 1.0f; a.out0 = w.hid; a.ldo = h->Dm;
            TPX_RC(gemm_linear(w.h16, D, l.W1, S * N, h->Dm, D, EPI_GELU, a, 0, st));
        }
        {
            GemmArgs a{};
            a.bias = l.b2; a.post_scale = 1.0f; a.xres = w.xres; a.ldx = D;
            a.gate = mod + 8 * D; a.gate_bstride = mod_bs; a.rows_per_batch = N; a.gate_batches = B;
            TPX_RC(gemm_linear(w.hid, h->Dm, l.W2, S * N, D, h->Dm, EPI_GATED, a, 0, st));
        }
        if (i == stop_block && stop_stage == TPX_DIT_STAGE_MLP) return TPX_OK;
    }
    // ---- final layer ----
    const __half* fmod = mod_base + static_cast<size_t>(h->L) * 9 * D;
    TPX_RC(launch_ln_modulate(w.xres, S * N, D, 1e-6f, fmod, fmod + D, mod_bs, N, B, w.h16, nullptr, nullptr, 0, st));
    {
        GemmArgs a{};
        a.bias = h->bfl; a.post_scale = 1.0f; a.out0 = use_cfg ? w.fin : static_cast<__half*>(out); a.ldo = h->Cout;
        TPX_RC(gemm_linear(w.h16, D, h->Wfl, S * N, h->Cout, D, EPI_STORE, a, 128, st));
    }
    if (use_cfg) TPX_RC(launch_cfg_combine(w.fin, static_cast<long long>(B) * N * h->Cout, cfg_scale, static_cast<__half*>(out), st));
#undef TPX_RC
    return TPX_OK;
}

int tpx_dit_forward(tpx_dit* h, const float* x, const int64_t* t, int B, int use_cfg, float cfg_scale, void* out, void* ws, size_t ws_bytes,
                    void* stream) {
    TPX_CHECK(t != nullptr, TPX_ERR_ARG, "dit_forward: null timesteps");
    return dit_forward_impl(h, x, t, nullptr, B, use_cfg, cfg_scale, out, ws, ws_bytes, stream);
}

size_t tpx_dit_timesteps_bytes(const tpx_dit* h, int K) {
    if (h == nullptr || K <= 0 || K > TS_MAX) return 0;
    return carve_ts(h, K, nullptr).total;
}

int tpx_dit_set_timesteps(tpx_dit* h, const int64_t* t_host, int K, void* ts_ws, size_t ts_bytes, void* stream) {
    TPX_CHECK(h != nullptr && t_host != nullptr && ts_ws != nullptr, TPX_ERR_ARG, "dit_set_timesteps: null argument");
    TPX_CHECK(h->params.finalized, TPX_ERR_STATE, "dit_set_timesteps: weights not finalized (load_state_dict first)");
    TPX_CHECK(K >= 1 && K <= TS_MAX, TPX_ERR_SHAPE, "dit_set_timesteps: %d timesteps (1..%d)", K, TS_MAX);
    TPX_CHECK(ts_bytes >= tpx_dit_timesteps_bytes(h, K), TPX_ERR_ARG, "dit_set_timesteps: table store too small (%zu < %zu)", ts_bytes,
              tpx_dit_timesteps_bytes(h, K));
    TPX_CHECK((reinterpret_cast<uintptr_t>(ts_ws) & 255) == 0, TPX_ERR_ARG, "dit_set_timesteps: store must be 256-B aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const TsWs w = carve_ts(h, K, ts_ws);
    h->ts_values.clear();
    h->ts_table = nullptr;
    // pageable source: the driver stages the values before the call returns, so t_host need not outlive it
    TPX_CUDA(cudaMemcpyAsync(w.t_dev, t_host, static_cast<size_t>(K) * 8, cudaMemcpyHostToDevice, st));
    const int D = h->D, Ltot = h->Ltot;
    for (int c = 0; c < K; c += TS_CHUNK) {
        const int nb = K - c < TS_CHUNK ? K - c : TS_CHUNK;
        // the same three launches a forward issues for its batch (utils.py:27-64, dit_crossattn.py:54,75), over 8 timesteps at once:
        // per output element the arithmetic does not depend on the batch it runs in, so a row equals what tpx_dit_forward computes
        int rc = launch_gemv(GEMV_IN_TIMESTEP, GEMV_OUT_F32_SILU, h->Wt0, h->bt0, nullptr, w.t_dev + c, nb, D, 256, w.th1, nullptr, D, st);
        if (rc != TPX_OK) return rc;
        rc = launch_gemv(GEMV_IN_F32, GEMV_OUT_F32_AND_SILU16, h->Wt2, h->bt2, w.th1, nullptr, nb, D, D, w.temb, w.ts16, D, st);
        if (rc != TPX_OK) return rc;
        rc = launch_gemv(GEMV_IN_F16, GEMV_OUT_F16, h->Wada, h->bada, w.ts16, nullptr, nb, Ltot, D, w.table + static_cast<size_t>(c) * Ltot, nullptr, Ltot, st);
        if (rc != TPX_OK) return rc;
    }
    h->ts_values.assign(t_host, t_host + K);
    h->ts_table = w.table;
    return TPX_OK;
}

int tpx_dit_forward_step(tpx_dit* h, const float* x, int64_t t, int B, int use_cfg, float cfg_scale, void* out, void* ws, size_t ws_bytes, void* stream) {
    TPX_CHECK(h != nullptr, TPX_ERR_ARG, "dit_forward_step: null handle");
    TPX_CHECK(h->ts_table != nullptr && !h->ts_values.empty(), TPX_ERR_STATE, "dit_forward_step: no timestep table (call tpx_dit_set_timesteps after loading weights)");
    size_t row = h->ts_values.size();
    for (size_t i = 0; i < h->ts_values.size(); ++i)
        if (h->ts_values[i] == static_cast<long long>(t)) { row = i; break; }
    TPX_CHECK(row < h->ts_values.size(), TPX_ERR_STATE, "dit_forward_step: timestep %lld is not in the table given to tpx_dit_set_timesteps", (long long)t);
    return dit_forward_impl(h, x, nullptr, h->ts_table + row * static_cast<size_t>(h->Ltot), B, use_cfg, cfg_scale, out, ws, ws_bytes, stream);
}

int tpx_dit_debug_stage(tpx_dit* h, const float* x, const int64_t* t, int B, int use_cfg, int block, int stage, void* ws, size_t ws_bytes, void* stream) {
    TPX_CHECK(stage >= TPX_DIT_STAGE_EMBED && stage <= TPX_DIT_STAGE_MLP, TPX_ERR_ARG, "dit_debug_stage: bad stage %d", stage);
    TPX_CHECK(h != nullptr && t != nullptr, TPX_ERR_ARG, "dit_debug_stage: null argument");
    TPX_CHECK(stage == TPX_DIT_STAGE_EMBED || (block >= 0 && block < h->L), TPX_ERR_ARG, "dit_debug_stage: bad block %d (depth %d)", block, h->L);
    return dit_forward_impl(h, x, t, nullptr, B, use_cfg, 0.0f, nullptr, ws, ws_bytes, stream, stage == TPX_DIT_STAGE_EMBED ? -1 : block, stage);
}

int tpx_dit_debug_tap(const tpx_dit* h, const void* ws, int n_seq, int which, int count, void* dst, void* stream) {
    TPX_CHECK(which >= TPX_DIT_TAP_RESIDUAL && which <= TPX_DIT_TAP_PRE_CFG, TPX_ERR_ARG, "dit_debug_tap: bad tap %d", which);
    TPX_CHECK(n_seq >= 1 && count >= 1 && count <= n_seq, TPX_ERR_ARG, "dit_debug_tap: count %d must be in [1, n_seq = %d]", count, n_seq);
    TPX_CHECK(h != nullptr && ws != nullptr && dst != nullptr, TPX_ERR_ARG, "dit_debug_tap: null argument");
    const DitWs w = carve_ws(h, n_seq, const_cast<void*>(ws));
    const size_t T = static_cast<size_t>(count) * h->N;
    const void* src = which == TPX_DIT_TAP_RESIDUAL ? static_cast<const void*>(w.xres)
                      : which == TPX_DIT_TAP_ATTN_OUT ? static_cast<const void*>(w.ao)
                      : which == TPX_DIT_TAP_MOD    ? static_cast<const void*>(w.mod)
                                                    : static_cast<const void*>(w.fin);
    const size_t bytes = which == TPX_DIT_TAP_RESIDUAL ? T * h->D * 4
                         : which == TPX_DIT_TAP_ATTN_OUT ? T * h->D * 2
                         : which == TPX_DIT_TAP_MOD    ? static_cast<size_t>(count) * h->Ltot * 2
                                                       : T * h->Cout * 2;
    TPX_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    return TPX_OK;
}

}  // extern "C"
