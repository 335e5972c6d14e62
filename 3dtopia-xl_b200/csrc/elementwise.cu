// HBM-bound kernels of the DiT step and the sampler: LayerNorm+adaLN-modulate, adaLN GEMV, timestep
// embedder, token embedder, CFG combine, fused DDIM / DDPM update, dtype conversion.
// All are warp-shuffle / 16-byte-vectorised SIMT kernels; none is GEMM shaped enough for tensor cores.
#include "kernels.cuh"

namespace tpx {

// =====================================================================================================
// LayerNorm(eps, no affine) + modulate -> fp16      (reference: dit_crossattn.py:55-57, utils.py:19-20)
//   y = LN(x) * float(h(1 + scale16)) + float(shift16)   -> fp16 (the cast autocast applies at the next Linear)
// One warp per token row; the row (<= 2048 floats) lives in registers.  Optional fused pre-add for the
// "uncond" rows of a CFG batch: x += h(gate16 * const16) (the collapsed cross-attention branch).
// =====================================================================================================
constexpr int LN_MAX_ITERS = 16;  // D <= 2048

template <int NI>   // NI = D / 128 float4 per lane: the row lives in exactly NI*4 registers
__global__ void __launch_bounds__(256) ln_modulate_kernel(float* __restrict__ x, int rows, float eps, const __half* __restrict__ shift,
                                                          const __half* __restrict__ scale, int mod_bstride, int rows_per_batch, int mod_batches,
                                                          __half* __restrict__ out, const __half* __restrict__ pre_gate,
                                                          const __half* __restrict__ pre_const, int pre_row0) {
    constexpr int D = NI * 128;
    pdl_launch_dependents();
    pdl_wait();
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const int bm = (row / rows_per_batch) % mod_batches;
    float4 v[NI];
    float* xr = x + static_cast<size_t>(row) * D;
#pragma unroll
    for (int i = 0; i < NI; ++i) v[i] = *reinterpret_cast<const float4*>(xr + (lane + 32 * i) * 4);
    if (pre_gate != nullptr && row >= pre_row0) {
        const __half* gp = pre_gate + static_cast<size_t>(bm) * mod_bstride;
#pragma unroll
        for (int i = 0; i < NI; ++i) {
            const int c = (lane + 32 * i) * 4;
            const __half2 g0 = *reinterpret_cast<const __half2*>(gp + c), g1 = *reinterpret_cast<const __half2*>(gp + c + 2);
            const __half2 c0 = *reinterpret_cast<const __half2*>(pre_const + c), c1 = *reinterpret_cast<const __half2*>(pre_const + c + 2);
            v[i].x += h2f_round(__low2float(g0) * __low2float(c0));
            v[i].y += h2f_round(__high2float(g0) * __high2float(c0));
            v[i].z += h2f_round(__low2float(g1) * __low2float(c1));
            v[i].w += h2f_round(__high2float(g1) * __high2float(c1));
            *reinterpret_cast<float4*>(xr + c) = v[i];
        }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NI; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) * (1.0f / D);
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < NI; ++i) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float rstd = rsqrtf(warp_sum(q) * (1.0f / D) + eps);
    const __half* shp = shift + static_cast<size_t>(bm) * mod_bstride;
    const __half* scp = scale + static_cast<size_t>(bm) * mod_bstride;
    __half* orow = out + static_cast<size_t>(row) * D;
#pragma unroll
    for (int i = 0; i < NI; ++i) {
        const int c = (lane + 32 * i) * 4;
        const uint2 shv = __ldg(reinterpret_cast<const uint2*>(shp + c)), scv = __ldg(reinterpret_cast<const uint2*>(scp + c));
        const __half2 sh0 = *reinterpret_cast<const __half2*>(&shv.x), sh1 = *reinterpret_cast<const __half2*>(&shv.y);
        const __half2 sc0 = *reinterpret_cast<const __half2*>(&scv.x), sc1 = *reinterpret_cast<const __half2*>(&scv.y);
        const float m0 = h2f_round(1.0f + __low2float(sc0)), m1 = h2f_round(1.0f + __high2float(sc0));
        const float m2 = h2f_round(1.0f + __low2float(sc1)), m3 = h2f_round(1.0f + __high2float(sc1));
        const float y0 = (v[i].x - mean) * rstd * m0 + __low2float(sh0);
        const float y1 = (v[i].y - mean) * rstd * m1 + __high2float(sh0);
        const float y2 = (v[i].z - mean) * rstd * m2 + __low2float(sh1);
        const float y3 = (v[i].w - mean) * rstd * m3 + __high2float(sh1);
        __half2 o0 = __floats2half2_rn(y0, y1), o1 = __floats2half2_rn(y2, y3);
        uint2 pk;
        pk.x = *reinterpret_cast<uint32_t*>(&o0);
        pk.y = *reinterpret_cast<uint32_t*>(&o1);
        *reinterpret_cast<uint2*>(orow + c) = pk;
    }
}

int launch_ln_modulate(float* x, int rows, int D, float eps, const __half* shift, const __half* scale, int mod_bstride, int rows_per_batch,
                       int mod_batches, __half* out, const __half* pre_gate, const __half* pre_const, int pre_row0, cudaStream_t st) {
    TPX_CHECK(D % 128 == 0 && D <= 128 * LN_MAX_ITERS, TPX_ERR_SHAPE, "ln_modulate: hidden size %d must be a multiple of 128 and <= %d", D, 128 * LN_MAX_ITERS);
    if (rows <= 0) return TPX_OK;
    ProfScope prof(PROF_LN, st);
    const dim3 grid((rows + 7) / 8), block(256);
#define TPX_LN_CASE(NI_)                                                                                                                         \
    case NI_:                                                                                                                                    \
        TPX_CUDA(launch_pdl(ln_modulate_kernel<NI_>, grid, block, 0, st, x, rows, eps, shift, scale, mod_bstride, rows_per_batch, mod_batches, out, \
                            pre_gate, pre_const, pre_row0));                                                                                     \
        break;
    switch (D / 128) {
        TPX_LN_CASE(1) TPX_LN_CASE(2) TPX_LN_CASE(3) TPX_LN_CASE(4) TPX_LN_CASE(5) TPX_LN_CASE(6) TPX_LN_CASE(7) TPX_LN_CASE(8)
        TPX_LN_CASE(9) TPX_LN_CASE(10) TPX_LN_CASE(11) TPX_LN_CASE(12) TPX_LN_CASE(13) TPX_LN_CASE(14) TPX_LN_CASE(15) TPX_LN_CASE(16)
    }
#undef TPX_LN_CASE
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

// =====================================================================================================
// Batched GEMV: out[b, j] = act( W[j,:] . in[b,:] + bias[j] ),  W fp16 [J,K], one warp per output row j,
// all b (<= 8) at once so each weight byte is read from HBM exactly once.
//   IN_TIMESTEP : in[b,:] = [cos(t_b f_k), sin(t_b f_k)] (utils.py:41-59), K = 256
//   IN_F32      : in fp32 [B,K]
//   IN_F16      : in fp16 [B,K]  (rounded like an autocast Linear input)
//   OUT_F32 / OUT_F32_SILU / OUT_F16 (single rounding h(acc+bias))
// Used for: t_embedder (2 launches), adaLN modulation of all 28 blocks + final layer in ONE launch
// (669 MB of fp16 weights per step at the shipped size: the HBM-bound part of a step), and the
// uncond cross-attention constants.
// =====================================================================================================
constexpr int GEMV_MAXB = 8;
enum { IN_TIMESTEP = GEMV_IN_TIMESTEP, IN_F32 = GEMV_IN_F32, IN_F16 = GEMV_IN_F16 };
enum { OUT_F32 = GEMV_OUT_F32, OUT_F32_SILU = GEMV_OUT_F32_SILU, OUT_F16 = GEMV_OUT_F16, OUT_F16_SILU_ALSO = GEMV_OUT_F32_AND_SILU16 };

constexpr int GEMV_R = 4;  // output rows per warp (input vector registers reused across them)

template <int IN, int OUT>
__global__ void __launch_bounds__(256) gemv_kernel(const __half* __restrict__ W, const __half* __restrict__ bias, const void* __restrict__ in_,
                                                   const long long* __restrict__ tsteps, int B, int J, int K, void* __restrict__ out_,
                                                   __half* __restrict__ out_silu16, int out_ld) {
    // input staged as fp32 in a lane-major permuted layout [b][it][part][lane][4] so that every lane's
    // 8 consecutive k-values are two conflict-free float4 reads.
    extern __shared__ float s_in[];
    const int nit = (K + 255) >> 8;
    for (int i = threadIdx.x; i < B * K; i += blockDim.x) {
        const int b = i / K, k = i - b * K;
        float val;
        if constexpr (IN == IN_TIMESTEP) {
            const int half_dim = K >> 1;
            const int kk = k < half_dim ? k : k - half_dim;
            const float f = expf(-9.210340371976184f * static_cast<float>(kk) / static_cast<float>(half_dim));
            const float a = static_cast<float>(tsteps[b]) * f;
            val = k < half_dim ? cosf(a) : sinf(a);
        } else if constexpr (IN == IN_F32) {
            val = static_cast<const float*>(in_)[i];
        } else {
            val = __half2float(static_cast<const __half*>(in_)[i]);
        }
        const int it = k >> 8, ln = (k & 255) >> 3, part = (k & 7) >> 2, e = k & 3;
        s_in[((((b * nit + it) * 2 + part) * 32 + ln) << 2) + e] = val;
    }
    __syncthreads();
    const int j0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * GEMV_R;
    if (j0 >= J) return;
    const int lane = threadIdx.x & 31;
    float acc[GEMV_R][GEMV_MAXB];
#pragma unroll
    for (int r = 0; r < GEMV_R; ++r)
#pragma unroll
        for (int b = 0; b < GEMV_MAXB; ++b) acc[r][b] = 0.f;
    for (int it = 0; it < nit; ++it) {
        const int k0 = (it << 8) + lane * 8;
        if (k0 >= K) break;
        float wf[GEMV_R][8];
#pragma unroll
        for (int r = 0; r < GEMV_R; ++r) {
            Pack8 w;
            w.u = (j0 + r < J) ? __ldg(reinterpret_cast<const uint4*>(W + static_cast<size_t>(j0 + r) * K + k0)) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int i = 0; i < 8; ++i) wf[r][i] = __half2float(w.h[i]);
        }
#pragma unroll
        for (int b = 0; b < GEMV_MAXB; ++b)
            if (b < B) {
                const float4 s0 = *reinterpret_cast<const float4*>(s_in + ((((b * nit + it) * 2 + 0) * 32 + lane) << 2));
                const float4 s1 = *reinterpret_cast<const float4*>(s_in + ((((b * nit + it) * 2 + 1) * 32 + lane) << 2));
#pragma unroll
                for (int r = 0; r < GEMV_R; ++r) {
                    float a = acc[r][b];
                    a = fmaf(wf[r][0], s0.x, a); a = fmaf(wf[r][1], s0.y, a); a = fmaf(wf[r][2], s0.z, a); a = fmaf(wf[r][3], s0.w, a);
                    a = fmaf(wf[r][4], s1.x, a); a = fmaf(wf[r][5], s1.y, a); a = fmaf(wf[r][6], s1.z, a); a = fmaf(wf[r][7], s1.w, a);
                    acc[r][b] = a;
                }
            }
    }
#pragma unroll
    for (int r = 0; r < GEMV_R; ++r)
#pragma unroll
        for (int b = 0; b < GEMV_MAXB; ++b)
            if (b < B) acc[r][b] = warp_sum(acc[r][b]);
    if (lane == 0) {
#pragma unroll
        for (int r = 0; r < GEMV_R; ++r) {
            const int j = j0 + r;
            if (j >= J) break;
            const float bj = bias != nullptr ? __half2float(bias[j]) : 0.f;
#pragma unroll
            for (int b = 0; b < GEMV_MAXB; ++b) {
                if (b >= B) break;
                const float res = acc[r][b] + bj;
                const size_t o = static_cast<size_t>(b) * out_ld + j;
                if constexpr (OUT == OUT_F32) static_cast<float*>(out_)[o] = res;
                else if constexpr (OUT == OUT_F32_SILU) static_cast<float*>(out_)[o] = silu(res);
                else if constexpr (OUT == OUT_F16) static_cast<__half*>(out_)[o] = __float2half_rn(res);
                else {  // fp32 result + fp16(silu(result)) side output (input of every adaLN Linear)
                    static_cast<float*>(out_)[o] = res;
                    out_silu16[o] = __float2half_rn(silu(res));
                }
            }
        }
    }
}

template <int IN, int OUT>
static int launch_gemv_t(const __half* W, const __half* bias, const void* in, const long long* t, int B, int J, int K, void* out, __half* out2,
                         int out_ld, cudaStream_t st) {
    TPX_CHECK(B >= 1 && B <= GEMV_MAXB, TPX_ERR_SHAPE, "gemv: batch %d must be in [1,%d]", B, GEMV_MAXB);
    TPX_CHECK(K % 8 == 0, TPX_ERR_SHAPE, "gemv: K %d must be a multiple of 8", K);
    ProfScope prof(PROF_GEMV, st);
    const size_t smem = static_cast<size_t>(B) * ((K + 255) / 256) * 256 * sizeof(float);
    auto kern = gemv_kernel<IN, OUT>;
    if (smem > 48 * 1024) TPX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    kern<<<(J + 8 * GEMV_R - 1) / (8 * GEMV_R), 256, smem, st>>>(W, bias, in, t, B, J, K, out, out2, out_ld);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int launch_gemv(int in_mode, int out_mode, const __half* W, const __half* bias, const void* in, const long long* t, int B, int J, int K, void* out,
                __half* out2, int out_ld, cudaStream_t st) {
    if (in_mode == IN_TIMESTEP && out_mode == OUT_F32_SILU) return launch_gemv_t<IN_TIMESTEP, OUT_F32_SILU>(W, bias, in, t, B, J, K, out, out2, out_ld, st);
    if (in_mode == IN_F32 && out_mode == OUT_F16_SILU_ALSO) return launch_gemv_t<IN_F32, OUT_F16_SILU_ALSO>(W, bias, in, t, B, J, K, out, out2, out_ld, st);
    if (in_mode == IN_F32 && out_mode == OUT_F32) return launch_gemv_t<IN_F32, OUT_F32>(W, bias, in, t, B, J, K, out, out2, out_ld, st);
    if (in_mode == IN_F16 && out_mode == OUT_F16) return launch_gemv_t<IN_F16, OUT_F16>(W, bias, in, t, B, J, K, out, out2, out_ld, st);
    set_error("gemv: unsupported mode %d/%d", in_mode, out_mode);
    return TPX_ERR_ARG;
}

// =====================================================================================================
// x_embedder: fp32 Linear Cin -> D outside the autocast region (dit_crossattn.py:191).  out rows may be
// duplicated into a second batch half (forward_with_cfg feeds cat([x, x])).
// =====================================================================================================
constexpr int XE_ROWS = 8;
__global__ void __launch_bounds__(256) x_embed_kernel(const float* __restrict__ x, const __half* __restrict__ W, const __half* __restrict__ bias,
                                                      int rows, int Cin, int D, float* __restrict__ out, long long dup_offset) {
    extern __shared__ float4 s_x4[];  // [XE_ROWS][Cin / 4]
    float* s_x = reinterpret_cast<float*>(s_x4);
    const int r0 = blockIdx.x * XE_ROWS;
    const int nr = min(XE_ROWS, rows - r0);
    for (int i = threadIdx.x; i < XE_ROWS * Cin; i += blockDim.x) s_x[i] = i < nr * Cin ? x[static_cast<size_t>(r0) * Cin + i] : 0.f;
    __syncthreads();
    const int C4 = Cin >> 2;
    for (int j = threadIdx.x; j < D; j += blockDim.x) {
        float acc[XE_ROWS];
#pragma unroll
        for (int r = 0; r < XE_ROWS; ++r) acc[r] = 0.f;
        const uint2* wr = reinterpret_cast<const uint2*>(W + static_cast<size_t>(j) * Cin);   // Cin % 4 == 0: 8-byte aligned rows
        for (int k4 = 0; k4 < C4; ++k4) {
            const uint2 wp = wr[k4];
            const float2 wa = __half22float2(*reinterpret_cast<const __half2*>(&wp.x)), wb = __half22float2(*reinterpret_cast<const __half2*>(&wp.y));
#pragma unroll
            for (int r = 0; r < XE_ROWS; ++r) {
                const float4 xv = s_x4[r * C4 + k4];       // same address across the warp: one broadcast wavefront
                acc[r] = fmaf(xv.w, wb.y, fmaf(xv.z, wb.x, fmaf(xv.y, wa.y, fmaf(xv.x, wa.x, acc[r]))));   // k ascending, as before
            }
        }
        const float bj = __half2float(bias[j]);
#pragma unroll
        for (int r = 0; r < XE_ROWS; ++r)
            if (r < nr) {
                const float v = acc[r] + bj;
                const size_t o = static_cast<size_t>(r0 + r) * D + j;
                out[o] = v;
                if (dup_offset > 0) out[o + dup_offset] = v;
            }
    }
}

int launch_x_embed(const float* x, const __half* W, const __half* bias, int rows, int Cin, int D, float* out, long long dup_offset, cudaStream_t st) {
    if (rows <= 0) return TPX_OK;
    TPX_CHECK(Cin % 4 == 0 && (reinterpret_cast<uintptr_t>(W) & 7) == 0, TPX_ERR_SHAPE, "x_embed: in_channels %d must be a multiple of 4", Cin);
    ProfScope prof(PROF_GEMV, st);
    x_embed_kernel<<<(rows + XE_ROWS - 1) / XE_ROWS, 256, XE_ROWS * Cin * sizeof(float), st>>>(x, W, bias, rows, Cin, D, out, dup_offset);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

// =====================================================================================================
// Classifier-free guidance on ALL output channels, in fp16 like the reference (dit_crossattn.py:210-213):
//   out = h( uncond + h( s * h(cond - uncond) ) )
// =====================================================================================================
__global__ void cfg_combine_kernel(const __half* __restrict__ both, long long n_half, float s, __half* __restrict__ out) {
    const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
    if (i >= n_half) return;
    Pack8 c, u, o;
    c.u = *reinterpret_cast<const uint4*>(both + i);
    u.u = *reinterpret_cast<const uint4*>(both + n_half + i);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float cu = __half2float(u.h[k]);
        const float d = h2f_round(__half2float(c.h[k]) - cu);
        const float m = h2f_round(s * d);
        o.h[k] = __float2half_rn(cu + m);
    }
    *reinterpret_cast<uint4*>(out + i) = o.u;
}

int launch_cfg_combine(const __half* both, long long n_half, float s, __half* out, cudaStream_t st) {
    TPX_CHECK(n_half % 8 == 0, TPX_ERR_SHAPE, "cfg_combine: element count %lld must be a multiple of 8", n_half);
    const long long thr = n_half / 8;
    ProfScope prof(PROF_ELEMWISE, st);
    cfg_combine_kernel<<<static_cast<unsigned>((thr + 255) / 256), 256, 0, st>>>(both, n_half, s, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

// =====================================================================================================
// Fused sampler update (gaussian_diffusion.py:280-338, 531-578, 397-440).  One thread per latent element;
// every reference tensor op is one explicitly rounded fp32 op (no FMA contraction) so the trajectory
// tracks the reference's eager arithmetic.
// =====================================================================================================
template <typename MO>
__device__ __forceinline__ float mo_load(const MO* p, size_t i);
template <>
__device__ __forceinline__ float mo_load<__half>(const __half* p, size_t i) { return __half2float(p[i]); }
template <>
__device__ __forceinline__ float mo_load<float>(const float* p, size_t i) { return p[i]; }

template <typename MO>
__global__ void ddim_step_kernel(const float* __restrict__ x, const MO* __restrict__ mo, const float* __restrict__ noise, long long n, int C,
                                 tpx_sampler_coefs k, float* __restrict__ x_prev, float* __restrict__ x0_out) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long tok = i / C;
    const int c = static_cast<int>(i - tok * C);
    const float v = mo_load<MO>(mo, static_cast<size_t>(tok) * 2 * C + c);
    const float xt = x[i];
    float x0 = __fsub_rn(__fmul_rn(k.sqrt_ab, xt), __fmul_rn(k.sqrt_1mab, v));
    if (k.clip) x0 = fminf(fmaxf(x0, -1.f), 1.f);
    const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(k.sqrt_recip_ab, xt), x0), k.sqrt_recipm1_ab);
    float s = __fadd_rn(__fmul_rn(x0, k.c_x0), __fmul_rn(k.c_eps, eps));
    if (k.sigma != 0.f && noise != nullptr) s = __fadd_rn(s, __fmul_rn(__fmul_rn(k.nonzero, k.sigma), noise[i]));
    x_prev[i] = s;
    x0_out[i] = x0;
}

template <typename MO>
__global__ void ddpm_step_kernel(const float* __restrict__ x, const MO* __restrict__ mo, const float* __restrict__ noise, long long n, int C,
                                 tpx_sampler_coefs k, float* __restrict__ x_prev, float* __restrict__ x0_out) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long tok = i / C;
    const int c = static_cast<int>(i - tok * C);
    const size_t base = static_cast<size_t>(tok) * 2 * C + c;
    const float v = mo_load<MO>(mo, base);
    float varv = mo_load<MO>(mo, base + C);
    float frac, one_m;
    if (sizeof(MO) == 2) {  // fp16 tensor arithmetic in the reference
        frac = h2f_round(h2f_round(varv + 1.0f) * 0.5f);
        one_m = h2f_round(1.0f - frac);
    } else {
        frac = __fdiv_rn(__fadd_rn(varv, 1.0f), 2.0f);
        one_m = __fsub_rn(1.0f, frac);
    }
    const float logvar = __fadd_rn(__fmul_rn(frac, k.max_log), __fmul_rn(one_m, k.min_log));
    const float xt = x[i];
    float x0 = __fsub_rn(__fmul_rn(k.sqrt_ab, xt), __fmul_rn(k.sqrt_1mab, v));
    if (k.clip) x0 = fminf(fmaxf(x0, -1.f), 1.f);
    const float mean = __fadd_rn(__fmul_rn(k.coef1, x0), __fmul_rn(k.coef2, xt));
    const float nz = noise != nullptr ? noise[i] : 0.f;
    x_prev[i] = __fadd_rn(mean, __fmul_rn(__fmul_rn(k.nonzero, expf(__fmul_rn(0.5f, logvar))), nz));
    x0_out[i] = x0;
}


// =====================================================================================================
// dtype conversion (weight ingestion: fp32/fp16 checkpoint tensor -> packed fp16 slot; y -> fp16)
// =====================================================================================================
template <typename T>
__global__ void to_half_kernel(const T* __restrict__ src, __half* __restrict__ dst, long long n) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = __float2half_rn(static_cast<float>(src[i]));
}
template <>
__global__ void to_half_kernel<__half>(const __half* __restrict__ src, __half* __restrict__ dst, long long n) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}

int launch_to_half(const void* src, int src_dtype, __half* dst, long long n, cudaStream_t st) {
    if (n <= 0) return TPX_OK;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    if (src_dtype == TPX_DTYPE_F32) to_half_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float*>(src), dst, n);
    else if (src_dtype == TPX_DTYPE_F16) to_half_kernel<__half><<<grid, 256, 0, st>>>(static_cast<const __half*>(src), dst, n);
    else { set_error("to_half: unsupported source dtype %d", src_dtype); return TPX_ERR_ARG; }
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

// packed fp16 slot -> fp32 / fp16 tensor (state_dict() export of a handle whose host copy was released)
template <typename T>
__global__ void from_half_kernel(const __half* __restrict__ src, T* __restrict__ dst, long long n) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = static_cast<T>(__half2float(src[i]));
}
template <>
__global__ void from_half_kernel<__half>(const __half* __restrict__ src, __half* __restrict__ dst, long long n) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i];
}
int launch_from_half(const __half* src, void* dst, int dst_dtype, long long n, cudaStream_t st) {
    if (n <= 0) return TPX_OK;
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    if (dst_dtype == TPX_DTYPE_F32) from_half_kernel<float><<<grid, 256, 0, st>>>(src, static_cast<float*>(dst), n);
    else if (dst_dtype == TPX_DTYPE_F16) from_half_kernel<__half><<<grid, 256, 0, st>>>(src, static_cast<__half*>(dst), n);
    else { set_error("from_half: unsupported destination dtype %d", dst_dtype); return TPX_ERR_ARG; }
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

// rows of `src` [rows, K] broadcast of one vector: dst[r,:] = h(vec)  (null-conditioning context rows)
__global__ void fill_rows_half_kernel(const __half* __restrict__ vec, __half* __restrict__ dst, long long rows, int K) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < rows * K) dst[i] = vec[i % K];
}
int launch_fill_rows_half(const __half* vec, __half* dst, long long rows, int K, cudaStream_t st) {
    const long long n = rows * K;
    if (n <= 0) return TPX_OK;
    fill_rows_half_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(vec, dst, rows, K);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

// =====================================================================================================
// Sample -> decode glue (SURVEY §8a a13 / a15).  Index layout is the contract with PrimSDF / the ray-marcher and is
// bit-exact; the arithmetic repeats the reference's eager CUDA ops one rounding at a time (a tensor divided by a Python
// scalar is a multiplication by the fp32 reciprocal on CUDA).
//   a13  inference.py:328-332, app.py:119-123 : v = x / latent_nf * latent_std + latent_mean ; srt = v[..., 0:4], z = v[..., 4:]
//        (without per-channel statistics: srt = x[..., 0:4], z = x[..., 4:] / latent_nf ; inference.py:337)
//   a15  inference.py:343-348, app.py:134-139 : feat[:, 0] /= 5 ; feat[:, 1:] = (feat[:, 1:] + 1) / 2 ; channel-major reshape ;
//        concat [srt | feat] -> [T, 4 + 6*512]   (without per-channel statistics: srt[..., 0] = srt[..., 0] / 10 + 0.05)
// =====================================================================================================
__global__ void latent_split_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ stdv, float inv_nf,
                                    long long T, int C, float* __restrict__ srt, float* __restrict__ z) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= T * C) return;
    const long long tok = i / C;
    const int c = static_cast<int>(i - tok * C);
    float v = x[i];
    if (mean != nullptr) v = __fadd_rn(__fmul_rn(__fmul_rn(v, inv_nf), stdv[c]), mean[c]);
    else if (c >= 4) v = __fmul_rn(v, inv_nf);
    if (c < 4) srt[tok * 4 + c] = v;
    else z[tok * (C - 4) + (c - 4)] = v;
}


template <typename T_IN>
__global__ void primvolume_pack_kernel(const float* __restrict__ srt, const T_IN* __restrict__ dec, long long T, int F, int vox, int srt_fix,
                                       float* __restrict__ out) {
    // one thread per 4 consecutive output floats; rows are 4 + F floats, F % 4 == 0 -> every group is 16-B aligned on both sides
    const int groups_per_row = 1 + F / 4;
    const long long gi = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (gi >= T * groups_per_row) return;
    const long long tok = gi / groups_per_row;
    const int g = static_cast<int>(gi - tok * groups_per_row);
    float4 o;
    if (g == 0) {
        o = *reinterpret_cast<const float4*>(srt + tok * 4);
        if (srt_fix) o.x = __fadd_rn(__fmul_rn(o.x, 0.1f), 0.05f);
    } else {
        const int f = (g - 1) * 4;              // feature index = channel * vox + voxel (channel-major, inference.py:347)
        const bool sdf = f < vox;               // channel 0
        float v[4];
        if constexpr (sizeof(T_IN) == 4) {
            const float4 d = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(dec) + tok * F + f);
            v[0] = d.x; v[1] = d.y; v[2] = d.z; v[3] = d.w;
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = sdf ? __fmul_rn(v[k], 0.2f) : __fmul_rn(__fadd_rn(v[k], 1.0f), 0.5f);
        } else {
            const uint2 d = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(dec) + tok * F + f);
            const __half2 a = *reinterpret_cast<const __half2*>(&d.x), b = *reinterpret_cast<const __half2*>(&d.y);
            v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = sdf ? h2f_round(__fmul_rn(v[k], 0.2f)) : h2f_round(__fmul_rn(h2f_round(__fadd_rn(v[k], 1.0f)), 0.5f));
        }
        o = make_float4(v[0], v[1], v[2], v[3]);
    }
    *reinterpret_cast<float4*>(out + tok * (4 + F) + g * 4) = o;
}


}  // namespace tpx

using namespace tpx;

extern "C" {

int tpx_ln_modulate(float* x, int rows, int D, float eps, const void* shift, const void* scale, int mod_bstride, int rows_per_batch, int mod_batches,
                    void* out, const void* pre_gate, const void* pre_const, int pre_row0, void* stream) {
    TPX_CHECK(x != nullptr && shift != nullptr && scale != nullptr && out != nullptr, TPX_ERR_ARG, "ln_modulate: null argument");
    TPX_CHECK(rows_per_batch > 0 && mod_batches > 0, TPX_ERR_ARG, "ln_modulate: bad batching");
    TPX_DEVICE_GUARD();
    return launch_ln_modulate(x, rows, D, eps, static_cast<const __half*>(shift), static_cast<const __half*>(scale), mod_bstride, rows_per_batch,
                              mod_batches, static_cast<__half*>(out), static_cast<const __half*>(pre_gate), static_cast<const __half*>(pre_const),
                              pre_row0, static_cast<cudaStream_t>(stream));
}

int tpx_cfg_combine(const void* both, int64_t n_half, float s, void* out, void* stream) {
    TPX_CHECK(both != nullptr && out != nullptr, TPX_ERR_ARG, "cfg_combine: null argument");
    TPX_DEVICE_GUARD();
    return launch_cfg_combine(static_cast<const __half*>(both), n_half, s, static_cast<__half*>(out), static_cast<cudaStream_t>(stream));
}

int tpx_sampler_step(int ddim, const float* x, const void* mo, int mo_dtype, const float* noise, int64_t n, int C, const tpx_sampler_coefs* k,
                     float* x_prev, float* x0, void* stream) {
    TPX_CHECK(x != nullptr && mo != nullptr && k != nullptr && x_prev != nullptr && x0 != nullptr, TPX_ERR_ARG, "sampler_step: null argument");
    TPX_CHECK(C > 0 && n % C == 0, TPX_ERR_SHAPE, "sampler_step: n %lld not a multiple of C %d", (long long)n, C);
    if (n <= 0) return TPX_OK;
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    ProfScope prof(PROF_ELEMWISE, st);
    if (ddim) {
        if (mo_dtype == TPX_DTYPE_F16) ddim_step_kernel<__half><<<grid, 256, 0, st>>>(x, static_cast<const __half*>(mo), noise, n, C, *k, x_prev, x0);
        else ddim_step_kernel<float><<<grid, 256, 0, st>>>(x, static_cast<const float*>(mo), noise, n, C, *k, x_prev, x0);
    } else {
        if (mo_dtype == TPX_DTYPE_F16) ddpm_step_kernel<__half><<<grid, 256, 0, st>>>(x, static_cast<const __half*>(mo), noise, n, C, *k, x_prev, x0);
        else ddpm_step_kernel<float><<<grid, 256, 0, st>>>(x, static_cast<const float*>(mo), noise, n, C, *k, x_prev, x0);
    }
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_latent_split(const float* sample, const float* mean, const float* stdv, float inv_nf, int64_t T, int C, float* srt, float* z, void* stream) {
    TPX_CHECK(sample != nullptr && srt != nullptr && z != nullptr, TPX_ERR_ARG, "latent_split: null argument");
    TPX_CHECK((mean == nullptr) == (stdv == nullptr), TPX_ERR_ARG, "latent_split: latent_mean and latent_std go together");
    TPX_CHECK(T >= 0 && C > 4, TPX_ERR_SHAPE, "latent_split: need more than 4 channels (got %d)", C);
    const long long n = T * C;
    if (n <= 0) return TPX_OK;
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_ELEMWISE, st);
    latent_split_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(sample, mean, stdv, inv_nf, T, C, srt, z);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

int tpx_primvolume_pack(const float* srt, const void* dec, int dec_dtype, int64_t T, int F, int vox, int srt_fix, float* out, void* stream) {
    TPX_CHECK(srt != nullptr && dec != nullptr && out != nullptr, TPX_ERR_ARG, "primvolume_pack: null argument");
    TPX_CHECK(dec_dtype == TPX_DTYPE_F32 || dec_dtype == TPX_DTYPE_F16, TPX_ERR_ARG, "primvolume_pack: dtype %d", dec_dtype);
    TPX_CHECK(F % 4 == 0 && vox % 4 == 0 && vox <= F, TPX_ERR_SHAPE, "primvolume_pack: feature length %d / voxel count %d must be multiples of 4", F, vox);
    const long long n = T * (1 + F / 4);
    if (n <= 0) return TPX_OK;
    TPX_DEVICE_GUARD();
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ProfScope prof(PROF_ELEMWISE, st);
    const unsigned grid = static_cast<unsigned>((n + 255) / 256);
    if (dec_dtype == TPX_DTYPE_F16) primvolume_pack_kernel<__half><<<grid, 256, 0, st>>>(srt, static_cast<const __half*>(dec), T, F, vox, srt_fix, out);
    else primvolume_pack_kernel<float><<<grid, 256, 0, st>>>(srt, static_cast<const float*>(dec), T, F, vox, srt_fix, out);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // extern "C"
