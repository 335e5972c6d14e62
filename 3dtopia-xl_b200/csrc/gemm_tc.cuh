// Persistent, warp-specialised wgmma GEMM for sm_90a:   C[M,N] = A[M,K] * W[N,K]^T  (+ fused epilogue)
//
//   warp 0          : TMA producer  (cp.async.bulk.tensor -> 128B/64B-swizzled smem ring, mbarrier complete_tx); warps 1-3 of its
//                     warpgroup only give their registers away (setmaxnreg)
//   warpgroups 1, 2 : consumers, in one of two schedules (gemm_pingpong):
//                     ping-pong (linear GEMMs at BN 128 / 144): consumer c owns WHOLE 128 x BN tiles, the CTA's tiles j = c, c + 2, ...
//                     The mainloops take turns through an ordered hand-off (named barriers), so one consumer's epilogue runs while
//                     the other issues wgmma; the producer loads in tile order into the one ring and each consumer steps past the
//                     other's k-blocks.
//                     cooperative (every other width, and the conv GEMMs): both consumers work on every 128 x BN tile, consumer c
//                     on columns [c BN/2, (c+1) BN/2) (tiles narrower than 64 columns run on one consumer).
//                     Either way a consumer holds ALL 128 rows of its columns as two wgmma m64 accumulators in registers.  The two A
//                     descriptors interleave the 8-row groups of the tile (stride 2 groups, starting at group 0 / 1), so warp q
//                     of a consumer ends up with rows 32 q .. 32 q + 31 of the tile: the fused epilogues (bias / GELU / gated
//                     residual / head split / conv scatter; bulk tensor stores) work on 32-row slabs, one row per thread, and
//                     get them through a warp-private shared-memory exchange (acc_rows) with no block-wide synchronisation.
//   The producer runs ahead into the next tile's k-blocks while a consumer is in its epilogue.
//
// A-operand modes: AMODE_LINEAR (2-D tensor map over a row-major [M,K] fp16 matrix) and AMODE_CONV3 (5-D tensor
// map over a channels-last [P,S,S,S,C] fp16 volume: the 27 taps of a 3x3x3 / pad 1 convolution are 27 shifted
// box loads, the halo comes from TMA out-of-bounds zero fill — implicit GEMM with no im2col buffer).
#pragma once
#include "tpx_common.cuh"

namespace tpx {

enum GemmEpiMode : int {
    EPI_STORE = 0,       // out0[row*ldo+col] = h( h(acc+bias) * post_scale )
    EPI_GELU = 1,        // out0 = h( gelu_tanh( h(acc+bias) ) )
    EPI_HEADS = 2,       // split columns into (which, head, d) -> out{which}[b,head,n,DhP]  (zero pad written)
    EPI_GATED = 3,       // xres[row*ldx+col] += float( h( gate[b,col] * h(acc+bias) ) )
    EPI_RESID_SCALE = 4, // out0 = h( (acc + bias + resid[row*ldo+col]) * alpha )
    EPI_NCDHW = 6,       // out[(p*Cout+co)*S3 + vox] = acc + bias   (fp32 or fp16 out, co < n_valid)
    EPI_MOMENTS = 7,     // VAE encoder tail: h = h(acc + bias) on columns 0, 1 (conv_out), then the 1x1 quant_conv 2 -> 2 on h:
                         // out[(p*2+c)*S3 + vox] = h(quant[2c] h0 + quant[2c+1] h1 + quant[4+c])   (fp32 or fp16 out)
};
enum GemmAMode : int { AMODE_LINEAR = 0, AMODE_CONV3 = 1 };

struct GemmArgs {
    int M, N, num_kb;
    int tiles_n, num_tiles;   // 128 x BN tiles: per row of tiles, in all (kernel parameters, so they cost the consumers no registers)
    int conv_S, chunks_per_tap;
    const __half* bias;
    float post_scale;
    __half* out0;
    __half* out1;
    __half* out2;
    int ldo;
    int split_cols, Dh, DhP, H, Nseq;
    int vt_which_plus1, vt_ld;   // EPI_HEADS: column group (which+1) stored TRANSPOSED as [b,head,DhP,vt_ld] (keys contiguous); 0 = none
    float* xres;
    int ldx;
    const __half* gate;
    int gate_bstride, rows_per_batch, gate_batches;
    const __half* resid;
    float alpha;
    float* out32;
    int n_valid, S3;
    int convt_store;  // EPI_STORE: 1 = rows are (primitive, 4^3 voxel) and the output map is the 5-D stride-2 lattice of one (a,b,c) offset of
                      // a ConvTranspose3d(k2,s2): a warp's 32 rows are one [2 z][4 y][4 x] box (vae3d_dib.py:220-226)
    int heads_tma;    // EPI_HEADS: 1 = outputs leave as 24-column bulk tensor stores (launcher checked the geometry, padding is pre-zeroed)
    const __half* quant;   // EPI_MOMENTS: quant_conv as [w00, w01, w10, w11, b0, b1] (vae3d_dib.py:428)
};

constexpr bool gemm_pingpong(int bn, int amode) { return amode == AMODE_LINEAR && (bn == 128 || bn == 144); }
constexpr int gemm_wn(int bn, int amode) { return gemm_pingpong(bn, amode) ? bn : (bn >= 64 ? bn / 2 : bn); }   // columns of one consumer warpgroup
constexpr int GEMM_MAX_WN = 144;

template <int BN, int BK, int AMODE>
struct GemmCfg {
    static constexpr int BM = 128;
    static constexpr int SW = BK * 2;
    static constexpr bool PP = gemm_pingpong(BN, AMODE);
    static constexpr int NWG = BN >= 64 ? 2 : 1;                 // consumer warpgroups
    static constexpr int WN = gemm_wn(BN, AMODE);
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    // per consumer warp: one 32-row x 128-B staging buffer for the bulk stores (1024-B aligned: 128-B swizzle) and one exchange buffer
    static constexpr int STAGING_BYTES = BN >= 64 ? 8 * 4096 : 0;
    static constexpr int XCHG_BYTES = NWG * 4 * XCHG_FLOATS * 4;
    static constexpr int TAIL_BYTES = 256 /*barriers*/ + 4 * GEMM_MAX_WN * 4 /*bias + gate columns of both consumers, fp32*/;
    // dynamic shared memory is declared __align__(1024) (the kernel traps if the base is not), so no alignment slack is budgeted
    static constexpr int STAGES_RAW = (227 * 1024 - STAGING_BYTES - XCHG_BYTES - TAIL_BYTES) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 8 ? 8 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + STAGING_BYTES + XCHG_BYTES + TAIL_BYTES;
    static constexpr int THREADS = 384;
    static_assert(STAGES >= 2 && SMEM_BYTES <= 227 * 1024, "shared memory budget");
    static_assert(B_BYTES % 1024 == 0 && A_BYTES % 1024 == 0, "stage operands must stay 1024-B aligned");
    static_assert(WN % 8 == 0 && WN <= GEMM_MAX_WN && (WN * SW) % 1024 == 0, "consumer tile: wgmma N, accumulator registers, swizzle alignment");
};

union Pack8 {
    uint4 u;
    __half2 h2[4];
    __half h[8];
};

// ---- epilogue ---------------------------------------------------------------------------------------------------
// One thread owns one accumulator row; columns arrive in chunks of CH (32) fp32 values from the accumulator exchange.  bias (and the
// adaLN gate when it is uniform over the tile's rows) are staged once per tile in shared memory as fp32, every
// global load of a chunk is issued before the first use, and the (which, head, d) split of a column is advanced
// incrementally instead of divided out per group.
struct HeadCursor {
    int which, head, d;
    int b, n;   // batch / token of this thread's row
};

// h(a), h(b) as floats through ONE packed conversion (F2FP.F16.F32.PACK_AB, ALU pipe); the scalar cvt.rn.f16.f32 is an XU-pipe
// instruction (16 / clk / SM, shared with MUFU) and was the bound of the GELU / gated epilogues.
__device__ __forceinline__ float2 round_h2(float a, float b) { return __half22float2(__floats2half2_rn(a, b)); }
// gelu_tanh(x) = 0.5 x (1 + tanh(u)) = x * sigmoid(2u),  u = sqrt(2/pi) (x + 0.044715 x^3):  x / (1 + 2^(-2 u log2 e)).
// Five FMA-pipe operations + MUFU.EX2 + MUFU.RCP; saturates cleanly (2^+inf -> rcp(inf) = 0, 2^-inf -> 1).
__device__ __forceinline__ float gelu_tanh_sigmoid(float x) {
    const float k0 = -2.0f * 0.7978845608028654f * 1.4426950408889634f, k1 = k0 * 0.044715f;
    const float t = x * x;
    const float arg = x * fmaf(k1, t, k0);
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(arg));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return x * r;
}

template <int EPI, int CH>
__device__ __forceinline__ void epi_chunk(const GemmArgs& g, const float* __restrict__ sb, const float* __restrict__ sg, bool gate_in_smem, int row,
                                          bool row_ok, int col0, int c0, const uint32_t* acc, HeadCursor& hc, size_t head_row_off) {
    constexpr int NG = CH / 8;
    float v[CH];
#pragma unroll
    for (int i = 0; i < CH; i += 4) {
        const float4 b4 = *reinterpret_cast<const float4*>(sb + c0 + i);
        v[i] = __uint_as_float(acc[i]) + b4.x;
        v[i + 1] = __uint_as_float(acc[i + 1]) + b4.y;
        v[i + 2] = __uint_as_float(acc[i + 2]) + b4.z;
        v[i + 3] = __uint_as_float(acc[i + 3]) + b4.w;
    }
    bool ok[NG];
#pragma unroll
    for (int j = 0; j < NG; ++j) ok[j] = row_ok && (col0 + j * 8 < g.N);

    if constexpr (EPI == EPI_STORE || EPI == EPI_GELU) {
        __half* op = g.out0 + static_cast<size_t>(row) * g.ldo + col0;
#pragma unroll
        for (int j = 0; j < NG; ++j) {
            Pack8 o;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float x = h2f_round(v[j * 8 + i]);
                if constexpr (EPI == EPI_GELU) x = gelu_tanh_sigmoid(x);   // the same evaluation as the bulk-store path: one result per input whatever the tile
                else if (g.post_scale != 1.0f) x = x * g.post_scale;
                o.h[i] = __float2half_rn(x);
            }
            if (ok[j]) *reinterpret_cast<uint4*>(op + j * 8) = o.u;
        }
    } else if constexpr (EPI == EPI_HEADS) {
#pragma unroll
        for (int j = 0; j < NG; ++j) {
            __half* base = hc.which == 0 ? g.out0 : (hc.which == 1 ? g.out1 : g.out2);
            const bool sc = g.post_scale != 1.0f && hc.which == 0;
            Pack8 o;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float x = h2f_round(v[j * 8 + i]);
                if (sc) x = x * g.post_scale;
                o.h[i] = __float2half_rn(x);
            }
            if (hc.which + 1 == g.vt_which_plus1) {
                // transposed store for the attention kernel's PV operand: [b, head, d, token] (tokens contiguous)
                __half* dst = base + (static_cast<size_t>(hc.b * g.H + hc.head) * g.DhP + hc.d) * g.vt_ld + hc.n;
                if (ok[j]) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) dst[static_cast<size_t>(i) * g.vt_ld] = o.h[i];
                    if (hc.d + 8 == g.Dh)
                        for (int p = g.Dh; p < g.DhP; ++p) dst[static_cast<size_t>(p - hc.d) * g.vt_ld] = __float2half_rn(0.f);
                }
            } else {
                __half* dst = base + head_row_off + static_cast<size_t>(hc.head) * g.Nseq * g.DhP + hc.d;
                if (ok[j]) {
                    *reinterpret_cast<uint4*>(dst) = o.u;
                    if (hc.d + 8 == g.Dh)   // last real group of this head: write the zero padding d in [Dh, DhP)
                        for (int p = g.Dh; p < g.DhP; p += 8) *reinterpret_cast<uint4*>(dst + (p - hc.d)) = make_uint4(0, 0, 0, 0);
                }
            }
            hc.d += 8;
            if (hc.d >= g.Dh) {
                hc.d = 0;
                if (++hc.head == g.H) { hc.head = 0; ++hc.which; }
            }
        }
    } else if constexpr (EPI == EPI_GATED) {
        float* xp = g.xres + static_cast<size_t>(row) * g.ldx + col0;
        float4 xr[2 * NG];
#pragma unroll
        for (int j = 0; j < NG; ++j) {
            xr[2 * j] = ok[j] ? *reinterpret_cast<const float4*>(xp + j * 8) : make_float4(0.f, 0.f, 0.f, 0.f);
            xr[2 * j + 1] = ok[j] ? *reinterpret_cast<const float4*>(xp + j * 8 + 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        float gt[CH];
        if (gate_in_smem) {
#pragma unroll
            for (int i = 0; i < CH; i += 4) {
                const float4 g4 = *reinterpret_cast<const float4*>(sg + c0 + i);
                gt[i] = g4.x; gt[i + 1] = g4.y; gt[i + 2] = g4.z; gt[i + 3] = g4.w;
            }
        } else {
            const int b = (row / g.rows_per_batch) % g.gate_batches;
            const __half* gp = g.gate + static_cast<size_t>(b) * g.gate_bstride + col0;
#pragma unroll
            for (int j = 0; j < NG; ++j) {
                Pack8 t;
                t.u = ok[j] ? *reinterpret_cast<const uint4*>(gp + j * 8) : make_uint4(0, 0, 0, 0);
#pragma unroll
                for (int i = 0; i < 8; ++i) gt[j * 8 + i] = __half2float(t.h[i]);
            }
        }
#pragma unroll
        for (int j = 0; j < NG; ++j) {
            float4 a = xr[2 * j], c = xr[2 * j + 1];
            a.x += h2f_round(gt[j * 8 + 0] * h2f_round(v[j * 8 + 0]));
            a.y += h2f_round(gt[j * 8 + 1] * h2f_round(v[j * 8 + 1]));
            a.z += h2f_round(gt[j * 8 + 2] * h2f_round(v[j * 8 + 2]));
            a.w += h2f_round(gt[j * 8 + 3] * h2f_round(v[j * 8 + 3]));
            c.x += h2f_round(gt[j * 8 + 4] * h2f_round(v[j * 8 + 4]));
            c.y += h2f_round(gt[j * 8 + 5] * h2f_round(v[j * 8 + 5]));
            c.z += h2f_round(gt[j * 8 + 6] * h2f_round(v[j * 8 + 6]));
            c.w += h2f_round(gt[j * 8 + 7] * h2f_round(v[j * 8 + 7]));
            if (ok[j]) {
                *reinterpret_cast<float4*>(xp + j * 8) = a;
                *reinterpret_cast<float4*>(xp + j * 8 + 4) = c;
            }
        }
    } else if constexpr (EPI == EPI_RESID_SCALE) {
        const size_t off = static_cast<size_t>(row) * g.ldo + col0;
        Pack8 rs[NG];
#pragma unroll
        for (int j = 0; j < NG; ++j) rs[j].u = (ok[j] && g.resid != nullptr) ? *reinterpret_cast<const uint4*>(g.resid + off + j * 8) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int j = 0; j < NG; ++j) {
            Pack8 o;
#pragma unroll
            for (int i = 0; i < 8; ++i) o.h[i] = __float2half_rn((v[j * 8 + i] + __half2float(rs[j].h[i])) * g.alpha);
            if (ok[j]) *reinterpret_cast<uint4*>(g.out0 + off + j * 8) = o.u;
        }
    } else if constexpr (EPI == EPI_NCDHW) {
        const int p = row / g.S3, vox = row - p * g.S3;
#pragma unroll
        for (int i = 0; i < CH; ++i) {
            const int co = col0 + i;
            if (row_ok && co < g.n_valid) {
                const size_t off = (static_cast<size_t>(p) * g.n_valid + co) * g.S3 + vox;
                if (g.out32 != nullptr) g.out32[off] = v[i];
                else g.out0[off] = __float2half_rn(v[i]);
            }
        }
    } else if constexpr (EPI == EPI_MOMENTS) {
        // conv_out's two channels at their fp16 rounding point (autocast), then quant_conv on those rounded values (not folded into
        // conv_out's weights: the reference rounds in between); channel 0 = mean, 1 = logvar (vae3d_dib.py:52-53)
        if (row_ok && col0 == 0) {
            const int p = row / g.S3, vox = row - p * g.S3;
            const float h0 = h2f_round(v[0]), h1 = h2f_round(v[1]);
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const float m = h2f_round(fmaf(__half2float(g.quant[2 * c + 1]), h1, fmaf(__half2float(g.quant[2 * c]), h0, __half2float(g.quant[4 + c]))));
                const size_t off = (static_cast<size_t>(p) * 2 + c) * g.S3 + vox;
                if (g.out32 != nullptr) g.out32[off] = m;
                else g.out0[off] = __float2half_rn(m);
            }
        }
    }
}


// ---- epilogue through shared memory + TMA (EPI_STORE / EPI_GELU / EPI_GATED) ------------------------------------------------------
// Each consumer warp owns 32 accumulator rows and walks its warpgroup's columns in 32-column chunks.  Results go to a 32-row x
// 128-B staging buffer in the 128-B-swizzled layout (conflict-free 16-B stores) and leave as ONE bulk tensor store per 128-B row
// group:
//   fp16 outputs: 64 columns per store (cp.async.bulk.tensor, full 128-B lines instead of 16-B pieces per thread);
//   gated residual: 32 fp32 columns per cp.reduce.async.bulk.tensor .add — the L2 performs  x += h(gate * h(acc + b)),  so the
//   epilogue never loads the residual (one add per element per launch: deterministic; the L2 adder flushes subnormals).  A width
//   of 32 k + 16 (144) ends with one 16-column reduce through its own 64-B-swizzled map.
// Rows >= M and columns >= N are clipped by the tensor map.  wn = columns of one consumer warpgroup.
constexpr bool gemm_tma_epilogue(int epi, int wn) {
    return ((epi == EPI_STORE || epi == EPI_GELU) && wn % 64 == 0) || (epi == EPI_GATED && wn % 16 == 0 && wn >= 64);
}

__device__ __forceinline__ void staging_acquire(int lane) {
    if (lane == 0) bulk_wait_read<0>();             // the bulk operation that last read the staging buffer is done
    __syncwarp();
}

// One CW-column (32 or 16) chunk of the gated residual: staged as 32 rows x CW fp32 in the tensor map's swizzle (128 B / 64 B rows:
// conflict-free 16-B stores), then one bulk reduce-add.
template <int CW, int NA>
__device__ __forceinline__ void epilogue_gated_chunk(const GemmArgs& g, const CUtensorMap* tm, const float* __restrict__ sb, const float* __restrict__ sg,
                                                     bool gate_in_smem, const float (&accv)[2][NA], float* xb, uint32_t stg, int row0, int n0, int c0,
                                                     int lane) {
    static_assert(CW == 32 || CW == 16, "gated chunk width");
    const uint32_t dst = stg + lane * (CW * 4);
    const int sw = ((lane * CW * 4) >> 7) & (CW / 4 - 1);     // the 16-B unit index bits the 128-B / 64-B swizzle XORs in
    uint32_t acc[CW];
    acc_rows<CW, 8, 16>(accv[0], accv[1], c0, xb, lane, acc);
    staging_acquire(lane);
    // a per-row gate stays packed fp16 until use (8 registers per 32 columns, not 32: the 144-wide accumulator leaves little room)
    Pack8 gh[CW / 8];
    if (!gate_in_smem) {
        const int b = ((row0 + lane) / g.rows_per_batch) % g.gate_batches;
        const __half* gp = g.gate + static_cast<size_t>(b) * g.gate_bstride + n0 + c0;
#pragma unroll
        for (int j = 0; j < CW / 8; ++j) gh[j].u = (n0 + c0 + j * 8 < g.N) ? *reinterpret_cast<const uint4*>(gp + j * 8) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int j = 0; j < CW / 4; ++j) {
        float4 g4;
        if (gate_in_smem) {
            g4 = *reinterpret_cast<const float4*>(sg + c0 + j * 4);
        } else {
            const float2 lo = __half22float2(gh[j >> 1].h2[(j & 1) * 2]), hi = __half22float2(gh[j >> 1].h2[(j & 1) * 2 + 1]);
            g4 = make_float4(lo.x, lo.y, hi.x, hi.y);
        }
        const float4 b4 = *reinterpret_cast<const float4*>(sb + c0 + j * 4);
        const float2 v01 = round_h2(__uint_as_float(acc[j * 4 + 0]) + b4.x, __uint_as_float(acc[j * 4 + 1]) + b4.y);
        const float2 v23 = round_h2(__uint_as_float(acc[j * 4 + 2]) + b4.z, __uint_as_float(acc[j * 4 + 3]) + b4.w);
        const float2 o01 = round_h2(g4.x * v01.x, g4.y * v01.y);
        const float2 o23 = round_h2(g4.z * v23.x, g4.w * v23.y);
        const float o[4] = {o01.x, o01.y, o23.x, o23.y};
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + ((j ^ sw) << 4)), "f"(o[0]), "f"(o[1]), "f"(o[2]), "f"(o[3]) : "memory");
    }
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
        tma_reduce_add_2d(tm, stg, n0 + c0, row0);
        bulk_commit();
    }
}

// tmC: the fp16 output map, or the 32-column residual map; tmD: the 16-column residual map (gated widths 32 k + 16)
template <int EPI, int WN, int NA>
__device__ __forceinline__ void epilogue_tma(const GemmArgs& g, const CUtensorMap* tmC, const CUtensorMap* tmD, const float* __restrict__ sb,
                                             const float* __restrict__ sg, bool gate_in_smem, const float (&accv)[2][NA], float* xb, uint32_t stg,
                                             int row0, int n0, int lane) {
    if constexpr (EPI == EPI_GATED) {
#pragma unroll
        for (int k = 0; k < WN / 32; ++k) epilogue_gated_chunk<32>(g, tmC, sb, sg, gate_in_smem, accv, xb, stg, row0, n0, k * 32, lane);
        if constexpr (WN % 32 != 0) epilogue_gated_chunk<16>(g, tmD, sb, sg, gate_in_smem, accv, xb, stg, row0, n0, WN - 16, lane);
    } else {
        const uint32_t dst = stg + lane * 128;
        const int sw = lane & 7;
#pragma unroll
        for (int k = 0; k < WN / 32; ++k) {
            uint32_t acc[32];
            acc_rows<32, 8, 16>(accv[0], accv[1], k * 32, xb, lane, acc);
            const int c0 = k * 32;
            if ((k & 1) == 0) staging_acquire(lane);
            uint32_t pk[16];
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
                const float4 b4 = *reinterpret_cast<const float4*>(sb + c0 + i);
                float x[4] = {__uint_as_float(acc[i]) + b4.x, __uint_as_float(acc[i + 1]) + b4.y, __uint_as_float(acc[i + 2]) + b4.z,
                              __uint_as_float(acc[i + 3]) + b4.w};
                if (EPI == EPI_GELU || g.post_scale != 1.0f) {     // otherwise the pack below is the one rounding
                    const float2 r01 = round_h2(x[0], x[1]), r23 = round_h2(x[2], x[3]);
                    x[0] = r01.x; x[1] = r01.y; x[2] = r23.x; x[3] = r23.y;
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        if constexpr (EPI == EPI_GELU) x[e] = gelu_tanh_sigmoid(x[e]);
                        else x[e] *= g.post_scale;
                    }
                }
                const __half2 h0 = __floats2half2_rn(x[0], x[1]), h1 = __floats2half2_rn(x[2], x[3]);
                pk[i >> 1] = *reinterpret_cast<const uint32_t*>(&h0);
                pk[(i >> 1) + 1] = *reinterpret_cast<const uint32_t*>(&h1);
            }
#pragma unroll
            for (int q = 0; q < 4; ++q)
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst + ((((k & 1) * 4 + q) ^ sw) << 4)), "r"(pk[4 * q]), "r"(pk[4 * q + 1]),
                             "r"(pk[4 * q + 2]), "r"(pk[4 * q + 3])
                             : "memory");
            if ((k & 1) == 1) {
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) {
                    if (g.convt_store != 0) tma_store_5d(tmC, stg, n0 + (k - 1) * 32, 0, 0, (row0 & 63) >> 4, row0 >> 6);
                    else tma_store_2d(tmC, stg, n0 + (k - 1) * 32, row0);
                    bulk_commit();
                }
            }
        }
    }
}

// ---- EPI_HEADS through shared memory + TMA ---------------------------------------------------------------------------------------
// Column groups of 24 (= Dh / 3 for Dh = 72; every consumer tile, head and q/k/v boundary is a multiple of 24): a warp's 32 rows x
// 24 columns are one box of the destination [B*H*Nseq, DhP] matrix (rows (b, head, n0 .. n0+31), columns d0 .. d0+23), or — for the
// transposed V the attention kernel reads — one 24-row x 32-token box of [B*H*DhP, vt_ld].  Needs Nseq % 32 == 0 (a 32-row slab
// never straddles a sequence), Dh % 24 == 0, and the head-dim padding columns d >= Dh already zero (the launcher's caller memsets).
constexpr int HG = 24;
template <int NG, int NA>
__device__ __forceinline__ void epilogue_heads_tma(const GemmArgs& g, const CUtensorMap* tmQ, const CUtensorMap* tmK, const CUtensorMap* tmV,
                                                   const float* __restrict__ sb, const float (&accv)[2][NA], float* xb, uint32_t stg, int row0, int n0,
                                                   int lane) {
    if (row0 >= g.M) return;                        // whole slab outside the matrix (M is a multiple of 32 here)
    const int b = row0 / g.Nseq, nfirst = row0 - b * g.Nseq;
#pragma unroll
    for (int k = 0; k < NG; ++k) {
        uint32_t acc[24];
        acc_rows<HG, 8, 16>(accv[0], accv[1], k * HG, xb, lane, acc);
        const int c0 = k * HG;
        const int col = n0 + c0;
        const int which = col / g.split_cols;
        const int cw = col - which * g.split_cols;
        const int head = cw / g.Dh;
        const int d0 = cw - head * g.Dh;
        const bool sc = g.post_scale != 1.0f && which == 0;
        uint32_t pk[12];
#pragma unroll
        for (int i = 0; i < HG; i += 4) {
            const float4 b4 = *reinterpret_cast<const float4*>(sb + c0 + i);
            float x[4] = {__uint_as_float(acc[i]) + b4.x, __uint_as_float(acc[i + 1]) + b4.y, __uint_as_float(acc[i + 2]) + b4.z,
                          __uint_as_float(acc[i + 3]) + b4.w};
            if (sc) {
                const float2 r01 = round_h2(x[0], x[1]), r23 = round_h2(x[2], x[3]);
                x[0] = r01.x * g.post_scale; x[1] = r01.y * g.post_scale; x[2] = r23.x * g.post_scale; x[3] = r23.y * g.post_scale;
            }
            const __half2 h0 = __floats2half2_rn(x[0], x[1]), h1 = __floats2half2_rn(x[2], x[3]);
            pk[i >> 1] = *reinterpret_cast<const uint32_t*>(&h0);
            pk[(i >> 1) + 1] = *reinterpret_cast<const uint32_t*>(&h1);
        }
        staging_acquire(lane);
        const bool transposed = which + 1 == g.vt_which_plus1;
        if (transposed) {
            // staging [24 d][32 tokens] fp16: lane = token
#pragma unroll
            for (int i = 0; i < 12; ++i) {
                const uint16_t lo = static_cast<uint16_t>(pk[i] & 0xFFFFu), hi = static_cast<uint16_t>(pk[i] >> 16);
                asm volatile("st.shared.b16 [%0], %1;" ::"r"(stg + (2 * i) * 64 + lane * 2), "h"(lo) : "memory");
                asm volatile("st.shared.b16 [%0], %1;" ::"r"(stg + (2 * i + 1) * 64 + lane * 2), "h"(hi) : "memory");
            }
        } else {
            // staging [32 rows][24 columns] fp16 (48-B rows: conflict-free 16-B stores)
#pragma unroll
            for (int q = 0; q < 3; ++q)
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(stg + lane * 48 + q * 16), "r"(pk[4 * q]), "r"(pk[4 * q + 1]), "r"(pk[4 * q + 2]),
                             "r"(pk[4 * q + 3])
                             : "memory");
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
            if (transposed) tma_store_2d(tmV, stg, nfirst, (b * g.H + head) * g.DhP + d0);
            else tma_store_2d(which == 0 ? tmQ : (which == 1 ? tmK : tmV), stg, d0, (b * g.H + head) * g.Nseq + nfirst);
            bulk_commit();
        }
    }
}

// named barrier of one consumer warpgroup (ids 1, 2; id 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int cw) { asm volatile("bar.sync %0, 128;" ::"r"(cw + 1) : "memory"); }

template <int BN, int BK, int AMODE, int EPI>
__global__ void __launch_bounds__(384, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
               const __grid_constant__ CUtensorMap tmD, const __grid_constant__ CUtensorMap tmE, const GemmArgs g) {
    using Cfg = GemmCfg<BN, BK, AMODE>;
    constexpr int STAGES = Cfg::STAGES, WN = Cfg::WN, NWG = Cfg::NWG, SW = Cfg::SW;
    constexpr bool kPP = Cfg::PP;
    constexpr bool kTmaEpi = gemm_tma_epilogue(EPI, WN);
    constexpr bool kHeadsTma = EPI == EPI_HEADS && WN % HG == 0 && Cfg::STAGING_BYTES > 0;   // taken when g.heads_tma is set
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;
    if ((smem_u32(smem_raw) & 1023u) != 0) __trap();   // the swizzled operand / staging tiles need a 1024-B aligned base
    // layout: [operand ring][epilogue staging][accumulator exchange][barriers 256 B][bias + gate columns, 2 x 2 x GEMM_MAX_WN fp32]
    constexpr int OFF_STG = STAGES * Cfg::STAGE_BYTES;
    constexpr int OFF_XCHG = OFF_STG + Cfg::STAGING_BYTES;
    constexpr int OFF_BAR = OFF_XCHG + Cfg::XCHG_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if constexpr (kTmaEpi) tma_prefetch_desc(&tmC);
        if constexpr (kTmaEpi && EPI == EPI_GATED && WN % 32 != 0) tma_prefetch_desc(&tmD);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kPP ? 4 : NWG * 4);   // one lane of every warp of the consumer(s) reading the stage
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    pdl_launch_dependents();   // the next kernel of the stream may start its own prologue
    pdl_wait();                // ... and ours ends here: the operands written by the previous kernel are now visible

    const int tiles_n = g.tiles_n;
    const int num_tiles = g.num_tiles;
    const int num_kb = g.num_kb;

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0) {
            // warp-converged producer: every lane follows the ring, one elected lane arms the barrier and issues the TMA
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int m_blk = tile / tiles_n, n_blk = tile - m_blk * tiles_n;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    if (elect_one()) {
                        uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                        mbar_arrive_expect_tx(&full_bar[stage], Cfg::STAGE_BYTES);
                        if constexpr (AMODE == AMODE_LINEAR) {
                            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m_blk * 128);
                        } else {
                            const int tap = kb / g.chunks_per_tap, chunk = kb - tap * g.chunks_per_tap;
                            const int dz = tap / 9, dy = (tap / 3) % 3, dx = tap % 3;
                            if (g.conv_S == 4) {  // 128 rows = 2 primitives x 4^3 voxels
                                tma_load_5d(sa, &tmA, &full_bar[stage], chunk * BK, dx - 1, dy - 1, dz - 1, m_blk * 2);
                            } else {              // S == 8: 128 rows = 2 z-slices of one primitive
                                tma_load_5d(sa, &tmA, &full_bar[stage], chunk * BK, dx - 1, dy - 1, (m_blk & 3) * 2 + dz - 1, m_blk >> 2);
                            }
                        }
                        tma_load_2d(sa + Cfg::A_BYTES, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
                    }
                    __syncwarp();
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = (warp >> 2) - 1;          // consumer warpgroup
        if (cw < NWG) {
            const int quad = warp & 3;           // rows 32 quad .. 32 quad + 31 of the tile
            const int et = threadIdx.x - 128 * (cw + 1);
            float* s_bias = reinterpret_cast<float*>(smem + OFF_BAR + 256) + cw * GEMM_MAX_WN;
            float* s_gate = s_bias + 2 * GEMM_MAX_WN;
            float* xb = reinterpret_cast<float*>(smem + OFF_XCHG) + (cw * 4 + quad) * XCHG_FLOATS;
            const uint32_t stg = smem_u32(smem) + OFF_STG + (cw * 4 + quad) * 4096;
            const uint32_t smem_u = smem_u32(smem);
            const bool gate_in_smem = (EPI == EPI_GATED) && (g.rows_per_batch % 128 == 0);
            float acc[2][WN / 2];
            // the CTA's tiles are j = 0, 1, ... (tile blockIdx.x + j gridDim.x); ping-pong: this consumer takes every other one
            for (int j = kPP ? cw : 0;; j += kPP ? 2 : 1) {
                const int tile = blockIdx.x + j * gridDim.x;
                if (tile >= num_tiles) break;
                const int m_blk = tile / tiles_n, n_blk = tile - m_blk * tiles_n;
                const int n0 = n_blk * BN + (kPP ? 0 : cw * WN);
                // the producer fills the ring in tile order: tile j's k-blocks are ring slots j num_kb, j num_kb + 1, ...
                const uint32_t slot0 = static_cast<uint32_t>(j) * static_cast<uint32_t>(num_kb);
                int stage = static_cast<int>(slot0 % STAGES);
                uint32_t phase = (slot0 / STAGES) & 1u;
                // stage this warpgroup's bias (and gate) columns; they are read after the main loop
                wg_bar_sync(cw);
                for (int c = et; c < WN; c += 128) {
                    const int col = n0 + c;
                    s_bias[c] = (g.bias != nullptr && col < g.N) ? __half2float(g.bias[col]) : 0.f;
                    if constexpr (EPI == EPI_GATED) {
                        if (gate_in_smem) {
                            const int b = ((m_blk * 128) / g.rows_per_batch) % g.gate_batches;
                            s_gate[c] = col < g.N ? __half2float(g.gate[static_cast<size_t>(b) * g.gate_bstride + col]) : 0.f;
                        }
                    }
                }
                if constexpr (kPP) {
                    if (j > 0) pp_turn_wait(cw);   // tile j - 1 (the other consumer's) has all its wgmma issued
                }
                int prev = -1;
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&full_bar[stage], phase);
                    const uint32_t a_addr = smem_u + stage * Cfg::STAGE_BYTES;
                    const uint64_t da0 = wgmma_desc_kmajor<SW>(a_addr, 2 * SW * 8), da1 = wgmma_desc_kmajor<SW>(a_addr + SW * 8, 2 * SW * 8);
                    const uint64_t db = wgmma_desc_kmajor<SW>(a_addr + Cfg::A_BYTES + (kPP ? 0 : cw * WN * SW));
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        wgmma_ss_n<WN>(acc[0], da0 + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u, SW);
                        wgmma_ss_n<WN>(acc[1], da1 + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u, SW);
                    }
                    wgmma_commit();
                    if (prev >= 0) {             // the previous k-block's products have retired: its smem slot is free
                        wgmma_wait<1>();
                        if (lane == 0) mbar_arrive(&empty_bar[prev]);
                    }
                    prev = stage;
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
                if constexpr (kPP) {
                    if (tile + static_cast<int>(gridDim.x) < num_tiles) pp_turn_pass(cw);   // the other consumer's tile j + 1 may start
                }
                wgmma_wait<0>();
                if (lane == 0) mbar_arrive(&empty_bar[prev]);
                acc_fence<WN / 2>(acc[0]);
                acc_fence<WN / 2>(acc[1]);
                wg_bar_sync(cw);

                const int row0 = m_blk * 128 + quad * 32;
                bool done = false;
                if constexpr (kHeadsTma) {
                    if (g.heads_tma != 0) {
                        epilogue_heads_tma<WN / HG>(g, &tmC, &tmD, &tmE, s_bias, acc, xb, stg, row0, n0, lane);
                        done = true;
                    }
                }
                if constexpr (kTmaEpi) {
                    epilogue_tma<EPI, WN>(g, &tmC, &tmD, s_bias, s_gate, gate_in_smem, acc, xb, stg, row0, n0, lane);
                } else if (!done) {
                    constexpr int CH = WN % 32 == 0 ? 32 : 16;
                    if constexpr (WN % CH == 0) {
                        const int row = row0 + lane;
                        const bool row_ok = row < g.M;
                        HeadCursor hc{0, 0, 0, 0, 0};
                        size_t head_row_off = 0;
                        if constexpr (EPI == EPI_HEADS) {
                            hc.which = n0 / g.split_cols;
                            const int c = n0 - hc.which * g.split_cols;
                            hc.head = c / g.Dh;
                            hc.d = c - hc.head * g.Dh;
                            hc.b = row / g.Nseq;
                            hc.n = row - hc.b * g.Nseq;
                            head_row_off = (static_cast<size_t>(hc.b) * g.H * g.Nseq + hc.n) * g.DhP;
                        }
#pragma unroll
                        for (int c0 = 0; c0 < WN; c0 += CH) {
                            uint32_t r[CH];
                            acc_rows<CH, 8, 16>(acc[0], acc[1], c0, xb, lane, r);
                            epi_chunk<EPI, CH>(g, s_bias, s_gate, gate_in_smem, row, row_ok, n0 + c0, c0, r, hc, head_row_off);
                        }
                    }
                }
            }
            if constexpr (kTmaEpi || kHeadsTma) {
                if (lane == 0) bulk_wait<0>();          // every bulk store / reduce of this warp has been performed
            }
        }
    }
}

// ---- host side ----------------------------------------------------------------------------------------
struct GemmProblem {
    // A operand
    const __half* A;
    int a_mode;         // AMODE_*
    int lda;            // linear: row stride in elements
    int conv_S, conv_C; // conv: spatial size (4|8) and channel count of the channels-last volume; P = M / S^3
    // W operand [N, K] row-major fp16 (K-major)
    const __half* W;
    int M, N, K;
    int BN;             // tile N (128/144/192/256/32/16; linear 128 / 144 run the ping-pong schedule); BK chosen from K (64, or 32 when conv_C == 32)
    int epi;
    GemmArgs args;      // epilogue fields (M, N, num_kb and the tile counts filled by the launcher)
};
int launch_gemm(const GemmProblem& p, cudaStream_t stream);
int gemm_pick_bn(const GemmProblem& p);
// linear GEMM out = A[M,K] W[N,K]^T through `epi`; tile_n: 0 = automatic (gemm_pick_bn), > 0 = that tile width
int gemm_linear(const __half* A, int lda, const __half* W, int M, int N, int K, int epi, const GemmArgs& args, int tile_n, cudaStream_t st);

}  // namespace tpx
