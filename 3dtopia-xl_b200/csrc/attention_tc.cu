// wgmma flash attention for head_dim 72 or 64 (padded to 80):  out = softmax(q k^T * scale) v
//   (contract of xformers.ops.memory_efficient_attention as called at models/attention.py:54,109)
//
// One CTA = 128 query rows of one (batch, head); K / V^T stream through a TMA ring in 128-key tiles.
//   warp 0           TMA producer (Q once, then K and V^T tiles, each with its own full / empty mbarriers, so K_{j+4} may land
//                    while V_j is still read); warps 1-3 of its warpgroup only give their registers away (setmaxnreg)
//   warpgroups 1, 2  consumers, 64 query rows each:  S = Q K^T  (wgmma m64n128k16 x 5, both operands from shared memory, fp32 in
//                    registers), online softmax on the accumulator fragment (a row lives in the four threads of a quad: row max
//                    by two shuffles, row sum kept as per-thread partials until the end), P converted in registers to the fp16 A
//                    fragments of  O += P V  (wgmma m64n72k16 x 8, A from registers, B = the V^T tile), O in registers.
// Overlap of the exponentials with tensor-core work, two ways:
//   ping-pong        the consumers take turns issuing their wgmma (named-barrier hand-off), so one's softmax runs under the other's
//                    products;
//   pipelining       within a consumer, S_{j+1} and PV_j are issued in one turn and S_{j+1}'s softmax runs while PV_j is in flight.
// The arithmetic is that of a serial loop (same tiles, exponent arguments, partial sums, fp16 P, rescale order): the output does
// not depend on the schedule.
//
// Layouts: q, k  [B,H,N,80] fp16 (d >= Dh zero: S = Q K^T runs over all 80);  vT [B,H,80,NkPad] fp16 (V transposed: keys contiguous,
// NkPad % 8 == 0, rows d >= Dh and key columns >= Nk finite);  out [B,Nq,H*Dh] fp16.
#include "kernels.cuh"

namespace tpx {

namespace {

constexpr int TA_DHP = 80;
constexpr int TA_DO = 72;                               // O columns computed (the stored head dims: 72, or 64 of them)
constexpr int TA_BQ = 128, TA_BKV = 128;
constexpr int TA_Q_BYTES = 128 * 128 + 128 * 32;        // 64-wide SW128 part + 16-wide SW32 part
constexpr int TA_K_BYTES = TA_Q_BYTES;
constexpr int TA_VBOX_BYTES = TA_DHP * 128;             // 80 rows x 64 keys
constexpr int TA_V_BYTES = 2 * TA_VBOX_BYTES;
constexpr int TA_KV_STAGE = TA_K_BYTES + TA_V_BYTES;
constexpr int TA_OFF_Q = 0;
constexpr int TA_OFF_KV = TA_Q_BYTES;
constexpr int TA_KV_STAGES = 4;
constexpr int TA_OFF_BAR = TA_OFF_KV + TA_KV_STAGES * TA_KV_STAGE;
constexpr int TA_SMEM = TA_OFF_BAR + 256 + 1024;
constexpr int TA_THREADS = 384;
static_assert(TA_Q_BYTES % 1024 == 0 && TA_VBOX_BYTES % 1024 == 0, "operand tiles must stay 1024-B aligned");
static_assert(TA_SMEM <= 227 * 1024, "shared memory budget");

__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}

// S = Q K^T for one 128-key tile (the 64-wide SW128 part of the head dim in four k16 steps, then the 16-wide SW32 part)
__device__ __forceinline__ void issue_qk(float* s, uint64_t dq, uint64_t dq2, uint32_t ka) {
    const uint64_t dk = wgmma_desc_kmajor<128>(ka), dk2 = wgmma_desc_kmajor<32>(ka + 128 * 128);
#pragma unroll
    for (int i = 0; i < 4; ++i) wgmma_ss<128>(s, dq + 2 * i, dk + 2 * i, i > 0 ? 1u : 0u);
    wgmma_ss<128>(s, dq2, dk2, 1u);
}

// O += P V for one 128-key tile: the score fragment of key block c (16 keys) is exactly the m64k16 A fragment; one m64n72k16 per
// block covers the 72 stored columns (V^T box rows are head dims, 128 B apart)
__device__ __forceinline__ void issue_pv(float* o, const uint32_t* pa, uint32_t va) {
#pragma unroll
    for (int c = 0; c < 8; ++c) wgmma_rs<TA_DO>(o, pa + 4 * c, wgmma_desc_kmajor<128>(va + (c >> 2) * TA_VBOX_BYTES) + 2 * (c & 3), 1u);
}

// Online softmax of one score tile in place: masks keys >= nvalid, updates the running row max and the per-thread partial row sums,
// leaves the probabilities in s and returns the rescale factor of O in alpha
__device__ __forceinline__ void softmax_tile(float* s, int nvalid, int qd, float scale_log2, float* m_run, float* l_part, float* alpha) {
    if (nvalid < TA_BKV) {
#pragma unroll
        for (int i = 0; i < 64; ++i)
            if (8 * (i >> 2) + 2 * qd + (i & 1) >= nvalid) s[i] = -INFINITY;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    float msc[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const float m_new = fmaxf(m_run[r], quad_max(mx[r]));
        alpha[r] = ex2((m_run[r] - m_new) * scale_log2);       // first tile: 2^-inf = 0 (O and the sum are still zero)
        m_run[r] = m_new;
        msc[r] = m_new * scale_log2;
    }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        s[i] = ex2(fmaf(s[i], scale_log2, -msc[(i >> 1) & 1]));
        sum[(i >> 1) & 1] += s[i];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) l_part[r] = l_part[r] * alpha[r] + sum[r];
}
// the probabilities as the fp16 A fragments of P V
__device__ __forceinline__ void pack_p(const float* s, uint32_t* pa) {
#pragma unroll
    for (int i = 0; i < 32; ++i) pa[i] = pack_h2(s[2 * i], s[2 * i + 1]);
}

__global__ void __launch_bounds__(TA_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tmQa, const __grid_constant__ CUtensorMap tmQb, const __grid_constant__ CUtensorMap tmKa,
                    const __grid_constant__ CUtensorMap tmKb, const __grid_constant__ CUtensorMap tmV, __half* __restrict__ out, int H, int Nq, int Nk,
                    int Dh, float scale_log2) {
    extern __shared__ __align__(1024) uint8_t ta_smem_raw[];
    // 1024-B alignment by pointer arithmetic on the __shared__ array (an integer round trip would demote every later
    // access to generic LD/ST instead of LDS/STS)
    uint8_t* smem = ta_smem_raw + ((1024u - (smem_u32(ta_smem_raw) & 1023u)) & 1023u);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + TA_OFF_BAR);
    uint64_t* q_full = bars;                             // 1
    uint64_t* k_full = bars + 1;                         // TA_KV_STAGES each
    uint64_t* v_full = bars + 1 + TA_KV_STAGES;
    uint64_t* k_empty = bars + 1 + 2 * TA_KV_STAGES;
    uint64_t* v_empty = bars + 1 + 3 * TA_KV_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * TA_BQ;
    const int h = blockIdx.y, b = blockIdx.z;
    const int bh = b * H + h;
    const int nkt = (Nk + TA_BKV - 1) / TA_BKV;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmQa); tma_prefetch_desc(&tmQb); tma_prefetch_desc(&tmKa); tma_prefetch_desc(&tmKb); tma_prefetch_desc(&tmV);
    }
    if (warp == 1 && lane == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < TA_KV_STAGES; ++i) {
            mbar_init(&k_full[i], 1);
            mbar_init(&v_full[i], 1);
            mbar_init(&k_empty[i], 8);       // one lane of each of the eight consumer warps
            mbar_init(&v_empty[i], 8);
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 0) {
            if (elect_one()) {
                mbar_arrive_expect_tx(q_full, TA_Q_BYTES);
                uint8_t* qs = smem + TA_OFF_Q;
                tma_load_2d(qs, &tmQa, q_full, 0, bh * Nq + q0);
                tma_load_2d(qs + 128 * 128, &tmQb, q_full, 64, bh * Nq + q0);
            }
            __syncwarp();
            for (int j = 0; j < nkt; ++j) {
                const int s = j % TA_KV_STAGES;
                const uint32_t ph = ((j / TA_KV_STAGES) & 1) ^ 1;
                uint8_t* ks = smem + TA_OFF_KV + s * TA_KV_STAGE;
                uint8_t* vs = ks + TA_K_BYTES;
                mbar_wait(&k_empty[s], ph);
                if (elect_one()) {
                    mbar_arrive_expect_tx(&k_full[s], TA_K_BYTES);
                    const int krow = bh * Nk + j * TA_BKV;
                    tma_load_2d(ks, &tmKa, &k_full[s], 0, krow);
                    tma_load_2d(ks + 128 * 128, &tmKb, &k_full[s], 64, krow);
                }
                __syncwarp();
                mbar_wait(&v_empty[s], ph);
                if (elect_one()) {
                    mbar_arrive_expect_tx(&v_full[s], TA_V_BYTES);
                    tma_load_2d(vs, &tmV, &v_full[s], j * TA_BKV, bh * TA_DHP);
                    tma_load_2d(vs + TA_VBOX_BYTES, &tmV, &v_full[s], j * TA_BKV + 64, bh * TA_DHP);
                }
                __syncwarp();
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int w = (warp >> 2) - 1;               // consumer warpgroup: query rows 64 w .. 64 w + 63 of the tile
        const int qd = lane & 3;
        const uint32_t sbase = smem_u32(smem);
        const uint64_t dq = wgmma_desc_kmajor<128>(sbase + TA_OFF_Q + w * 64 * 128);
        const uint64_t dq2 = wgmma_desc_kmajor<32>(sbase + TA_OFF_Q + 128 * 128 + w * 64 * 32);
        float o[TA_DO / 2];
#pragma unroll
        for (int i = 0; i < TA_DO / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};   // rows lane/4 and lane/4 + 8 of this warp's 16
        float alpha[2];
        uint32_t pa[32];                             // P of the tile whose PV is issued next

        // Turn r (0 .. nkt) issues S_r = Q K_r^T (r < nkt) and O += P_{r-1} V_{r-1} (r > 0).  Consumer 0 takes turn 0 without waiting;
        // every other turn waits for the other consumer's pass, and a pass is made only when the other consumer has a turn left.
        // Both consumers take all nkt + 1 turns whichever of their rows exist, so every bar.arrive meets its bar.sync.
        const auto turn_begin = [&](int r) { if (w == 1 || r > 0) pp_turn_wait(w); };
        const auto turn_end = [&](int r) { if (w == 0 || r < nkt) pp_turn_pass(w); };
        const auto k_addr = [&](int j) { return sbase + TA_OFF_KV + (j % TA_KV_STAGES) * TA_KV_STAGE; };
        const auto release = [&](uint64_t* empty, int j) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[j % TA_KV_STAGES]);
        };

        mbar_wait(q_full, 0);
        mbar_wait(&k_full[0], 0);
        float s[64];
        turn_begin(0);
        wgmma_fence();
        issue_qk(s, dq, dq2, k_addr(0));
        wgmma_commit();
        turn_end(0);
        wgmma_wait<0>();
        acc_fence<64>(s);
        release(k_empty, 0);
        softmax_tile(s, Nk, qd, scale_log2, m_run, l_part, alpha);   // O is still zero: no rescale
        pack_p(s, pa);
        mbar_wait(&v_full[0], 0);

        // FA3 order: S_j's softmax runs while PV_{j-1} is in flight, and O is rescaled by alpha_j once PV_{j-1} has landed, so
        // O_j = O_{j-1} alpha_j + P_j V_j exactly as a serial loop computes it
        for (int j = 1; j < nkt; ++j) {
            const uint32_t ph = (j / TA_KV_STAGES) & 1;
            mbar_wait(&k_full[j % TA_KV_STAGES], ph);
            float s[64];                             // fresh each tile: the first wgmma overwrites it (scale-d 0)
            turn_begin(j);
            wgmma_fence();
            issue_qk(s, dq, dq2, k_addr(j));
            wgmma_commit();
            issue_pv(o, pa, k_addr(j - 1) + TA_K_BYTES);
            wgmma_commit();
            turn_end(j);
            wgmma_wait<1>();                         // S_j complete; PV_{j-1} may still run
            acc_fence<64>(s);
            release(k_empty, j);
            softmax_tile(s, Nk - j * TA_BKV, qd, scale_log2, m_run, l_part, alpha);
            // V_j for the next turn.  Waited between the softmax (pinned ahead of it) and the wait for PV_{j-1}: its spin loop is what
            // keeps ptxas from hoisting that wgmma wait above the exponentials, which would serialise them behind PV_{j-1}
            acc_fence<64>(s);
            mbar_wait(&v_full[j % TA_KV_STAGES], ph);
            wgmma_wait<0>();
            acc_fence<TA_DO / 2>(o);
            release(v_empty, j - 1);
#pragma unroll
            for (int i = 0; i < TA_DO / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
            pack_p(s, pa);                           // only now: P_{j-1} in pa is read by its wgmma until the wait above
        }

        turn_begin(nkt);
        wgmma_fence();
        issue_pv(o, pa, k_addr(nkt - 1) + TA_K_BYTES);
        wgmma_commit();
        turn_end(nkt);
        wgmma_wait<0>();
        acc_fence<TA_DO / 2>(o);
        release(v_empty, nkt - 1);

#pragma unroll
        for (int r = 0; r < 2; ++r) {
            float l = l_part[r];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = 1.0f / l;
            const int row = q0 + w * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
            if (row < Nq) {
                __half* orow = out + (static_cast<size_t>(b) * Nq + row) * (H * Dh) + h * Dh + 2 * qd;
#pragma unroll
                for (int nb = 0; nb < TA_DO / 8; ++nb)
                    if (8 * nb < Dh) *reinterpret_cast<__half2*>(orow + 8 * nb) = __floats2half2_rn(o[4 * nb + 2 * r] * inv, o[4 * nb + 2 * r + 1] * inv);
            }
        }
    }
}

}  // namespace

int launch_attention_tc(const __half* q, const __half* k, const __half* vT, __half* out, int B, int H, int Nq, int Nk, int NkPad, int Dh, float scale,
                        cudaStream_t st) {
    TPX_CHECK(B > 0 && H > 0 && Nq > 0 && Nk > 0, TPX_ERR_SHAPE, "attention_tc: empty problem");
    TPX_CHECK(Dh == 72 || Dh == 64, TPX_ERR_SHAPE, "attention_tc: head dim %d (kernel covers Dh = 72 and 64 in 80-wide tiles)", Dh);
    TPX_CHECK(NkPad % 8 == 0 && NkPad >= Nk, TPX_ERR_SHAPE, "attention_tc: NkPad %d must be a multiple of 8 and >= Nk %d", NkPad, Nk);
    TPX_CHECK(H <= 65535 && B <= 65535, TPX_ERR_SHAPE, "attention_tc: grid too large");
    CUtensorMap mQa, mQb, mKa, mKb, mV;
    int rc;
    const long long qrows = static_cast<long long>(B) * H * Nq, krows = static_cast<long long>(B) * H * Nk;
    if ((rc = make_tensor_map_2d(q, qrows, TA_DHP, TA_DHP, 128, 64, &mQa)) != TPX_OK) return rc;
    if ((rc = make_tensor_map_2d(q, qrows, TA_DHP, TA_DHP, 128, 16, &mQb)) != TPX_OK) return rc;
    if ((rc = make_tensor_map_2d(k, krows, TA_DHP, TA_DHP, 128, 64, &mKa)) != TPX_OK) return rc;
    if ((rc = make_tensor_map_2d(k, krows, TA_DHP, TA_DHP, 128, 16, &mKb)) != TPX_OK) return rc;
    if ((rc = make_tensor_map_2d(vT, static_cast<long long>(B) * H * TA_DHP, NkPad, NkPad, TA_DHP, 64, &mV)) != TPX_OK) return rc;
    static bool attr_set = false;
    if (!attr_set) {
        TPX_CUDA(cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TA_SMEM));
        attr_set = true;
    }
    ProfScope prof(PROF_ATTENTION, st);
    dim3 grid((Nq + TA_BQ - 1) / TA_BQ, H, B);
    TPX_CUDA(launch_pdl(attention_tc_kernel, grid, dim3(TA_THREADS), TA_SMEM, st, mQa, mQb, mKa, mKb, mV, out, H, Nq, Nk, Dh, scale * 1.4426950408889634f));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // namespace tpx

using namespace tpx;

extern "C" int tpx_attention_tc(const void* q, const void* k, const void* vT, void* out, int B, int H, int Nq, int Nk, int NkPad, int Dh, float scale,
                                void* stream) {
    TPX_CHECK(q != nullptr && k != nullptr && vT != nullptr && out != nullptr, TPX_ERR_ARG, "attention_tc: null argument");
    TPX_DEVICE_GUARD();
    return launch_attention_tc(static_cast<const __half*>(q), static_cast<const __half*>(k), static_cast<const __half*>(vT), static_cast<__half*>(out), B, H,
                               Nq, Nk, NkPad, Dh, scale, static_cast<cudaStream_t>(stream));
}
