// Flash-style attention for head_dim 72 (padded to 80) and friends:  out = softmax(q k^T * scale) v
//   (contract of xformers.ops.memory_efficient_attention as called at models/attention.py:54,109 and
//    models/vae3d_dib.py:42 — fp16 q/k/v, fp32 scores / softmax / accumulation, fp16 output)
//
// Layouts: q [B,H,Nq,DHP], k/v [B,H,Nk,DHP] fp16 with zeros in d >= Dh (written by the QKV GEMM epilogue);
//          out [B,Nq,H*Dh] fp16 (the row-major A operand of the following proj GEMM).
// One CTA = 128 query rows of one (batch, head): 8 warps x 16 rows, K/V streamed in 64-key tiles through a
// cp.async double buffer, S and O in registers (mma.sync m16n8k16), online softmax with quad shuffles.
// mma.sync kernel for every head size; attention_tc.cu is the wgmma kernel the released head size (72) runs on.
#include "kernels.cuh"

namespace tpx {

namespace {

constexpr int ATT_BM = 128, ATT_BN = 64, ATT_THREADS = 256;

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
    const uint32_t d = smem_u32(dst);
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float fast_exp2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&h);
}

template <int DHP>
__global__ void __launch_bounds__(ATT_THREADS, (DHP > 80 ? 1 : 2))
attention_kernel(const __half* __restrict__ q, const __half* __restrict__ k, const __half* __restrict__ v, __half* __restrict__ out, int H, int Nq,
                 int Nk, int Dh, float scale_log2) {
    constexpr int LDS = DHP + 8;          // padded smem row (halves): row stride is an odd multiple of 16 B -> conflict-free ldmatrix
    constexpr int KSTEPS = DHP / 16;      // k-steps of Q K^T
    constexpr int DT = DHP / 8;           // 8-wide output d tiles
    constexpr int CPR = DHP / 8;          // 16-B chunks per row
    extern __shared__ __align__(16) uint8_t att_smem[];
    __half* sQ = reinterpret_cast<__half*>(att_smem);
    __half* sK = sQ + ATT_BM * LDS;       // [2][ATT_BN][LDS]
    __half* sV = sK + 2 * ATT_BN * LDS;   // [2][ATT_BN][LDS]

    const int q0 = blockIdx.x * ATT_BM;
    const int h = blockIdx.y, b = blockIdx.z;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t bh = static_cast<size_t>(b) * H + h;
    const __half* qg = q + bh * Nq * DHP;
    const __half* kg = k + bh * Nk * DHP;
    const __half* vg = v + bh * Nk * DHP;

    // ---- prologue: Q tile + first K/V tile ----
    for (int c = threadIdx.x; c < ATT_BM * CPR; c += ATT_THREADS) {
        const int r = c / CPR, cc = c - r * CPR;
        const bool ok = q0 + r < Nq;
        cp_async16(sQ + r * LDS + cc * 8, qg + static_cast<size_t>(ok ? q0 + r : 0) * DHP + cc * 8, ok);
    }
    auto load_kv = [&](int kt, int buf) {
        const int n0 = kt * ATT_BN;
        for (int c = threadIdx.x; c < ATT_BN * CPR; c += ATT_THREADS) {
            const int r = c / CPR, cc = c - r * CPR;
            const bool ok = n0 + r < Nk;
            const size_t off = static_cast<size_t>(ok ? n0 + r : 0) * DHP + cc * 8;
            cp_async16(sK + (buf * ATT_BN + r) * LDS + cc * 8, kg + off, ok);
            cp_async16(sV + (buf * ATT_BN + r) * LDS + cc * 8, vg + off, ok);
        }
    };
    load_kv(0, 0);
    cp_async_commit();

    const int nkt = (Nk + ATT_BN - 1) / ATT_BN;
    float o_acc[DT][4];
#pragma unroll
    for (int i = 0; i < DT; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    uint32_t qf[KSTEPS][4];

    for (int kt = 0; kt < nkt; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nkt) load_kv(kt + 1, buf ^ 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (kt == 0) {
#pragma unroll
            for (int kk = 0; kk < KSTEPS; ++kk) {
                const int row = warp * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                const int col = kk * 16 + (lane >> 4) * 8;
                ldsm_x4(smem_u32(sQ + row * LDS + col), qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3]);
            }
        }
        // ---- S = Q K^T ----
        float s[ATT_BN / 8][4];
#pragma unroll
        for (int i = 0; i < ATT_BN / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
        const __half* sKb = sK + buf * ATT_BN * LDS;
#pragma unroll
        for (int kk = 0; kk < KSTEPS; ++kk) {
#pragma unroll
            for (int np = 0; np < ATT_BN / 16; ++np) {
                const int row = np * 16 + (lane & 7) + ((lane >> 4) & 1) * 8;
                const int col = kk * 16 + ((lane >> 3) & 1) * 8;
                uint32_t b0, b1, b2, b3;
                ldsm_x4(smem_u32(sKb + row * LDS + col), b0, b1, b2, b3);
                mma_16816(s[2 * np], qf[kk], b0, b1);
                mma_16816(s[2 * np + 1], qf[kk], b2, b3);
            }
        }
        // ---- mask the key tail ----
        const int n0 = kt * ATT_BN;
        if (n0 + ATT_BN > Nk) {
#pragma unroll
            for (int i = 0; i < ATT_BN / 8; ++i) {
                const int n = n0 + i * 8 + (lane & 3) * 2;
                if (n >= Nk) s[i][0] = s[i][2] = -INFINITY;
                if (n + 1 >= Nk) s[i][1] = s[i][3] = -INFINITY;
            }
        }
        // ---- online softmax (rows lane/4 and lane/4 + 8) ----
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < ATT_BN / 8; ++i) {
            mx[0] = fmaxf(mx[0], fmaxf(s[i][0], s[i][1]));
            mx[1] = fmaxf(mx[1], fmaxf(s[i][2], s[i][3]));
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        }
        float alpha[2], mscaled[2], rs[2] = {0.f, 0.f};
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const float m_new = fmaxf(m_run[r], mx[r]);
            alpha[r] = fast_exp2((m_run[r] - m_new) * scale_log2);
            m_run[r] = m_new;
            mscaled[r] = m_new * scale_log2;
        }
#pragma unroll
        for (int i = 0; i < ATT_BN / 8; ++i) {
            s[i][0] = fast_exp2(fmaf(s[i][0], scale_log2, -mscaled[0]));
            s[i][1] = fast_exp2(fmaf(s[i][1], scale_log2, -mscaled[0]));
            s[i][2] = fast_exp2(fmaf(s[i][2], scale_log2, -mscaled[1]));
            s[i][3] = fast_exp2(fmaf(s[i][3], scale_log2, -mscaled[1]));
            rs[0] += s[i][0] + s[i][1];
            rs[1] += s[i][2] + s[i][3];
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) l_run[r] = l_run[r] * alpha[r] + rs[r];
#pragma unroll
        for (int i = 0; i < DT; ++i) {
            o_acc[i][0] *= alpha[0];
            o_acc[i][1] *= alpha[0];
            o_acc[i][2] *= alpha[1];
            o_acc[i][3] *= alpha[1];
        }
        // ---- O += P V ----
        const __half* sVb = sV + buf * ATT_BN * LDS;
#pragma unroll
        for (int j = 0; j < ATT_BN / 16; ++j) {
            uint32_t pa[4];
            pa[0] = pack_h2(s[2 * j][0], s[2 * j][1]);
            pa[1] = pack_h2(s[2 * j][2], s[2 * j][3]);
            pa[2] = pack_h2(s[2 * j + 1][0], s[2 * j + 1][1]);
            pa[3] = pack_h2(s[2 * j + 1][2], s[2 * j + 1][3]);
#pragma unroll
            for (int dp = 0; dp < DT / 2; ++dp) {
                const int row = j * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                const int col = dp * 16 + (lane >> 4) * 8;
                uint32_t b0, b1, b2, b3;
                ldsm_x4_t(smem_u32(sVb + row * LDS + col), b0, b1, b2, b3);
                mma_16816(o_acc[2 * dp], pa, b0, b1);
                mma_16816(o_acc[2 * dp + 1], pa, b2, b3);
            }
        }
        __syncthreads();
    }
    cp_async_wait<0>();

    // ---- normalise and store ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const int D = H * Dh;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = q0 + warp * 16 + (lane >> 2) + r * 8;
        if (row >= Nq) continue;
        const float inv = 1.0f / l_run[r];
        __half* orow = out + (static_cast<size_t>(b) * Nq + row) * D + h * Dh;
#pragma unroll
        for (int i = 0; i < DT; ++i) {
            const int d = i * 8 + (lane & 3) * 2;
            if (d < Dh) {
                __half2 o2 = __floats2half2_rn(o_acc[i][2 * r] * inv, o_acc[i][2 * r + 1] * inv);
                *reinterpret_cast<__half2*>(orow + d) = o2;
            }
        }
    }
}

template <int DHP>
int launch_att(const __half* q, const __half* k, const __half* v, __half* out, int B, int H, int Nq, int Nk, int Dh, float scale, cudaStream_t st) {
    constexpr int LDS = DHP + 8;
    constexpr int SMEM = (ATT_BM + 4 * ATT_BN) * LDS * 2;
    auto kern = attention_kernel<DHP>;
    static bool attr_set = false;
    if (!attr_set) {
        TPX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
        attr_set = true;
    }
    dim3 grid((Nq + ATT_BM - 1) / ATT_BM, H, B);
    ProfScope prof(PROF_ATTENTION, st);
    kern<<<grid, ATT_THREADS, SMEM, st>>>(q, k, v, out, H, Nq, Nk, Dh, scale * 1.4426950408889634f);
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // namespace

int launch_attention(const __half* q, const __half* k, const __half* v, __half* out, int B, int H, int Nq, int Nk, int Dh, int DhP, float scale,
                     cudaStream_t st) {
    TPX_CHECK(B > 0 && H > 0 && Nq > 0 && Nk > 0, TPX_ERR_SHAPE, "attention: empty problem B=%d H=%d Nq=%d Nk=%d", B, H, Nq, Nk);
    TPX_CHECK(Dh % 2 == 0 && Dh <= DhP, TPX_ERR_SHAPE, "attention: head dim %d / padded %d", Dh, DhP);
    TPX_CHECK(H <= 65535 && B <= 65535, TPX_ERR_SHAPE, "attention: grid too large (H=%d, B=%d)", H, B);
    switch (DhP) {
        case 16: return launch_att<16>(q, k, v, out, B, H, Nq, Nk, Dh, scale, st);
        case 32: return launch_att<32>(q, k, v, out, B, H, Nq, Nk, Dh, scale, st);
        case 64: return launch_att<64>(q, k, v, out, B, H, Nq, Nk, Dh, scale, st);
        case 80: return launch_att<80>(q, k, v, out, B, H, Nq, Nk, Dh, scale, st);
        case 128: return launch_att<128>(q, k, v, out, B, H, Nq, Nk, Dh, scale, st);
        default: set_error("attention: padded head dim %d not instantiated (16/32/64/80/128)", DhP); return TPX_ERR_SHAPE;
    }
}

}  // namespace tpx

using namespace tpx;

extern "C" int tpx_attention(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk, int Dh, int DhP, float scale,
                             void* stream) {
    TPX_CHECK(q != nullptr && k != nullptr && v != nullptr && out != nullptr, TPX_ERR_ARG, "attention: null argument");
    TPX_DEVICE_GUARD();
    return launch_attention(static_cast<const __half*>(q), static_cast<const __half*>(k), static_cast<const __half*>(v), static_cast<__half*>(out), B, H,
                            Nq, Nk, Dh, DhP, scale, static_cast<cudaStream_t>(stream));
}
