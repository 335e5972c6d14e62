// 3x3x3 / pad 1 convolution on channels-last [P, 8, 8, 8, C] fp16 volumes with narrow outputs (Cout <= 32): the 8^3 tail of the
// VAE decoder (models/vae3d_dib.py:259-267 ResnetBlock convs at the upsampled resolution, :383-385 conv_out).
//
// The general implicit-GEMM kernel (gemm_tc.cuh, AMODE_CONV3) fetches one shifted 128-voxel A tile per tap: 27 L2 -> shared
// memory transfers of the same data per output tile, which is what bounds these layers (N = 32 gives the tensor core nothing
// to amortise them over: 14.5 GB of L2 reads for the 256 -> 32 layer).  Here the input block of an output tile is staged ONCE,
// with its halo, and the 27 taps are 27 shifted VIEWS of it:
//
//   tile   = one primitive x two z-planes = 2 x (8 x 8) output voxels
//   stage  = [4 z][10 y][10 x] voxels x 32 channels (one 5-D TMA box starting at (-1,-1,z0-1); the halo is the TMA's out-of-
//            bounds zero fill), 64-B rows in the 64-B swizzle, + the 27 weight tiles [Cout x 32] of that channel chunk
//   MMA    = per tap and z-plane one wgmma M = 64 (rows = (y, x) of the plane): the A descriptor starts at voxel
//            (z + kz, ky, kx) of the block, rows x -> x+1 are 64 B apart, row groups y -> y+1 are one block line (10 x 64 B)
//            apart (the descriptor's stride-byte-offset), so no data is moved or repacked.  The two z-planes are the two
//            register accumulators of the consumer warpgroup.
//   K loop = channel chunks of 32 (x 27 taps x 2 k-steps of 16).
// Roles: warp 0 TMA producer, warps 4-7 one consumer warpgroup (wgmma + the per-thread epilogue shared with the GEMM: bias /
// residual-scale / NCDHW output; warp q holds rows 16 q .. 16 q + 15 of both planes and hands them to one-row-per-thread form
// through its exchange buffer).
#include "kernels.cuh"

namespace tpx {

namespace {

constexpr int CH_XH = 10, CH_YH = 10, CH_ZH = 4;                 // staged block extent (voxels)
constexpr int CH_ROWS = CH_ZH * CH_YH * CH_XH;                   // 400
constexpr int CH_KC = 32;                                        // channels per chunk
constexpr int CH_A_BYTES = CH_ROWS * CH_KC * 2;                  // 25600

template <int BN>
struct HaloCfg {
    static constexpr int B_TAP_BYTES = BN * CH_KC * 2;
    static constexpr int B_BYTES = 27 * B_TAP_BYTES;
    static constexpr int STAGE_BYTES = CH_A_BYTES + B_BYTES;
    static constexpr int XCHG_BYTES = 4 * XCHG_FLOATS * 4;
    static constexpr int STAGES_RAW = (200 * 1024) / STAGE_BYTES;
    static constexpr int STAGES = STAGES_RAW > 4 ? 4 : STAGES_RAW;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + XCHG_BYTES + 256 + 2048;
    static_assert(STAGE_BYTES % 1024 == 0 && B_TAP_BYTES % 512 == 0, "operand tiles must stay aligned to the swizzle pattern");
    static_assert(STAGES >= 2 && SMEM_BYTES <= 227 * 1024, "shared memory budget");
};

struct HaloArgs {
    int P, C, nchunks;
    GemmArgs g;
};

template <int BN, int EPI>
__global__ void __launch_bounds__(256, 1)
conv3_halo_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const HaloArgs ha) {
    using Cfg = HaloCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw;
    if ((smem_u32(smem_raw) & 1023u) != 0) __trap();
    constexpr int OFF_XCHG = STAGES * Cfg::STAGE_BYTES;
    constexpr int OFF_BAR = OFF_XCHG + Cfg::XCHG_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    uint64_t* empty_bar = full_bar + STAGES;
    float* s_bias = reinterpret_cast<float*>(smem + OFF_BAR + 256);
    const GemmArgs& g = ha.g;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
    }
    if (warp == 1 && lane == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 4);             // one lane of every consumer warp
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    if (threadIdx.x >= 128) {
        for (int c = threadIdx.x - 128; c < BN; c += 128) s_bias[c] = (g.bias != nullptr && c < g.N) ? __half2float(g.bias[c]) : 0.f;   // weights: not produced by the previous kernel
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();

    const int num_tiles = ha.P * 4;
    const int nchunks = ha.nchunks;

    if (warp == 0) {
        int stage = 0, it = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int p = tile >> 2, z0 = (tile & 3) * 2;
            for (int ck = 0; ck < nchunks; ++ck, ++it) {
                mbar_wait(&empty_bar[stage], phase ^ 1);
                if (elect_one()) {
                    uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
                    // a single-chunk layer has one weight set: each stage slot keeps its copy after its first fill
                    const bool load_b = nchunks > 1 || it < STAGES;
                    mbar_arrive_expect_tx(&full_bar[stage], CH_A_BYTES + (load_b ? Cfg::B_BYTES : 0));
                    tma_load_5d(sa, &tmA, &full_bar[stage], ck * CH_KC, -1, -1, z0 - 1, p);
                    if (load_b) {
#pragma unroll 1
                        for (int tap = 0; tap < 27; ++tap)
                            tma_load_2d(sa + CH_A_BYTES + tap * Cfg::B_TAP_BYTES, &tmB, &full_bar[stage], tap * ha.C + ck * CH_KC, 0);
                    }
                }
                __syncwarp();
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp >= 4) {
        const int quad = warp & 3;
        const uint32_t smem_u = smem_u32(smem);
        float* xb = reinterpret_cast<float*>(smem + OFF_XCHG) + quad * XCHG_FLOATS;
        // exchange row l of warp q: z-plane (l >> 4), row 16 q + (l & 15) of the (y, x) plane
        const int zt = lane >> 4, prow = quad * 16 + (lane & 15);
        const int y = prow >> 3, x = prow & 7;
        float acc[2][BN / 2];
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int p = tile >> 2, z0 = (tile & 3) * 2;
            const int row = (((p * 8 + z0 + zt) * 8 + y) * 8) + x;
            int prev = -1;
            for (int ck = 0; ck < nchunks; ++ck) {
                mbar_wait(&full_bar[stage], phase);
                const uint32_t a_base = smem_u + stage * Cfg::STAGE_BYTES;
                // 27 taps x 2 planes x 2 k-steps, fully unrolled: every descriptor is the stage's base descriptor plus a compile-time
                // constant in its 16-byte-unit address field
                const uint64_t adesc0 = wgmma_desc_kmajor<64>(a_base, CH_XH * CH_KC * 2);
                const uint64_t bdesc0 = wgmma_desc_kmajor<64>(a_base + CH_A_BYTES);
                const uint32_t acc0 = ck != 0 ? 1u : 0u;
                wgmma_fence();
#pragma unroll
                for (int tap = 0; tap < 27; ++tap) {
                    const int kz = tap / 9, ky = (tap / 3) % 3, kx = tap % 3;
#pragma unroll
                    for (int z = 0; z < 2; ++z) {
                        const uint32_t a_off = static_cast<uint32_t>((((z + kz) * CH_YH + ky) * CH_XH + kx) * (CH_KC * 2)) >> 4;
#pragma unroll
                        for (int ks = 0; ks < CH_KC / 16; ++ks)
                            wgmma_ss<BN>(acc[z], adesc0 + a_off + 2 * ks, bdesc0 + ((tap * Cfg::B_TAP_BYTES) >> 4) + 2 * ks, (tap | ks) != 0 ? 1u : acc0);
                    }
                }
                wgmma_commit();
                if (prev >= 0) {                     // the previous chunk's products have retired: its smem slot is free
                    wgmma_wait<1>();
                    if (lane == 0) mbar_arrive(&empty_bar[prev]);
                }
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            acc_fence<BN / 2>(acc[0]);
            acc_fence<BN / 2>(acc[1]);
            HeadCursor hc{0, 0, 0, 0, 0};
            constexpr int CH = BN >= 32 ? 32 : 16;
            uint32_t r[CH];
            acc_rows<CH, 16, 8>(acc[0], acc[1], 0, xb, lane, r);
            epi_chunk<EPI, CH>(g, s_bias, s_bias, false, row, true, 0, 0, r, hc, 0);
        }
    }
}

template <int BN, int EPI>
int launch_halo(const CUtensorMap& ta, const CUtensorMap& tb, const HaloArgs& ha, cudaStream_t st) {
    using Cfg = HaloCfg<BN>;
    auto kern = conv3_halo_kernel<BN, EPI>;
    static bool attr_set = false;
    if (!attr_set) {
        TPX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
        attr_set = true;
    }
    const int tiles = ha.P * 4;
    const int grid = tiles < gemm_num_sms() ? tiles : gemm_num_sms();
    TPX_CUDA(launch_pdl(kern, dim3(grid), dim3(256), Cfg::SMEM_BYTES, st, ta, tb, ha));
    TPX_LAUNCH_CHECK();
    return TPX_OK;
}

}  // namespace

bool conv3_halo_supported(int S, int C, int Cout, int epi) {
    if (S != 8 || C % CH_KC != 0) return false;
    if (Cout == 32) return epi == EPI_STORE || epi == EPI_RESID_SCALE;
    if (Cout == 16) return epi == EPI_NCDHW;
    return false;
}

int launch_conv3_halo(const __half* x, const __half* W, const __half* bias, const __half* resid, float alpha, __half* out, float* out32, int n_valid, int P,
                      int C, int Cout, int epi, cudaStream_t st) {
    TPX_CHECK(conv3_halo_supported(8, C, Cout, epi), TPX_ERR_SHAPE, "conv3_halo: unsupported layer (C %d -> %d, epilogue %d)", C, Cout, epi);
    ProfScope prof(PROF_CONV_GEMM, st);
    HaloArgs ha{};
    ha.P = P; ha.C = C; ha.nchunks = C / CH_KC;
    GemmArgs& a = ha.g;
    a.M = P * 512; a.N = Cout; a.bias = bias; a.post_scale = 1.0f; a.out0 = out; a.ldo = Cout; a.resid = resid; a.alpha = alpha; a.out32 = out32;
    a.n_valid = n_valid; a.S3 = 512;
    CUtensorMap ta, tb;
    const long long dims[5] = {C, 8, 8, 8, P};
    const long long strides[4] = {static_cast<long long>(C) * 2, static_cast<long long>(C) * 16, static_cast<long long>(C) * 128, static_cast<long long>(C) * 1024};
    const int box[5] = {CH_KC, CH_XH, CH_YH, CH_ZH, 1};
    int rc = make_tensor_map_nd(x, 5, dims, strides, box, 64, &ta);
    if (rc != TPX_OK) return rc;
    rc = make_tensor_map_2d(W, Cout, 27LL * C, 27LL * C, Cout, CH_KC, &tb);        // [Cout, 27 C], box Cout rows x 32 channels, 64-B swizzle
    if (rc != TPX_OK) return rc;
    if (Cout == 32 && epi == EPI_STORE) return launch_halo<32, EPI_STORE>(ta, tb, ha, st);
    if (Cout == 32 && epi == EPI_RESID_SCALE) return launch_halo<32, EPI_RESID_SCALE>(ta, tb, ha, st);
    return launch_halo<16, EPI_NCDHW>(ta, tb, ha, st);
}

}  // namespace tpx
