// Common helpers of libtpx_b200.  Host: error plumbing, buffer carving and the model handles' parameter store.  Device: mbarrier,
// TMA and wgmma PTX wrappers, inline PTX for CUDA 12.x / sm_90a; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <functional>
#include <string>
#include <vector>

#include "../../include/tpx.h"

namespace tpx {

// ------------------------------------------------------------------------------------------------
// error plumbing (host)
// ------------------------------------------------------------------------------------------------
// status codes (TPX_OK, TPX_ERR_*) and dtype tags come from include/tpx.h
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
#define TPX_CUDA(call)                                                   \
    do {                                                                 \
        cudaError_t _e = (call);                                         \
        if (_e != cudaSuccess) return ::tpx::cuda_fail(_e, #call);       \
    } while (0)
#define TPX_CHECK(cond, code, ...)                                       \
    do {                                                                 \
        if (!(cond)) { ::tpx::set_error(__VA_ARGS__); return (code); }   \
    } while (0)
// Device guard of the stateless entry points: after the argument checks, before the first CUDA call, so that a device
// other than sm_90 fails here with TPX_ERR_CUDA and a message naming the check rather than at some later launch.
#define TPX_DEVICE_GUARD()                              \
    do {                                                \
        const int _rc = tpx_device_check();             \
        if (_rc != TPX_OK) return _rc;                  \
    } while (0)
void note_launch();
#define TPX_LAUNCH_CHECK()              \
    do {                                \
        ::tpx::note_launch();           \
        TPX_CUDA(cudaGetLastError());   \
    } while (0)

// Optional per-kernel-class device timing (bench.py roofline leg): RAII scope that brackets the launches
// issued inside it with a CUDA event pair on the launching stream when profiling is enabled.
enum ProfClass : int { PROF_GEMM = 0, PROF_ATTENTION = 1, PROF_LN = 2, PROF_GEMV = 3, PROF_ELEMWISE = 4, PROF_CONV_GEMM = 5, PROF_GROUPNORM = 6, PROF_VAE_MISC = 7, PROF_NCLASS = 8 };
struct ProfScope {
    ProfScope(int cls, cudaStream_t st);
    ~ProfScope();
    int idx;
    cudaStream_t st;
};

// SM count of the current device (cached on first use): the grid of the persistent kernels.
int gemm_num_sms();

// ------------------------------------------------------------------------------------------------
// buffer carving and parameter stores (host)
// ------------------------------------------------------------------------------------------------
inline size_t align_up(size_t bytes, size_t align) { return (bytes + align - 1) / align * align; }

// Bump allocator over one buffer: take<T>(n) hands out the next n elements and moves on by n * sizeof(T) rounded up to `align`
// bytes.  With a null base it hands out nulls and only counts, so a *_bytes query and the call it sizes share one layout.
struct Carve {
    uint8_t* base;
    size_t align = 256;
    size_t off = 0;
    template <class T>
    T* take(size_t n) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += align_up(n * sizeof(T), align);
        return p;
    }
};

// How a reference tensor is repacked into its fp16 slot (vae_kernels.cu): as it is; a Conv3d k3 weight [Cout, Cin, 3,3,3] as
// [Cout, 27 Cin]; a ConvTranspose3d k3 weight [Cin, Cout, 3,3,3] the same way (rows >= Cout stay zero); a ConvTranspose3d k2 weight
// as 8 [Cout, Cin] matrices; a bias copied 8 times (one per k2 output offset); a stride-2 Conv3d k3 weight for the space-to-depth input.
enum ParamKind { PK_PLAIN, PK_CONV3, PK_CONV3_T, PK_CONVT2, PK_BIAS_REP8, PK_CONV3_S2D };

// The fp16 parameters of a model handle, keyed by the reference's state_dict names: one zero-filled device allocation carved
// into slots, and one declaration per key (slot, expected shape, repack, required).  `what` names the entry point in messages.
class ParamStore {
public:
    bool finalized = false;                  // cleared by every successful set()
    std::vector<std::string> ignored;        // key prefixes of the checkpoint's other half: set() returns 1 and records nothing

    ParamStore() = default;
    ParamStore(const ParamStore&) = delete;
    ParamStore& operator=(const ParamStore&) = delete;
    ~ParamStore();

    // Runs `layout` once to size the store (slots `align` bytes apart), allocates and zero-fills it, then runs `layout` again on it.
    // Zero-fill is part of the contract: padded rows and optional tensors that are never given read as 0.
    int create(size_t align, const std::function<void(ParamStore&)>& layout);
    // for `layout`: a slot that is no key, and the declaration of a key in a slot (which it returns)
    __half* take(size_t n) { return carve_.take<__half>(n); }
    __half* param_at(__half* slot, const std::string& key, std::vector<int64_t> shape, int kind = PK_PLAIN, bool required = true);
    __half* param(const std::string& key, std::vector<int64_t> shape, int kind = PK_PLAIN, bool required = true);
    // `name`.weight of shape w_shape and `name`.bias of shape [w_shape[0]], in the slots given or in two new ones
    void weight_bias_at(const std::string& name, __half* W, __half* b, std::vector<int64_t> w_shape, int kind = PK_PLAIN, bool bias_required = true);
    void weight_bias(const std::string& name, __half*& W, __half*& b, std::vector<int64_t> w_shape, int kind = PK_PLAIN, bool bias_required = true);

    // null check, ignored prefixes, lookup (TPX_ERR_KEY), shape check (TPX_ERR_SHAPE), repack on `st`, then mark seen
    int set(const char* what, const char* key, const void* src, int dtype, const int64_t* shape, int ndim, cudaStream_t st);
    int get(const char* what, const char* key, void* dst, int dtype, cudaStream_t st);
    bool seen(const __half* slot) const;
    int complete(const char* what) const;    // TPX_ERR_STATE naming the first required key not set yet

private:
    struct Entry {
        std::string key;
        __half* ptr;
        std::vector<int64_t> shape;
        int kind;
        bool required, seen;
    };
    Entry* find(const char* key);
    __half* dev_ = nullptr;
    Carve carve_{nullptr};
    std::vector<Entry> entries_;
};

#ifdef __CUDACC__
// Launch with the programmatic-stream-serialization attribute (PDL).  The kernel MUST call pdl_wait() before its
// first access to global memory that an earlier kernel in the stream may have written.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    static const bool pdl_on = !(getenv("TPX_NO_PDL") != nullptr && getenv("TPX_NO_PDL")[0] == '1');   // debugging switch
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = pdl_on ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif

// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ uint32_t elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
        "elect.sync rx|px, 0xffffffff;\n\t"
        "selp.b32 %0, 1, 0, px;\n\t}\n"
        : "=r"(pred));
    return pred;
}

// ---- programmatic dependent launch ------------------------------------------------------------------
// Every kernel launched through launch_pdl() runs its prologue (barrier init, descriptor prefetch)
// while the previous kernel of the stream drains, then waits here before touching global memory.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (-> launch failure) instead of hanging the device.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) __trap();   // no printf here: a call inside the wgmma pipeline makes ptxas serialise it
    }
}

// ---- TMA ----------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
        : "memory");
}

// TMA stores: shared::cta -> global through a tensor map (rows / columns outside the tensor are clipped), bulk-group completion.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src_smem, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src_smem),
                 "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, uint32_t src_smem, int c0, int c1, int c2, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
                 "r"(src_smem), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
                 : "memory");
}
// element-wise  global += shared  performed by the L2 (fp32 add, one add per element: deterministic)
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, uint32_t src_smem, int c0, int c1) {
    asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
                 "r"(src_smem), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }   // sources reusable
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }             // writes performed

// ---- wgmma (warpgroup MMA, fp16 x fp16 -> fp32 in registers) ---------------------------------------
// Issued by all 128 threads of a warpgroup.  Sequence: wgmma_fence(); wgmma_*(...) ...; wgmma_commit(); wgmma_wait<N>();
// the accumulator registers may be read only after the wait (acc_fence pins them behind it for the compiler).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor, K-major operand, rows of SW bytes (SW in {128,64,32}) written by TMA with the matching
// swizzle; consecutive 8-row groups are sbo_bytes apart.  Bit layout: start>>4 [0,14), LBO>>4 [16,30) (unused for swizzled
// K-major), SBO>>4 [32,46), swizzle mode [62,64) (1 = 128 B, 2 = 64 B, 3 = 32 B).  A k-step of 16 elements is +32 B: desc + 2.
template <int SW>
__device__ __forceinline__ uint64_t wgmma_desc_kmajor(uint32_t smem_addr, uint32_t sbo_bytes = SW * 8) {
    constexpr uint64_t layout = SW == 128 ? 1ull : (SW == 64 ? 2ull : 3ull);
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(sbo_bytes >> 4) << 32;
    d |= layout << 62;
    return d;
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T  (N in {8, 16, 32, 64, 128, 144} for _ss, 72 for _rs).  d: this thread's N/2 accumulator registers (row lane/4 (+8) of the warp's 16 rows,
// columns 8 j + 2 (lane%4) (+1) for d[4 j .. 4 j + 3]); scale_d = 0 overwrites D.  _ss: A and B from shared memory;
// _rs: A from registers (the m64k16 fragment: a[0], a[2] row lane/4, a[1], a[3] row lane/4 + 8; k = 2 (lane%4) (+8)).
template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t da, uint64_t db, uint32_t scale_d);
template <int N>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_ss<8>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<16>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<32>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<64>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<128>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_ss<144>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n144k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_rs<72>(float* d, const uint32_t* a, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %41, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n72k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35}, {%36, %37, %38, %39}, %40, p, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// Ping-pong hand-off of the tensor cores between the two consumer warpgroups of a CTA (named barriers 3, 4; id 0 is __syncthreads):
// consumer cw waits on 3 + cw until the other one has issued its wgmma for the current turn, then passes the turn back.  Every
// arrive must be matched by exactly one wait, or the CTA hangs.
__device__ __forceinline__ void pp_turn_wait(int cw) { asm volatile("bar.sync %0, 256;" ::"r"(cw + 3) : "memory"); }
__device__ __forceinline__ void pp_turn_pass(int cw) { asm volatile("bar.arrive %0, 256;" ::"r"((cw ^ 1) + 3) : "memory"); }

// A 64 x N product for any N that is a multiple of 8, as the widest instructions that tile it (144 is one instruction); the B
// descriptor advances by n rows of b_row_bytes (n stays a multiple of 8, so every piece starts on an 8-row group).
template <int N>
__device__ __forceinline__ void wgmma_ss_n(float* d, uint64_t da, uint64_t db, uint32_t scale_d, uint32_t b_row_bytes) {
    static_assert(N % 8 == 0 && N > 0 && N <= 256, "wgmma N");
    constexpr int W = N == 144 ? 144 : N >= 128 ? 128 : N >= 64 ? 64 : N >= 32 ? 32 : N >= 16 ? 16 : 8;
    wgmma_ss<W>(d, da, db, scale_d);
    if constexpr (N > W) wgmma_ss_n<N - W>(d + W / 2, da, db + ((W * b_row_bytes) >> 4), scale_d, b_row_bytes);
}

// Hands a warp's accumulator fragment to a row-per-thread epilogue through a warp-private shared-memory buffer (32 rows x 33
// fp32): on return r[i] is column c0 + i of row `lane`.  acc0 / acc1 are the two 64-row accumulators of the thread; fragment
// row lane/4 (+8 for registers 2, 3) of accumulator b is buffer row  b * RB + (e >> 1) * RE + lane / 4.
constexpr int XCHG_FLOATS = 32 * 33;
template <int CW, int RB, int RE>
__device__ __forceinline__ void acc_rows(const float* acc0, const float* acc1, int c0, float* xb, int lane, uint32_t* r) {
    static_assert(CW % 8 == 0 && CW <= 32, "chunk width");
    __syncwarp();
#pragma unroll
    for (int j = 0; j < CW / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int row = (e >> 1) * RE + (lane >> 2), col = 8 * j + 2 * (lane & 3) + (e & 1);
            xb[row * 33 + col] = acc0[(c0 / 8 + j) * 4 + e];
            xb[(row + RB) * 33 + col] = acc1[(c0 / 8 + j) * 4 + e];
        }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < CW; ++i) r[i] = __float_as_uint(xb[lane * 33 + i]);
}


// ---- small numerics -------------------------------------------------------------------------------
__device__ __forceinline__ float h2f_round(float x) { return __half2float(__float2half_rn(x)); }
__device__ __forceinline__ float gelu_tanh(float x) {
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    float inner = k0 * (x + k1 * x * x * x);
    return 0.5f * x * (1.0f + tanhf(inner));
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
#endif  // __CUDACC__

}  // namespace tpx
