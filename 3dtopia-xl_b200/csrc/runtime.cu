// Library-wide runtime of libtpx_b200: the thread-local error message, the device check, the launch counter and the optional
// per-kernel-class event profiling, with their C entry points.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <vector>

#include "tpx_common.cuh"

namespace tpx {

// ---- error plumbing -------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) at %s", static_cast<int>(e), cudaGetErrorString(e), what);
    return TPX_ERR_CUDA;
}

// ---- launch counter + optional event profiling ------------------------------------------------------------------
static std::atomic<long long> g_launches{0};
void note_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

struct ProfRec { int cls; cudaEvent_t a, b; };
static bool g_prof_on = false;
static std::vector<ProfRec> g_prof_recs;
static std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}
ProfScope::ProfScope(int cls, cudaStream_t s) : idx(-1), st(s) {
    if (!g_prof_on) return;
    ProfRec r{cls, prof_event(), prof_event()};
    cudaEventRecord(r.a, st);
    idx = static_cast<int>(g_prof_recs.size());
    g_prof_recs.push_back(r);
}
ProfScope::~ProfScope() {
    if (idx >= 0) cudaEventRecord(g_prof_recs[idx].b, st);
}

int gemm_num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

}  // namespace tpx

using namespace tpx;

extern "C" {

int tpx_version(void) { return TPX_VERSION; }
const char* tpx_last_error(void) { return g_err; }

int tpx_device_check(void) {
    static int checked[64] = {0};   // per device ordinal: 0 unknown, 1 ok (attribute queries are cheap, but this sits on per-kernel entry points)
    int dev = 0;
    TPX_CUDA(cudaGetDevice(&dev));
    if (dev >= 0 && dev < 64 && checked[dev] == 1) return TPX_OK;
    int major = 0, minor = 0;
    TPX_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    TPX_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    TPX_CHECK(major == 9, TPX_ERR_CUDA, "libtpx_b200 is built for sm_90a only; device %d is sm_%d%d (no fallback path exists)", dev, major, minor);
    if (dev >= 0 && dev < 64) checked[dev] = 1;
    return TPX_OK;
}

int64_t tpx_launch_count(void) { return g_launches.load(); }

int tpx_profile_begin(void) {
    for (auto& r : g_prof_recs) { g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b); }
    g_prof_recs.clear();
    g_prof_on = true;
    return TPX_OK;
}

int tpx_profile_end(float* ms_by_class, int64_t* launches_by_class) {
    TPX_CHECK(ms_by_class != nullptr && launches_by_class != nullptr, TPX_ERR_ARG, "profile_end: null argument");
    g_prof_on = false;
    TPX_CUDA(cudaDeviceSynchronize());
    for (int i = 0; i < PROF_NCLASS; ++i) { ms_by_class[i] = 0.f; launches_by_class[i] = 0; }
    for (auto& r : g_prof_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { ms_by_class[r.cls] += ms; launches_by_class[r.cls] += 1; }
        g_prof_pool.push_back(r.a);
        g_prof_pool.push_back(r.b);
    }
    g_prof_recs.clear();
    return TPX_OK;
}

}  // extern "C"
