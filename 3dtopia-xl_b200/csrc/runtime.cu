// Library-wide runtime of libtpx_b200: the thread-local error message, the device check, the launch counter, the optional
// per-kernel-class event profiling with their C entry points, and the parameter store of the model handles.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

#include "kernels.cuh"

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

// ---- parameter store ------------------------------------------------------------------------------------
static long long numel(const std::vector<int64_t>& shape) {
    long long n = 1;
    for (int64_t d : shape) n *= d;
    return n;
}

ParamStore::~ParamStore() {
    if (dev_ != nullptr) cudaFree(dev_);
}

int ParamStore::create(size_t align, const std::function<void(ParamStore&)>& layout) {
    carve_ = Carve{nullptr, align};
    layout(*this);
    const size_t bytes = carve_.off;
    TPX_CUDA(cudaMalloc(&dev_, bytes));
    TPX_CUDA(cudaMemset(dev_, 0, bytes));
    entries_.clear();
    carve_ = Carve{reinterpret_cast<uint8_t*>(dev_), align};
    layout(*this);
    return TPX_OK;
}

__half* ParamStore::param_at(__half* slot, const std::string& key, std::vector<int64_t> shape, int kind, bool required) {
    entries_.push_back(Entry{key, slot, std::move(shape), kind, required, false});
    return slot;
}

__half* ParamStore::param(const std::string& key, std::vector<int64_t> shape, int kind, bool required) {
    __half* slot = take(numel(shape));
    return param_at(slot, key, std::move(shape), kind, required);
}

void ParamStore::weight_bias_at(const std::string& name, __half* W, __half* b, std::vector<int64_t> w_shape, int kind, bool bias_required) {
    const int64_t rows = w_shape[0];
    param_at(W, name + ".weight", std::move(w_shape), kind);
    param_at(b, name + ".bias", {rows}, PK_PLAIN, bias_required);
}

void ParamStore::weight_bias(const std::string& name, __half*& W, __half*& b, std::vector<int64_t> w_shape, int kind, bool bias_required) {
    W = take(numel(w_shape));
    b = take(w_shape[0]);
    weight_bias_at(name, W, b, std::move(w_shape), kind, bias_required);
}

ParamStore::Entry* ParamStore::find(const char* key) {
    for (Entry& e : entries_)
        if (e.key == key) return &e;
    return nullptr;
}

int ParamStore::set(const char* what, const char* key, const void* src, int dtype, const int64_t* shape, int ndim, cudaStream_t st) {
    TPX_CHECK(key != nullptr && src != nullptr && shape != nullptr, TPX_ERR_ARG, "%s: null argument", what);
    for (const std::string& p : ignored)
        if (strncmp(key, p.c_str(), p.size()) == 0) return 1;
    Entry* e = find(key);
    TPX_CHECK(e != nullptr, TPX_ERR_KEY, "%s: unexpected key '%s'", what, key);
    bool ok = ndim == static_cast<int>(e->shape.size());
    for (int i = 0; ok && i < ndim; ++i) ok = shape[i] == e->shape[i];
    std::string want;
    for (int64_t d : e->shape) want += (want.empty() ? "" : ",") + std::to_string(d);
    TPX_CHECK(ok, TPX_ERR_SHAPE, "%s: size mismatch for %s: expected [%s], got %d-d", what, key, want.c_str(), ndim);
    const int64_t* s = e->shape.data();
    int rc = TPX_OK;
    switch (e->kind) {
        case PK_PLAIN: rc = launch_to_half(src, dtype, e->ptr, numel(e->shape), st); break;
        case PK_CONV3: rc = launch_pack_conv3(src, dtype, e->ptr, static_cast<int>(s[0]), static_cast<int>(s[1]), 0, st); break;
        case PK_CONV3_T: rc = launch_pack_conv3(src, dtype, e->ptr, static_cast<int>(s[1]), static_cast<int>(s[0]), 1, st); break;
        case PK_CONVT2: rc = launch_pack_convt2(src, dtype, e->ptr, static_cast<int>(s[0]), static_cast<int>(s[1]), st); break;
        case PK_CONV3_S2D: rc = launch_pack_conv3_s2d(src, dtype, e->ptr, static_cast<int>(s[0]), static_cast<int>(s[1]), st); break;
        case PK_BIAS_REP8:
            for (int j = 0; j < 8 && rc == TPX_OK; ++j) rc = launch_to_half(src, dtype, e->ptr + j * s[0], s[0], st);
            break;
    }
    if (rc != TPX_OK) return rc;
    e->seen = true;
    finalized = false;
    return TPX_OK;
}

int ParamStore::get(const char* what, const char* key, void* dst, int dtype, cudaStream_t st) {
    TPX_CHECK(key != nullptr && dst != nullptr, TPX_ERR_ARG, "%s: null argument", what);
    const Entry* e = find(key);
    TPX_CHECK(e != nullptr, TPX_ERR_KEY, "%s: unexpected key '%s'", what, key);
    return launch_from_half(e->ptr, dst, dtype, numel(e->shape), st);
}

bool ParamStore::seen(const __half* slot) const {
    for (const Entry& e : entries_)
        if (e.ptr == slot) return e.seen;
    return false;
}

int ParamStore::complete(const char* what) const {
    for (const Entry& e : entries_) TPX_CHECK(e.seen || !e.required, TPX_ERR_STATE, "%s: missing key '%s' in state_dict", what, e.key.c_str());
    return TPX_OK;
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
