// cuda_shim.cpp -- an LD_PRELOAD wrapper of the CUDA runtime calls that create and release resources, for
// tests/test_gpu_lifecycle.py.  libctmr links libcudart.so.12 dynamically, so these definitions take the place of the
// runtime's for every call the library makes; each forwards to the real function, found through the runtime that is
// already loaded (dlopen RTLD_NOLOAD: ctypes loads libctmr RTLD_LOCAL, so RTLD_NEXT would find nothing).
//
// It keeps, per kind (0 device buffers, 1 pinned host buffers, 2 streams, 3 events), the set of live resources and the
// number created.  shim_fail_nth(kind, n) makes the n-th creation of that kind from now on return
// cudaErrorMemoryAllocation without calling the runtime; from that failure until shim_fail_nth(-1, 0), every
// cudaLaunchKernel is refused and counted, so a test can tell that no kernel ran after a failed allocation.
#include <dlfcn.h>

#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <unordered_set>

extern "C" {
typedef int cudaError_t;
typedef void* cudaStream_t;
typedef void* cudaEvent_t;
struct dim3 { unsigned x, y, z; };
}

namespace {
constexpr cudaError_t kSuccess = 0, kMemoryAllocation = 2;
constexpr int kKinds = 4;

std::mutex mu;
std::unordered_set<void*> live[kKinds];
long created[kKinds];
int fail_kind = -1;
long fail_countdown = 0;
bool refusing = false;
long refused = 0;
long get_device_count_calls = 0;

void* real(const char* name) {
    static void* rt = dlopen("libcudart.so.12", RTLD_NOW | RTLD_NOLOAD);
    void* f = rt ? dlsym(rt, name) : nullptr;
    if (!f) {
        std::fprintf(stderr, "cuda_shim: no %s in the loaded libcudart.so.12\n", name);
        std::abort();
    }
    return f;
}
#define REAL(name) reinterpret_cast<decltype(&name)>(real(#name))

bool inject(int kind) {  // under mu: this creation fails
    if (kind != fail_kind || fail_countdown <= 0 || --fail_countdown) return false;
    refusing = true;
    return true;
}

template <class F> cudaError_t make(int kind, void** out, F call) {
    {
        std::lock_guard<std::mutex> g(mu);
        if (inject(kind)) return kMemoryAllocation;
    }
    const cudaError_t e = call();
    if (e == kSuccess && *out) {
        std::lock_guard<std::mutex> g(mu);
        live[kind].insert(*out);
        ++created[kind];
    }
    return e;
}

cudaError_t drop(int kind, void* p, cudaError_t e) {
    if (e == kSuccess && p) {
        std::lock_guard<std::mutex> g(mu);
        live[kind].erase(p);
    }
    return e;
}
}  // namespace

extern "C" {

cudaError_t cudaMalloc(void** p, size_t n) { return make(0, p, [&] { return REAL(cudaMalloc)(p, n); }); }
cudaError_t cudaFree(void* p) { return drop(0, p, REAL(cudaFree)(p)); }
cudaError_t cudaMallocHost(void** p, size_t n) { return make(1, p, [&] { return REAL(cudaMallocHost)(p, n); }); }
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned flags) { return make(1, p, [&] { return REAL(cudaHostAlloc)(p, n, flags); }); }
cudaError_t cudaFreeHost(void* p) { return drop(1, p, REAL(cudaFreeHost)(p)); }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned flags) {
    return make(2, s, [&] { return REAL(cudaStreamCreateWithFlags)(s, flags); });
}
cudaError_t cudaStreamDestroy(cudaStream_t s) { return drop(2, s, REAL(cudaStreamDestroy)(s)); }
cudaError_t cudaEventCreate(cudaEvent_t* e) { return make(3, e, [&] { return REAL(cudaEventCreate)(e); }); }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned flags) {
    return make(3, e, [&] { return REAL(cudaEventCreateWithFlags)(e, flags); });
}
cudaError_t cudaEventDestroy(cudaEvent_t e) { return drop(3, e, REAL(cudaEventDestroy)(e)); }

cudaError_t cudaLaunchKernel(const void* func, dim3 grid, dim3 block, void** args, size_t smem, cudaStream_t s) {
    {
        std::lock_guard<std::mutex> g(mu);
        if (refusing) {
            ++refused;
            return kMemoryAllocation;
        }
    }
    return REAL(cudaLaunchKernel)(func, grid, block, args, smem, s);
}

cudaError_t cudaGetDeviceCount(int* n) {
    {
        std::lock_guard<std::mutex> g(mu);
        ++get_device_count_calls;
    }
    return REAL(cudaGetDeviceCount)(n);
}

// ---- queries and control (ctypes) ----
void shim_counts(long* live_out, long* created_out) {
    std::lock_guard<std::mutex> g(mu);
    for (int k = 0; k < kKinds; ++k) {
        live_out[k] = (long)live[k].size();
        created_out[k] = created[k];
    }
}
void shim_fail_nth(int kind, long n) {  // kind -1: stop failing and refusing
    std::lock_guard<std::mutex> g(mu);
    fail_kind = kind;
    fail_countdown = kind < 0 ? 0 : n;
    refusing = false;
    refused = 0;
}
long shim_refused_launches() {
    std::lock_guard<std::mutex> g(mu);
    return refused;
}
long shim_get_device_count_calls() {
    std::lock_guard<std::mutex> g(mu);
    return get_device_count_calls;
}

}  // extern "C"
