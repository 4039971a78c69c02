// The CUDA resources behind the C ABI and their errors, host code only (the *_layout.h headers stay free of it).
//
// Every device buffer, pinned host buffer, stream and event a handle holds is one of the move-only owners below: it is
// released when its holder goes away, so a create path that fails half-way and a destroy path free the same things.  A
// handle's destroy function sets the handle's device and drains its streams before its owners go.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <map>
#include <mutex>
#include <string>
#include <utility>

// A failing call records "<call>: <CUDA error string>" in owner->err (what the *_last_error entry points return), or in
// *owner when owner is a std::string*, and makes the calling function return `ret`.
#define VB_CUDA_CHECK(owner, ret, call)                                                   \
    do {                                                                                  \
        const cudaError_t vb_err_ = (call);                                               \
        if (vb_err_ != cudaSuccess) {                                                     \
            vb::error_of(owner) = std::string(#call) + ": " + cudaGetErrorString(vb_err_); \
            return ret;                                                                   \
        }                                                                                 \
    } while (0)

namespace vb {

inline std::string& error_of(std::string* s) { return *s; }
template <class Owner>
auto error_of(Owner& o) -> decltype((o->err)) {
    return o->err;
}

// Owners alive in the process, all kinds together (vb_debug_live_cuda_objects): tests check that it returns to its
// baseline after handles are created, fail and are destroyed.
inline std::atomic<long long> g_live_cuda_objects{0};

// true when `device` names a CUDA device.  cudaGetDeviceCount's error (no driver, no device) is cleared so that it does
// not surface in a later cudaGetLastError.
inline bool device_available(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return device >= 0 && device < n;
}

// One owned handle H, released by Release(H).
template <class H, auto Release>
class CudaOwner {
  public:
    CudaOwner() = default;
    CudaOwner(const CudaOwner&) = delete;
    CudaOwner& operator=(const CudaOwner&) = delete;
    CudaOwner(CudaOwner&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    CudaOwner& operator=(CudaOwner&& o) noexcept {
        std::swap(h_, o.h_);
        return *this;
    }
    ~CudaOwner() { reset(); }
    operator H() const { return h_; }
    H get() const { return h_; }
    void reset() {
        if (!h_) return;
        Release(h_);
        h_ = nullptr;
        g_live_cuda_objects.fetch_sub(1);
    }

  protected:
    // Takes what a successful create call produced (a zero-byte allocation produces nothing to own).
    cudaError_t take(cudaError_t e, H h) {
        reset();
        if (e == cudaSuccess && h) {
            h_ = h;
            g_live_cuda_objects.fetch_add(1);
        }
        return e;
    }

  private:
    H h_ = nullptr;
};

// n elements of T in device memory (cudaMalloc).
template <class T>
class DeviceArray : public CudaOwner<T*, cudaFree> {
  public:
    cudaError_t alloc(size_t n) {
        void* p = nullptr;
        const cudaError_t e = cudaMalloc(&p, n * sizeof(T));
        return this->take(e, static_cast<T*>(p));
    }
};

// n elements of T in page-locked host memory (cudaHostAlloc).
template <class T>
class PinnedArray : public CudaOwner<T*, cudaFreeHost> {
  public:
    cudaError_t alloc(size_t n) {
        void* p = nullptr;
        const cudaError_t e = cudaHostAlloc(&p, n * sizeof(T), cudaHostAllocDefault);
        return this->take(e, static_cast<T*>(p));
    }
};

// A stream that does not synchronise with the legacy default stream.
class Stream : public CudaOwner<cudaStream_t, cudaStreamDestroy> {
  public:
    cudaError_t create() {
        cudaStream_t s = nullptr;
        const cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
        return take(e, s);
    }
};

class Event : public CudaOwner<cudaEvent_t, cudaEventDestroy> {
  public:
    cudaError_t create() {
        cudaEvent_t ev = nullptr;
        const cudaError_t e = cudaEventCreate(&ev);
        return take(e, ev);
    }
};

// Raises `kernel`'s opt-in to dynamic shared memory on the current device to at least `bytes`.  The opt-in is a
// per-device function attribute and handles may live on different GPUs of one process, so the largest value set so far
// is kept per (device, kernel); cudaFuncSetAttribute runs only when a launch asks for more.
inline cudaError_t raise_dynamic_smem(const void* kernel, int bytes) {
    static std::mutex m;
    static std::map<std::pair<int, const void*>, int> raised;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    std::lock_guard<std::mutex> lock(m);
    int& cur = raised[{dev, kernel}];
    if (bytes <= cur) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) cur = bytes;
    return e;
}

}  // namespace vb
