// gcra_owned.cuh -- one owner for every CUDA resource of the host code; the only file of the engine that creates or
// releases one directly.  Each owner holds one handle, releases it when it goes, and can only be moved.  `make`
// replaces the handle by a new one and returns the CUDA error code (the owner stays empty on failure); `get` is the
// raw handle.  So a failed call releases what it made, and a replacement can be built completely before it is swapped in.
#pragma once
#include <cuda_runtime.h>

#include <utility>

namespace gcra {

template <typename H, auto Release>    // Release(H): cudaFree, cudaStreamDestroy, ...
class Owned {
  public:
    Owned() = default;
    Owned(Owned &&o) noexcept : h_(std::exchange(o.h_, H{})) {}
    Owned &operator=(Owned &&o) noexcept { std::swap(h_, o.h_); return *this; }   // (`o` releases the old handle)
    ~Owned() { reset(); }
    void reset() { if (h_) Release(std::exchange(h_, H{})); }
  protected:
    template <typename E> E took(E e) { if (e) h_ = H{}; return e; }     // e: a CUDA or NCCL result, 0 = success
    H h_{};
};

template <typename T>   // device memory for n elements
struct DevBuf : Owned<void *, cudaFree> {
    cudaError_t make(size_t n) { reset(); return took(cudaMalloc(&h_, n * sizeof(T))); }
    T *get() const { return static_cast<T *>(h_); }
};

// device memory for n elements from the stream-ordered allocator: allocated and released in the order of `stream`'s
// work (cudaMallocAsync / cudaFreeAsync), so neither waits for the device.  The stream must outlive the buffer.
template <typename T>
class StreamBuf {
  public:
    StreamBuf() = default;
    StreamBuf(StreamBuf &&o) noexcept : p_(std::exchange(o.p_, nullptr)), s_(o.s_) {}
    StreamBuf &operator=(StreamBuf &&o) noexcept { std::swap(p_, o.p_); std::swap(s_, o.s_); return *this; }
    ~StreamBuf() { reset(); }
    void reset() { if (p_) cudaFreeAsync(std::exchange(p_, nullptr), s_); }
    cudaError_t make(size_t n, cudaStream_t stream) {
        reset();
        s_ = stream;
        const cudaError_t e = cudaMallocAsync(&p_, n * sizeof(T), stream);
        if (e) p_ = nullptr;
        return e;
    }
    T *get() const { return static_cast<T *>(p_); }
  private:
    void *p_ = nullptr;
    cudaStream_t s_ = nullptr;
};

template <typename T>   // pinned host memory for n elements (cudaHostAllocDefault: what cudaMallocHost allocates)
struct PinnedBuf : Owned<void *, cudaFreeHost> {
    cudaError_t make(size_t n, unsigned flags = cudaHostAllocDefault) { reset(); return took(cudaHostAlloc(&h_, n * sizeof(T), flags)); }
    T *get() const { return static_cast<T *>(h_); }
};

struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
    cudaError_t make() { reset(); return took(cudaStreamCreateWithFlags(&h_, cudaStreamNonBlocking)); }
    // priority: as cudaDeviceGetStreamPriorityRange reports it (lower numbers are higher priorities)
    cudaError_t make(int priority) { reset(); return took(cudaStreamCreateWithPriority(&h_, cudaStreamNonBlocking, priority)); }
    cudaStream_t get() const { return h_; }
};

struct Event : Owned<cudaEvent_t, cudaEventDestroy> {   // flags: cudaEventDisableTiming, or cudaEventDefault to time
    cudaError_t make(unsigned flags) { reset(); return took(cudaEventCreateWithFlags(&h_, flags)); }
    cudaEvent_t get() const { return h_; }
};

struct IpcMapping : Owned<void *, cudaIpcCloseMemHandle> {     // another process's device memory, mapped into this one
    cudaError_t make(cudaIpcMemHandle_t hd) { reset(); return took(cudaIpcOpenMemHandle(&h_, hd, cudaIpcMemLazyEnablePeerAccess)); }
    void *get() const { return h_; }
};

}  // namespace gcra
