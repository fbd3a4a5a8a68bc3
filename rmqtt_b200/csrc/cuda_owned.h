// Owning types for the CUDA resources of the engine and the router: device buffers, pinned host blocks, streams, events,
// graph executables and the NCCL communicator.  Each is move-only and releases what it holds when it is destroyed, so a
// resource is declared once and needs no release list.  Destroying an empty owner makes no CUDA call: a host-only engine
// never touches the runtime (a cudaFree(nullptr) would create a context).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <cstring>
#include <string>

#include "../../include/gpumqtt.h"

struct ncclComm;   // nccl.h's communicator (ncclComm_t is a pointer to it)

namespace gm {

extern thread_local std::string g_err;   // the text of gm_last_error (defined in engine.cu)

#define CUDA_TRY(expr)                                                                                                  \
    do {                                                                                                                \
        const cudaError_t _e = (expr);                                                                                  \
        if (_e != cudaSuccess) {                                                                                        \
            ::gm::g_err = std::string(#expr) + ": " + cudaGetErrorString(_e);                                           \
            return (_e == cudaErrorNoDevice || _e == cudaErrorInsufficientDriver) ? GM_ERR_NO_DEVICE : GM_ERR_CUDA;     \
        }                                                                                                               \
    } while (0)
#define GM_TRY(expr) do { const int32_t _st = (expr); if (_st != GM_OK) return _st; } while (0)   // pass a failing status on

// an owning allocation of `cap` bytes at `p`, handed back to `Free` (cudaFree, cudaFreeHost) when the owner lets go of it
template <class P, auto Free>
struct Block {
    P* p = nullptr;
    size_t cap = 0;
    Block() = default;
    Block(Block&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    Block& operator=(Block&& o) noexcept { if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; } return *this; }
    ~Block() { release(); }
    void release() { if (p) Free(p); p = nullptr; cap = 0; }
    template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

struct DevBuf : Block<void, cudaFree> {   // device memory (freed on destruction, also on the early-return error paths)
    // grow to at least `bytes`; `keep` copies the old contents over on stream `s` and waits for that stream
    cudaError_t ensure(size_t bytes, bool keep = false, cudaStream_t s = nullptr) {
        if (bytes <= cap) return cudaSuccess;
        size_t ncap = std::max(bytes, cap + cap / 2);
        ncap = (ncap + 255) & ~size_t(255);
        void* np = nullptr;
        cudaError_t e = cudaMalloc(&np, ncap);
        if (e != cudaSuccess) return e;
        if (keep && p && cap) {
            e = cudaMemcpyAsync(np, p, cap, cudaMemcpyDeviceToDevice, s);
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
            if (e != cudaSuccess) { cudaFree(np); return e; }
        }
        release();
        p = np; cap = ncap;
        return cudaSuccess;
    }
};

struct PinnedBuf : Block<char, cudaFreeHost> {   // page-locked host memory
    // a block of exactly `bytes` unless the current one holds them; the first `keep` bytes of the old block are carried over
    cudaError_t ensure(size_t bytes, size_t keep = 0) {
        if (bytes <= cap) return cudaSuccess;
        void* np = nullptr;
        const cudaError_t e = cudaMallocHost(&np, bytes);
        if (e != cudaSuccess) return e;
        if (p && keep) std::memcpy(np, p, std::min(keep, cap));
        release();
        p = static_cast<char*>(np); cap = bytes;
        return cudaSuccess;
    }
};

// an owning handle: `Destroy` runs on a non-null handle when the owner is destroyed, reset or assigned
template <class H, auto Destroy>
class Owned {
  public:
    Owned() = default;
    Owned(Owned&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    Owned& operator=(Owned&& o) noexcept { if (this != &o) { reset(o.h_); o.h_ = nullptr; } return *this; }
    ~Owned() { reset(); }
    void reset(H h = nullptr) { if (h_) Destroy(h_); h_ = h; }
    H* put() { reset(); return &h_; }       // for the create call: releases the old handle, receives the new one
    operator H() const { return h_; }
  private:
    H h_ = nullptr;
};

using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using GraphExec = Owned<cudaGraphExec_t, cudaGraphExecDestroy>;

void nccl_comm_destroy(ncclComm* c);   // ncclCommDestroy through NcclApi, which binds libnccl at run time (engine.cu)
using NcclComm = Owned<ncclComm*, nccl_comm_destroy>;

}  // namespace gm
