// gm_msgstore_*: the message store (msgstore.cuh) over an engine, through the engine's C ABI.  Its kernels run on a stream of
// its own; every call holds the store's mutex, and the store's device work is done when a call returns.
#include <cuda_runtime.h>

#include <memory>

#include "../../include/gpumqtt.h"
#include "cuda_owned.h"
#include "msgstore.cuh"

using namespace gm;

namespace {

struct CudaBackend {
    gm_engine* e;
    int dev;
    Stream s;
    struct Buf {
        DevBuf b;
        void* p = nullptr;
        int ensure(size_t bytes) { CUDA_TRY(b.ensure(std::max<size_t>(bytes, 1))); p = b.p; return GM_OK; }
    };
    CudaBackend(gm_engine* eng, int device) : e(eng), dev(device) {}
    int init() {
        if (dev < 0) return GM_OK;
        CUDA_TRY(cudaSetDevice(dev));
        CUDA_TRY(cudaStreamCreateWithFlags(s.put(), cudaStreamNonBlocking));
        return GM_OK;
    }
    bool device() const { return dev >= 0; }
    cudaStream_t stream() const { return s; }
    int h2d(void* d, const void* h, size_t n) { CUDA_TRY(cudaMemcpyAsync(d, h, n, cudaMemcpyHostToDevice, s)); return GM_OK; }
    int d2h(void* h, const void* d, size_t n) { CUDA_TRY(cudaMemcpyAsync(h, d, n, cudaMemcpyDeviceToHost, s)); return GM_OK; }
    int fill(void* d, int v, size_t n) { CUDA_TRY(cudaMemsetAsync(d, v, n, s)); return GM_OK; }
    int sync() { CUDA_TRY(cudaStreamSynchronize(s)); return GM_OK; }
    int launched() { CUDA_TRY(cudaGetLastError()); return GM_OK; }
    int walk(u64 now, const void* blob, u64 bytes, const u32* offs, u64 n, gm_span* spans, u32* ids, u64 cap, u64* needed, int32_t* status) {
        return gm_retain_match_batch_device_at(e, now, blob, bytes, offs, n, spans, ids, cap, needed, status, s);
    }
    int set_ttl(const char* key, u32 len, u32 handle, u64 deadline) { return gm_retain_set_ttl(e, key, len, handle, deadline, nullptr, nullptr); }
    int bulk_ttl(const char* blob, const u32* offs, const u32* handles, const u64* deadlines, u64 n, u64* n_set) {
        return gm_retain_bulk_load_ttl(e, blob, offs, handles, deadlines, n, n_set);
    }
    int remove_batch(const char* blob, const u32* offs, u64 n) { return gm_retain_remove_batch(e, blob, offs, n, nullptr, nullptr); }
    int remove_expired(u64 now, u32* out, u64 cap, u64* n) { return gm_retain_remove_expired(e, now, out, cap, n); }
};

}  // namespace

struct gm_msgstore : MsCore<CudaBackend> {
    using MsCore::MsCore;
};

extern "C" {

int32_t gm_msgstore_create(gm_engine* e, const gm_msgstore_config* cfg, gm_msgstore** out) {
    if (!e || !out) return GM_ERR_INVALID_ARG;
    *out = nullptr;
    gm_msgstore_config c{};
    c.struct_size = sizeof(c);
    if (cfg) std::memcpy(&c, cfg, std::min<size_t>(cfg->struct_size ? cfg->struct_size : sizeof(c), sizeof(c)));
    if (c.initial_mark_slots && (c.initial_mark_slots < 64 || (c.initial_mark_slots & (c.initial_mark_slots - 1)))) {
        g_err = "initial_mark_slots is a power of two >= 64";
        return GM_ERR_INVALID_ARG;
    }
    const int dev = engine_device(e);
    auto ms = std::make_unique<gm_msgstore>(e, dev);
    GM_TRY(ms->be.init());
    if (dev >= 0) {
        cudaDeviceProp prop{};
        CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
        ms->num_sms = prop.multiProcessorCount;
    }
    if (c.initial_mark_slots) ms->init_slots = c.initial_mark_slots;
    *out = ms.release();
    return GM_OK;
}

void gm_msgstore_destroy(gm_msgstore* ms) {
    if (!ms) return;
    if (ms->be.device()) { cudaSetDevice(ms->be.dev); cudaStreamSynchronize(ms->be.s); }
    delete ms;
}

#define MS_DEVICE(ms) do { if ((ms)->be.device()) CUDA_TRY(cudaSetDevice((ms)->be.dev)); } while (0)

int32_t gm_msgstore_store(gm_msgstore* ms, const char* topic, uint32_t len, uint32_t handle, uint64_t expiry_time_at_ms, const uint32_t* client_keys,
                          const uint32_t* share_keys, uint32_t n_marks) {
    if (!ms) return GM_ERR_INVALID_ARG;
    return ms->store(topic, len, handle, expiry_time_at_ms, client_keys, share_keys, n_marks);
}

int32_t gm_msgstore_store_batch(gm_msgstore* ms, const char* blob, const uint32_t* offsets, const uint32_t* handles, const uint64_t* expiry_time_at_ms, uint64_t n,
                                const uint32_t* mark_offsets, const uint32_t* client_keys, const uint32_t* share_keys) {
    if (!ms) return GM_ERR_INVALID_ARG;
    return ms->store_batch(blob, offsets, handles, expiry_time_at_ms, n, mark_offsets, client_keys, share_keys);
}

int32_t gm_msgstore_get_batch(gm_msgstore* ms, uint64_t now_ms, const char* blob, const uint32_t* offsets, uint64_t n, const uint32_t* client_keys,
                              const uint32_t* share_keys, gm_span* out_spans, uint32_t* out_handles, uint64_t cap, uint64_t* needed, int32_t* status) {
    if (!ms) return GM_ERR_INVALID_ARG;
    MS_DEVICE(ms);
    return ms->get_batch(now_ms, blob, offsets, n, client_keys, share_keys, out_spans, out_handles, cap, needed, status);
}

int32_t gm_msgstore_remove_expired(gm_msgstore* ms, uint64_t now_ms, uint32_t* out_handles, uint64_t cap, uint64_t* n_removed) {
    if (!ms) return GM_ERR_INVALID_ARG;
    return ms->remove_expired(now_ms, out_handles, cap, n_removed);
}

int32_t gm_msgstore_stats_get(gm_msgstore* ms, gm_msgstore_stats* out) {
    if (!ms || !out) return GM_ERR_INVALID_ARG;
    MS_DEVICE(ms);
    return ms->stats(out);
}

}  // extern "C"
