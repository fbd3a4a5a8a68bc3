// Allocator for the host mirrors of the big device tables (multi-GB open-addressing tables that the mutation path
// probes at random): large blocks come from anonymous mmap with MADV_HUGEPAGE, so a random probe costs one
// translation out of a 2-MiB-page TLB instead of a 4-level walk per 4-KiB page.  Purely a host-side speed-up of
// gm_sub_add / gm_bulk_load / gm_compact; a kernel without transparent huge pages simply ignores the advice.
#pragma once
#include <sys/mman.h>

#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <new>
#include <utility>
#include <vector>

#include "host_par.h"

namespace gm {

template <class T>
struct HugeAlloc {
    using value_type = T;
    static constexpr size_t kHugeThreshold = size_t(4) << 20;
    static constexpr size_t kTouchThreshold = size_t(8) << 20;
    static constexpr size_t kAlign = alignof(T) > 64 ? alignof(T) : 64;
    HugeAlloc() = default;
    template <class U> HugeAlloc(const HugeAlloc<U>&) {}
    static size_t rounded(size_t bytes) { return (bytes + (size_t(2) << 20) - 1) & ~((size_t(2) << 20) - 1); }
    T* allocate(size_t n) {
        const size_t bytes = n * sizeof(T);
        if (bytes >= kHugeThreshold) {
            void* p = mmap(nullptr, rounded(bytes), PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
            if (p == MAP_FAILED) throw std::bad_alloc();
            madvise(p, rounded(bytes), MADV_HUGEPAGE);
            // first touch from many threads: the page faults of a multi-GB table are what a bulk load waits for when one
            // thread takes them; several threads take them in a fraction of the time
            if (bytes >= kTouchThreshold && host_threads() > 1) {
                char* c = static_cast<char*>(p);
                parallel_chunks(rounded(bytes) >> 21, host_threads(), [c](unsigned, size_t b, size_t e) { std::memset(c + (b << 21), 0, (e - b) << 21); });
            }
            return static_cast<T*>(p);
        }
        void* p = std::aligned_alloc(kAlign, (bytes + kAlign - 1) / kAlign * kAlign + kAlign);
        if (!p) throw std::bad_alloc();
        return static_cast<T*>(p);
    }
    void deallocate(T* p, size_t n) noexcept {
        const size_t bytes = n * sizeof(T);
        if (bytes >= kHugeThreshold) munmap(p, rounded(bytes));
        else std::free(p);
    }
    template <class U> bool operator==(const HugeAlloc<U>&) const { return true; }
    template <class U> bool operator!=(const HugeAlloc<U>&) const { return false; }
};

// std::vector for the multi-MB working arrays of the bulk paths: its pages are first touched by all host threads
template <class T> using BigVec = std::vector<T, HugeAlloc<T>>;

// Fixed-size table of plain records whose empty state is all-zero bytes (the open-addressing tables: edges, dictionary):
// `assign_zero` takes fresh zero pages from the allocator — the parallel first touch above IS the initialisation, there is
// no second pass writing T{} over several GB as std::vector::assign would do.
template <class T>
class ZeroTable {
  public:
    ZeroTable() = default;
    ~ZeroTable() { release(); }
    ZeroTable(const ZeroTable&) = delete;
    ZeroTable& operator=(const ZeroTable&) = delete;
    ZeroTable(ZeroTable&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    ZeroTable& operator=(ZeroTable&& o) noexcept { if (this != &o) { release(); p_ = o.p_; n_ = o.n_; o.p_ = nullptr; o.n_ = 0; } return *this; }
    void assign_zero(size_t n) {
        release();
        if (!n) return;
        p_ = HugeAlloc<T>().allocate(n);
        n_ = n;
        if (n * sizeof(T) < HugeAlloc<T>::kTouchThreshold || host_threads() <= 1) std::memset(static_cast<void*>(p_), 0, n * sizeof(T));   // big blocks were zeroed by the first touch
    }
    void swap(ZeroTable& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); }
    size_t size() const { return n_; }
    T* data() { return p_; }
    const T* data() const { return p_; }
    T& operator[](size_t i) { return p_[i]; }
    const T& operator[](size_t i) const { return p_[i]; }
    const T* begin() const { return p_; }
    const T* end() const { return p_ + n_; }

  private:
    void release() { if (p_) HugeAlloc<T>().deallocate(p_, n_); p_ = nullptr; n_ = 0; }
    T* p_ = nullptr;
    size_t n_ = 0;
};

// Append-only array whose BASE ADDRESS NEVER MOVES: the whole 32-bit index space is reserved as virtual memory up
// front (MAP_NORESERVE: pages materialise on first touch), so growing never re-allocates.  Used for the host mirror
// of `values` / `ranges`: descriptor-mode match results (gm_desc, include/gpumqtt.h) are resolved by the caller
// against these arrays through plain pointers (gm_values_view), concurrently with mutations that append.
template <class T>
class StableVec {
  public:
    StableVec() { reserve_space(); }
    ~StableVec() { if (base_) munmap(base_, bytes_); }
    StableVec(const StableVec&) = delete;
    StableVec& operator=(const StableVec&) = delete;
    StableVec(StableVec&& o) noexcept : base_(o.base_), bytes_(o.bytes_), size_(o.size_) { o.base_ = nullptr; o.size_ = 0; o.bytes_ = 0; }
    // keeps THIS object's mapping (addresses handed out stay valid): the other array's content is copied in
    StableVec& operator=(StableVec&& o) noexcept {
        if (this != &o) { size_ = 0; append(o.begin(), o.end()); }
        return *this;
    }
    size_t size() const { return size_; }
    bool empty() const { return size_ == 0; }
    T* data() { return base_; }
    const T* data() const { return base_; }
    T& operator[](size_t i) { return base_[i]; }
    const T& operator[](size_t i) const { return base_[i]; }
    const T* begin() const { return base_; }
    const T* end() const { return base_ + size_; }
    void clear() { size_ = 0; }
    void push_back(const T& v) { base_[size_++] = v; }
    template <class It> void append(It first, It last) { for (; first != last; ++first) base_[size_++] = *first; }
    void assign(size_t n, const T& v) { size_ = 0; for (size_t i = 0; i < n; ++i) base_[size_++] = v; }
    static constexpr size_t kMaxElems = (size_t(1) << 32) + 64;

  private:
    void reserve_space() {
        bytes_ = HugeAlloc<T>::rounded(kMaxElems * sizeof(T));
        void* p = mmap(nullptr, bytes_, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_NORESERVE, -1, 0);
        if (p == MAP_FAILED) throw std::bad_alloc();
        base_ = static_cast<T*>(p);
    }
    T* base_ = nullptr;
    size_t bytes_ = 0, size_ = 0;
};

}  // namespace gm
