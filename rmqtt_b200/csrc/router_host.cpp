// GpuRouter — see router_host.h.
#include "router_host.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>

namespace gm {

namespace {
std::string ckey(uint64_t node, const std::string& client) { std::string k = std::to_string(node); k.push_back('\0'); k += client; return k; }
std::string ikey(uint64_t node, const std::string& client, uint64_t tag) { std::string k = ckey(node, client); k.push_back('\0'); k += std::to_string(tag); return k; }
}  // namespace

// client keys number the (node id, client id) pairs in order of first appearance; a new key starts online
uint32_t GpuRouter::client_key(uint64_t node_id, const std::string& client) {
    const uint32_t k = intern(client_key_, ckey(node_id, client));
    if (online_words_.size() * 32 <= k) {
        const uint32_t w0 = static_cast<uint32_t>(online_words_.size());
        online_words_.resize(k / 32 + 1, 0xFFFFFFFFu);
        online_dirty_.mark(w0, static_cast<uint32_t>(online_words_.size()));
    }
    return k;
}

void GpuRouter::set_online(uint64_t node_id, const std::string& client, bool online) {
    const uint32_t k = client_key(node_id, client);
    const uint32_t bit = 1u << (k & 31);
    online_words_[k / 32] = online ? (online_words_[k / 32] | bit) : (online_words_[k / 32] & ~bit);
    online_dirty_.mark(k / 32, k / 32 + 1);
}

// the device record of a relation: everything k_relations needs to apply router.rs:184-200 and types.rs:488-506
void GpuRouter::set_rel(uint32_t handle, const Rel& r) {
    if (rel_host_.size() <= handle) rel_host_.resize(handle + 1, gm_rel{0, 0, 0, 0, 0});
    gm_rel d{0, 0, 0, 0, 0};
    uint32_t group = 0;
    if (r.live) {
        d.node_id = r.id.node_id;
        d.client_key = client_key(r.id.node_id, r.client);
        d.id_idx = intern(id_idx_, ikey(r.id.node_id, r.id.client_id, r.id.tag));
        d.sub_id = r.opts.sub_id;
        if (!r.opts.group.empty()) {
            std::string key = filter_names_[r.filter_idx]; key.push_back('\0'); key += r.opts.group;
            const auto ins = group_index_.emplace(key, static_cast<uint32_t>(group_index_.size() + 1));
            group = ins.first->second;
            if (ins.second) {                                          // a new group: an empty block
                grp_hdr_.push_back(gm_span{static_cast<uint32_t>(member_pool_.size()), 0}); grp_cap_.push_back(0);
                grp_filter_.push_back(filter_names_[r.filter_idx]); grp_name_.push_back(r.opts.group);
                hdr_dirty_.mark(group, group + 1);
            }
        }
        d.flags = GM_REL_LIVE | (r.opts.is_v5 ? GM_REL_V5 : 0u) | (r.opts.no_local ? GM_REL_NO_LOCAL : 0u) | (group << 8);
    }
    rel_host_[handle] = d;
    rel_dirty_lo_ = std::min(rel_dirty_lo_, handle); rel_dirty_hi_ = std::max(rel_dirty_hi_, handle + 1);
    if (member_group_.size() <= handle) { member_group_.resize(handle + 1, 0); member_slot_.resize(handle + 1, 0); }
    if (member_group_[handle] != group) {                              // a re-subscribe may change or drop the group
        if (member_group_[handle]) member_remove(handle);
        if (group) member_add(group, handle);
    }
}

void GpuRouter::member_add(uint32_t group, uint32_t handle) {
    if (grp_hdr_[group].cnt == grp_cap_[group]) {                      // full: the block moves to the pool's end with twice the room
        const gm_span old = grp_hdr_[group];
        const uint32_t ncap = std::max<uint32_t>(4, 2 * grp_cap_[group]);
        const uint32_t noff = static_cast<uint32_t>(member_pool_.size());
        member_pool_.resize(member_pool_.size() + ncap, 0xFFFFFFFFu);
        std::copy(member_pool_.begin() + old.off, member_pool_.begin() + old.off + old.cnt, member_pool_.begin() + noff);
        pool_garbage_ += grp_cap_[group];
        grp_hdr_[group].off = noff; grp_cap_[group] = ncap;
        pool_dirty_.mark(noff, noff + old.cnt);
    }
    gm_span& b = grp_hdr_[group];
    member_pool_[b.off + b.cnt] = handle;
    member_group_[handle] = group; member_slot_[handle] = b.cnt;
    pool_dirty_.mark(b.off + b.cnt, b.off + b.cnt + 1);
    b.cnt++;
    hdr_dirty_.mark(group, group + 1);
    groups_changed_ = true;
    if (pool_garbage_ > 4096 && pool_garbage_ * 2 > member_pool_.size()) repack_groups();
}

void GpuRouter::member_remove(uint32_t handle) {                       // the block's last entry takes the freed slot
    const uint32_t group = member_group_[handle];
    gm_span& b = grp_hdr_[group];
    const uint32_t slot = member_slot_[handle], last = member_pool_[b.off + b.cnt - 1];
    member_pool_[b.off + slot] = last; member_slot_[last] = slot;
    member_pool_[b.off + b.cnt - 1] = 0xFFFFFFFFu;
    b.cnt--;
    member_group_[handle] = 0;
    pool_dirty_.mark(b.off + slot, b.off + slot + 1);
    hdr_dirty_.mark(group, group + 1);
    groups_changed_ = true;
}

void GpuRouter::repack_groups() {
    std::vector<uint32_t> pool;
    for (size_t g = 1; g < grp_hdr_.size(); ++g) {
        const gm_span old = grp_hdr_[g];
        const uint32_t off = static_cast<uint32_t>(pool.size());
        pool.insert(pool.end(), member_pool_.begin() + old.off, member_pool_.begin() + old.off + old.cnt);
        pool.resize(off + grp_cap_[g], 0xFFFFFFFFu);
        grp_hdr_[g].off = off;
    }
    member_pool_.swap(pool);
    pool_garbage_ = 0;
    hdr_dirty_.mark(0, static_cast<uint32_t>(grp_hdr_.size()));
    pool_dirty_.mark(0, static_cast<uint32_t>(member_pool_.size()));
}

bool GpuRouter::group(uint32_t g, const std::string** filter, const std::string** name, const uint32_t** members, uint32_t* cnt) const {
    if (g == 0 || g >= grp_hdr_.size()) return false;
    *filter = &grp_filter_[g]; *name = &grp_name_[g];
    *members = member_pool_.data() + grp_hdr_[g].off; *cnt = grp_hdr_[g].cnt;
    return true;
}

int32_t GpuRouter::add(const char* filter, uint32_t len, const Id& id, const Opts& opts) {
    std::string f(filter, len);
    uint32_t fi;
    auto fit = filter_index_.find(f);
    const bool new_filter_name = fit == filter_index_.end();
    fi = new_filter_name ? static_cast<uint32_t>(filter_names_.size()) : fit->second;
    auto rit = relations_.find(fi);
    uint32_t handle = 0;
    bool existing = false;
    if (rit != relations_.end()) {
        auto cit = rit->second.find(id.client_id);
        if (cit != rit->second.end()) { handle = cit->second; existing = true; }
    }
    if (!existing) {
        if (!free_handles_.empty()) {
            // a handle freed by remove() may still be in the DEVICE trie of an engine that only flushes on demand
            // (GM_FLAG_MANUAL_FLUSH): ship the pending removals before the handle can mean another subscription
            if (unflushed_removes_) { const int32_t frc = gm_flush(e_); if (frc != GM_OK) return frc; unflushed_removes_ = false; }
            handle = free_handles_.back();
        }
        else handle = static_cast<uint32_t>(by_handle_.size());
    }
    // Topic::from_str + topics.insert (router.rs:419-421): an invalid filter is an Err before any state changes
    int32_t changed = 0;
    int32_t rc = gm_sub_add(e_, filter, len, handle, &changed);
    if (rc != GM_OK) return rc;
    if (new_filter_name) { filter_index_.emplace(f, fi); filter_names_.push_back(f); }
    if (!existing) {
        if (!free_handles_.empty()) free_handles_.pop_back();
        else by_handle_.emplace_back();
    }
    auto& clients = relations_[fi];
    if (clients.empty()) topics_++;                                  // or_insert_with(|| topics_count.inc()) (router.rs:426-429)
    Rel& r = by_handle_[handle];
    r.filter_idx = fi; r.client = id.client_id; r.id = id; r.opts = opts; r.live = true;
    if (clients.emplace(id.client_id, handle).second) routes_++;     // HashMap::insert: replace keeps the count (router.rs:430-433)
    set_rel(handle, r);
    return GM_OK;
}

int32_t GpuRouter::remove(const char* filter, uint32_t len, const Id& id, bool* removed) {
    if (removed) *removed = false;
    auto fit = filter_index_.find(std::string(filter, len));
    if (fit == filter_index_.end()) return GM_OK;
    auto rit = relations_.find(fit->second);
    if (rit == relations_.end()) return GM_OK;
    auto cit = rit->second.find(id.client_id);
    if (cit == rit->second.end()) return GM_OK;
    const uint32_t handle = cit->second;
    if (!(by_handle_[handle].id == id)) return GM_OK;                 // "input id not the same" (router.rs:444-451)
    rit->second.erase(cit);
    routes_--;
    if (rit->second.empty()) { relations_.erase(rit); topics_--; }    // router.rs:466-473
    by_handle_[handle].live = false;
    set_rel(handle, by_handle_[handle]);
    free_handles_.push_back(handle);
    unflushed_removes_ = true;
    int32_t changed = 0;
    int32_t rc = gm_sub_remove(e_, filter, len, handle, &changed);
    if (rc != GM_OK) return rc;
    if (removed) *removed = true;
    return GM_OK;
}

bool GpuRouter::relation(uint32_t handle, const std::string** filter, const std::string** client) const {
    if (handle >= by_handle_.size() || !by_handle_[handle].live) return false;
    *filter = &filter_names_[by_handle_[handle].filter_idx];
    *client = &by_handle_[handle].client;
    return true;
}

int32_t GpuRouter::matched_filters_batch(const char* blob, const uint32_t* offs, uint64_t n, std::vector<gm_span>& spans, std::vector<uint32_t>& filters,
                                         std::vector<int32_t>& status) {
    spans.assign(n, gm_span{0, 0}); status.assign(n, 0); filters.clear();
    if (n == 0) return GM_OK;
    std::vector<gm_span> dsp(n);
    std::vector<gm_desc> descs(std::max<uint64_t>(64, 8 * n));
    uint64_t needed = 0;
    for (;;) {
        const int32_t rc = gm_match_batch_desc(e_, blob, offs, n, dsp.data(), descs.data(), descs.size(), &needed, status.data());
        if (rc == GM_ERR_CAPACITY) { descs.resize(needed + 64); continue; }
        if (rc != GM_OK) return rc;
        break;
    }
    gm_values vv{};
    GM_TRY(gm_values_view(e_, &vv));
    for (uint64_t i = 0; i < n; ++i) {
        const size_t begin = filters.size();
        if (status[i] == 0) {
            for (uint32_t k = 0; k < dsp[i].cnt; ++k) {
                const gm_desc& d = descs[dsp[i].off + k];
                uint32_t h;                                                   // any member of the set names the filter
                if (d.cnt == 1) h = d.ref;
                else if (d.cnt == 0xFFFFu) h = vv.values[vv.ranges[d.ref].off];
                else h = vv.values[d.ref];
                if (h < by_handle_.size()) filters.push_back(by_handle_[h].filter_idx);
            }
            std::sort(filters.begin() + begin, filters.end());                 // .unique(): a literal '+' / '#' topic level visits a wildcard child twice
            filters.erase(std::unique(filters.begin() + begin, filters.end()), filters.end());
        }
        spans[i] = gm_span{static_cast<uint32_t>(begin), static_cast<uint32_t>(filters.size() - begin)};
    }
    return GM_OK;
}

bool GpuRouter::filter(uint32_t fi, const std::string** name, std::vector<uint64_t>& node_ids) const {
    if (fi >= filter_names_.size()) return false;
    *name = &filter_names_[fi];
    node_ids.clear();
    auto it = relations_.find(fi);
    if (it != relations_.end()) for (const auto& kv : it->second) node_ids.push_back(by_handle_[kv.second].id.node_id);
    std::sort(node_ids.begin(), node_ids.end());
    node_ids.erase(std::unique(node_ids.begin(), node_ids.end()), node_ids.end());
    return true;
}

// per-client de-dup of ONE topic on the host — only for topics the kernel flagged (more v5 relations than it stages).  A v5
// relation joins the de-dup unless it is a shared member of the plain call (`chosen` false: every member passes through); as on
// the device, the client's smallest handle represents it, with that record's group field, and the ids accumulate in list order.
int32_t GpuRouter::host_dedup_topic(const gm_sub_relation* in, uint32_t cnt, bool chosen, std::vector<gm_sub_relation>& rels, std::vector<uint32_t>& sub_ids) {
    struct V5Entry { size_t rel_pos; std::vector<uint32_t> ids; };
    std::unordered_map<uint32_t, V5Entry> v5;                 // client_key -> (its relation, accumulated ids)
    for (uint32_t k = 0; k < cnt; ++k) {
        const uint32_t h = in[k].handle;
        const gm_rel& d = rel_host_[h];
        const gm_sub_relation sr{d.node_id, h, in[k].group, 0, 0};
        if (!(d.flags & GM_REL_V5) || (!chosen && (d.flags >> 8))) { rels.push_back(sr); continue; }
        auto it = v5.find(d.client_key);
        if (it == v5.end()) { it = v5.emplace(d.client_key, V5Entry{rels.size(), {}}).first; rels.push_back(sr); }
        else if (h < rels[it->second.rel_pos].handle) rels[it->second.rel_pos] = sr;
        if (d.sub_id) it->second.ids.push_back(d.sub_id);
    }
    for (auto& kv : v5) {
        gm_sub_relation& sr = rels[kv.second.rel_pos];
        sr.sub_ids_off = static_cast<uint32_t>(sub_ids.size()); sr.sub_ids_cnt = static_cast<uint32_t>(kv.second.ids.size());
        sub_ids.insert(sub_ids.end(), kv.second.ids.begin(), kv.second.ids.end());
    }
    return GM_OK;
}

// the group header, member pool and online bitmap: what changed since the last choosing call (a table that grows keeps its
// contents: only the dirty range is shipped)
int32_t GpuRouter::ship_groups(cudaStream_t s) {
    auto ship = [&](DevBuf& d, const void* host, size_t elem, size_t count, Dirty& dirty) -> int32_t {
        CUDA_TRY(d.ensure(std::max<size_t>(count, 256) * elem, true, s));
        if (dirty.any()) {
            const size_t lo = dirty.lo, hi = std::min<size_t>(dirty.hi, count);
            if (hi > lo) CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(d.p) + lo * elem, static_cast<const char*>(host) + lo * elem, (hi - lo) * elem, cudaMemcpyHostToDevice, s));
            dirty = Dirty{};
        }
        return GM_OK;
    };
    GM_TRY(ship(d_ghdr_, grp_hdr_.data(), sizeof(gm_span), grp_hdr_.size(), hdr_dirty_));
    GM_TRY(ship(d_gmem_, member_pool_.data(), 4, member_pool_.size(), pool_dirty_));
    GM_TRY(ship(d_online_, online_words_.data(), 4, online_words_.size(), online_dirty_));
    return GM_OK;
}

// Router::matches for a batch.  Everything per relation happens on the device (engine match, then k_relations writes the
// finished gm_sub_relation records); the records are copied straight into the caller's arrays.  Returns GM_ERR_CAPACITY with
// *needed_* set when an output is too small.
int32_t GpuRouter::matches_batch(const gm_id* publishers, const char* blob, const uint32_t* offs, uint64_t n, gm_span* out_spans,
                                 gm_sub_relation* out_rels, uint64_t cap_rels, uint32_t* out_sub_ids, uint64_t cap_sub_ids,
                                 uint64_t* needed_rels, uint64_t* needed_sub_ids, int32_t* status, const uint64_t* share_seed) {
    if (needed_rels) *needed_rels = 0;
    if (needed_sub_ids) *needed_sub_ids = 0;
    if (n == 0) return GM_OK;
    using Clk = std::chrono::steady_clock;
    const auto t0 = Clk::now();
    if (!stream_) CUDA_TRY(cudaStreamCreateWithFlags(stream_.put(), cudaStreamNonBlocking));
    const cudaStream_t s = stream_;
    if (share_seed) {
        // a group's representative must be in the device trie, also on an engine that only flushes when told to
        if (groups_changed_) { GM_TRY(gm_flush(e_)); groups_changed_ = false; unflushed_removes_ = false; }
        GM_TRY(ship_groups(s));
    }
    // ---- the relation table: ship what changed since the last call
    if (rel_dirty_hi_ > rel_dirty_lo_) {
        CUDA_TRY(d_rels_.ensure(std::max<size_t>(rel_host_.size(), 1024) * sizeof(gm_rel), true, s));
        CUDA_TRY(cudaMemcpyAsync(static_cast<gm_rel*>(d_rels_.p) + rel_dirty_lo_, rel_host_.data() + rel_dirty_lo_, (rel_dirty_hi_ - rel_dirty_lo_) * sizeof(gm_rel), cudaMemcpyHostToDevice, s));
        rel_dirty_lo_ = 0xFFFFFFFFu; rel_dirty_hi_ = 0;
    }
    // ---- topics and publishers to the device, match (ids = relation handles stay in HBM)
    const uint64_t blob_bytes = offs[n];
    CUDA_TRY(d_blob_.ensure(blob_bytes + 16)); CUDA_TRY(d_offs_.ensure((n + 1) * 4)); CUDA_TRY(d_spans_.ensure(n * 8)); CUDA_TRY(d_status_.ensure(n * 4));
    CUDA_TRY(d_needed_.ensure(4 * 8)); CUDA_TRY(d_ospans_.ensure(n * 8));
    if (blob_bytes) CUDA_TRY(cudaMemcpyAsync(d_blob_.p, blob, blob_bytes, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(d_offs_.p, offs, (n + 1) * 4, cudaMemcpyHostToDevice, s));
    if (publishers) {
        pubs_.resize(n);
        for (uint64_t i = 0; i < n; ++i) {
            auto it = id_idx_.find(ikey(publishers[i].node_id, publishers[i].client_id ? std::string(publishers[i].client_id, publishers[i].client_len) : std::string(), publishers[i].tag));
            pubs_[i] = it == id_idx_.end() ? 0xFFFFFFFFu : it->second;       // an Id no subscriber holds cannot equal any relation's Id
        }
        CUDA_TRY(d_pubs_.ensure(n * 4));
        CUDA_TRY(cudaMemcpyAsync(d_pubs_.p, pubs_.data(), n * 4, cudaMemcpyHostToDevice, s));
    }
    if (d_ids_.cap < 4096) CUDA_TRY(d_ids_.ensure(std::max<size_t>(4096, 32 * n) * 4));
    uint64_t need[4] = {0, 0, 0, 0};
    for (;;) {
        gm_match_args a{};
        a.struct_size = sizeof(a); a.d_blob = d_blob_.p; a.blob_bytes = blob_bytes; a.d_offsets = static_cast<const uint32_t*>(d_offs_.p); a.n_entries = n; a.n = n;
        a.d_spans = static_cast<gm_span*>(d_spans_.p); a.d_out = d_ids_.p; a.cap = d_ids_.cap / 4; a.d_needed = static_cast<uint64_t*>(d_needed_.p) + 3;
        a.d_status = static_cast<int32_t*>(d_status_.p); a.stream = s;
        GM_TRY(gm_match_batch_device_ex(e_, &a));
        CUDA_TRY(cudaMemcpyAsync(&need[3], static_cast<uint64_t*>(d_needed_.p) + 3, 8, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        if (need[3] > 0xFFFFFFFFull) return GM_ERR_TOO_LARGE;
        if (need[3] * 4 <= d_ids_.cap) break;
        CUDA_TRY(d_ids_.ensure((need[3] + 1024) * 4));
    }
    // ---- relation expansion on the device: at most one record and one sub id per matched id
    CUDA_TRY(d_orels_.ensure(std::max<uint64_t>(need[3], 1) * sizeof(gm_sub_relation)));
    CUDA_TRY(d_subs_.ensure(std::max<uint64_t>(need[3], 1) * 4));
    gm_rel_out o{};
    o.d_spans = static_cast<gm_span*>(d_ospans_.p); o.d_rels = static_cast<gm_sub_relation*>(d_orels_.p); o.cap_rels = d_orels_.cap / sizeof(gm_sub_relation);
    o.d_sub_ids = static_cast<uint32_t*>(d_subs_.p); o.cap_sub_ids = d_subs_.cap / 4;
    o.d_needed = static_cast<uint64_t*>(d_needed_.p); o.d_status = static_cast<int32_t*>(d_status_.p);
    if (share_seed) {
        gm_rel_groups gr{};
        gr.d_groups = static_cast<const gm_span*>(d_ghdr_.p); gr.n_groups = static_cast<uint32_t>(grp_hdr_.size()); gr.d_members = static_cast<const uint32_t*>(d_gmem_.p);
        gr.d_online = static_cast<const uint32_t*>(d_online_.p); gr.n_online_bits = static_cast<uint32_t>(client_key_.size()); gr.seed = *share_seed;
        GM_TRY(gm_relations_choose_device(e_, static_cast<const gm_span*>(d_spans_.p), static_cast<const uint32_t*>(d_ids_.p), n, publishers ? static_cast<const uint32_t*>(d_pubs_.p) : nullptr,
                                         static_cast<const gm_rel*>(d_rels_.p), rel_host_.size(), &gr, &o, s));
    } else
        GM_TRY(gm_relations_expand_device(e_, static_cast<const gm_span*>(d_spans_.p), static_cast<const uint32_t*>(d_ids_.p), n, publishers ? static_cast<const uint32_t*>(d_pubs_.p) : nullptr,
                                         static_cast<const gm_rel*>(d_rels_.p), rel_host_.size(), &o, s));
    CUDA_TRY(cudaMemcpyAsync(need, d_needed_.p, 2 * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(status, d_status_.p, n * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(out_spans, d_ospans_.p, n * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    bool flagged = false;
    for (uint64_t i = 0; i < n && !flagged; ++i) flagged = status[i] == 1;
    if (!flagged) {      // the common case: the device's records ARE the result
        if (needed_rels) *needed_rels = need[0];
        if (needed_sub_ids) *needed_sub_ids = need[1];
        if (need[0] > cap_rels || need[1] > cap_sub_ids) return GM_ERR_CAPACITY;
        if (need[0]) CUDA_TRY(cudaMemcpyAsync(out_rels, d_orels_.p, need[0] * sizeof(gm_sub_relation), cudaMemcpyDeviceToHost, s));
        if (need[1]) CUDA_TRY(cudaMemcpyAsync(out_sub_ids, d_subs_.p, need[1] * 4, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        last_device_ms = std::chrono::duration<double, std::milli>(Clk::now() - t0).count();
        last_host_ms = 0;
        return GM_OK;
    }
    // ---- some topic had more v5 relations than the kernel stages: finish those on the host and re-assemble
    const auto t1 = Clk::now();
    std::vector<gm_sub_relation> dev(need[0]), rels;
    std::vector<uint32_t> dsub(need[1]), sub_ids;
    if (need[0]) CUDA_TRY(cudaMemcpyAsync(dev.data(), d_orels_.p, need[0] * sizeof(gm_sub_relation), cudaMemcpyDeviceToHost, s));
    if (need[1]) CUDA_TRY(cudaMemcpyAsync(dsub.data(), d_subs_.p, need[1] * 4, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    rels.reserve(need[0]);
    for (uint64_t i = 0; i < n; ++i) {
        const size_t begin = rels.size();
        const uint32_t off = out_spans[i].off, cnt = out_spans[i].cnt;
        if (status[i] == 1) { status[i] = 0; GM_TRY(host_dedup_topic(dev.data() + off, cnt, share_seed != nullptr, rels, sub_ids)); }
        else if (status[i] == 0)
            for (uint32_t k = 0; k < cnt; ++k) {
                gm_sub_relation sr = dev[off + k];
                if (sr.sub_ids_cnt) { const uint32_t so = static_cast<uint32_t>(sub_ids.size()); sub_ids.insert(sub_ids.end(), dsub.begin() + sr.sub_ids_off, dsub.begin() + sr.sub_ids_off + sr.sub_ids_cnt); sr.sub_ids_off = so; }
                rels.push_back(sr);
            }
        out_spans[i] = gm_span{static_cast<uint32_t>(begin), static_cast<uint32_t>(rels.size() - begin)};
    }
    if (needed_rels) *needed_rels = rels.size();
    if (needed_sub_ids) *needed_sub_ids = sub_ids.size();
    if (rels.size() > cap_rels || sub_ids.size() > cap_sub_ids) return GM_ERR_CAPACITY;
    std::copy(rels.begin(), rels.end(), out_rels);
    std::copy(sub_ids.begin(), sub_ids.end(), out_sub_ids);
    last_device_ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    last_host_ms = std::chrono::duration<double, std::milli>(Clk::now() - t1).count();
    return GM_OK;
}

}  // namespace gm
