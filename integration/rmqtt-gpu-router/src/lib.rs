//! `rmqtt-gpu-router`: an rmqtt plugin that keeps the broker's `Router` and `RetainStorage` traits and forwards the hot calls
//! (`Router::matches`, `RetainStorage::get`) to libgpumqtt.  UNTESTED SOURCE — written against rmqtt 4f9f2185 without a
//! compiler (no cargo in the image that builds libgpumqtt.so; see ../README.md).  The C++ twin of `GpuRouter`
//! (`rmqtt_b200/csrc/router_host.cpp`, `gmr_*`) is what the repository's tests exercise; this file shows the same state and
//! rules on the Rust side of the boundary.
//!
//! Shape follows the reference's own plugins:
//!   plugin  : rmqtt-plugins/rmqtt-retainer/src/lib.rs:35-160 (`#[derive(Plugin)]`, `register!`, config, `start()` swaps the trait object)
//!   router  : rmqtt-plugins/rmqtt-cluster-broadcast/src/router.rs:21-170 (wrap `DefaultRouter`, forward the cold calls)
//!   retainer: rmqtt-plugins/rmqtt-retainer/src/ram.rs:18-93
#![deny(unsafe_code)] // all `unsafe` lives in `engine` below, a private module with a safe surface
use std::sync::atomic::{AtomicU32, Ordering};
use std::sync::Arc;
use std::time::Duration;

use async_trait::async_trait;
use dashmap::DashMap;
use itertools::Itertools;
use rmqtt::{
    context::ServerContext,
    utils::timestamp_millis,   // ms since the Unix epoch (rmqtt-utils/src/lib.rs:504): the unit of the engine's deadlines
    macros::Plugin,
    plugin::{PackageInfo, Plugin},
    register,
    retain::RetainStorage,
    router::{DefaultRouter, Router},
    types::*,
    Result,
};
use serde::{Deserialize, Serialize};
use tokio::sync::oneshot;

mod engine {
    //! Safe surface over gpumqtt-sys: the engine handle, the library's own micro-batcher, the retained lookup.
    #![allow(unsafe_code)]
    use gpumqtt_sys as sys;
    use std::ffi::{c_void, CStr};
    use tokio::sync::oneshot;

    pub type MatchReply = std::result::Result<Vec<u32>, i32>; // ids, or the per-topic status (GM_ERR_INVALID_TOPIC = Topic::from_str Err)

    pub struct Engine(pub(super) *mut sys::gm_engine);
    unsafe impl Send for Engine {} // libgpumqtt handles are thread-safe (include/gpumqtt.h)
    unsafe impl Sync for Engine {}

    impl Engine {
        pub fn new(device: i32, filters_hint: u64) -> anyhow::Result<Self> {
            let cfg = sys::gm_config { struct_size: std::mem::size_of::<sys::gm_config>() as u32, device, max_levels: 0, flags: 0, filters_hint };
            let mut h = std::ptr::null_mut();
            let rc = unsafe { sys::gm_create(&cfg, &mut h) };
            if rc != sys::GM_OK {
                anyhow::bail!("gm_create: {rc} (no CUDA device means no router: libgpumqtt has no CPU fallback)")
            }
            Ok(Self(h))
        }
        fn err(&self, what: &str, rc: i32) -> anyhow::Error {
            let msg = unsafe { CStr::from_ptr(sys::gm_last_error(self.0)) }.to_string_lossy().into_owned();
            anyhow::anyhow!("{what}: {rc} {msg}")
        }
        pub fn sub_add(&self, filter: &str, value: u32) -> anyhow::Result<bool> {
            let mut ch = 0;
            let rc = unsafe { sys::gm_sub_add(self.0, filter.as_ptr(), filter.len() as u32, value, &mut ch) };
            if rc != sys::GM_OK { return Err(self.err("gm_sub_add", rc)) }
            Ok(ch != 0)
        }
        pub fn sub_remove(&self, filter: &str, value: u32) -> anyhow::Result<bool> {
            let mut ch = 0;
            let rc = unsafe { sys::gm_sub_remove(self.0, filter.as_ptr(), filter.len() as u32, value, &mut ch) };
            if rc != sys::GM_OK { return Err(self.err("gm_sub_remove", rc)) }
            Ok(ch != 0)
        }
        /// Raft restore / snapshot load (rmqtt-cluster-raft/src/router.rs:557-561): every filter in one call, all host threads.
        pub fn bulk_load(&self, filters: &[(&str, u32)]) -> anyhow::Result<u64> {
            let (mut blob, mut offs, mut vals) = (Vec::new(), vec![0u32], Vec::with_capacity(filters.len()));
            for (f, v) in filters { blob.extend_from_slice(f.as_bytes()); offs.push(blob.len() as u32); vals.push(*v); }
            let mut changed = 0u64;
            let rc = unsafe { sys::gm_bulk_load(self.0, blob.as_ptr(), offs.as_ptr(), vals.as_ptr(), vals.len() as u64, &mut changed) };
            if rc != sys::GM_OK { return Err(self.err("gm_bulk_load", rc)) }
            Ok(changed)
        }
        pub fn values_size(&self) -> anyhow::Result<usize> {
            let mut st = sys::gm_stats::default();
            let rc = unsafe { sys::gm_get_stats(self.0, &mut st) };
            if rc != sys::GM_OK { return Err(self.err("gm_get_stats", rc)) }
            Ok(st.values as usize)
        }
        pub fn retain_set(&self, topic: &str, value: u32) -> anyhow::Result<Option<u32>> {
            let (mut had, mut old) = (0, 0);
            let rc = unsafe { sys::gm_retain_set(self.0, topic.as_ptr(), topic.len() as u32, value, &mut had, &mut old) };
            if rc != sys::GM_OK { return Err(self.err("gm_retain_set", rc)) }
            Ok((had != 0).then_some(old))
        }
        pub fn retain_remove(&self, topic: &str) -> anyhow::Result<Option<u32>> {
            let (mut had, mut old) = (0, 0);
            let rc = unsafe { sys::gm_retain_remove(self.0, topic.as_ptr(), topic.len() as u32, &mut had, &mut old) };
            if rc != sys::GM_OK { return Err(self.err("gm_retain_remove", rc)) }
            Ok((had != 0).then_some(old))
        }
        /// set_with_timeout: `deadline_ms` in ms since the Unix epoch (0 = none); the lookups drop the handle from then on.
        pub fn retain_set_ttl(&self, topic: &str, value: u32, deadline_ms: u64) -> anyhow::Result<Option<u32>> {
            let (mut had, mut old) = (0, 0);
            let rc = unsafe { sys::gm_retain_set_ttl(self.0, topic.as_ptr(), topic.len() as u32, value, deadline_ms, &mut had, &mut old) };
            if rc != sys::GM_OK { return Err(self.err("gm_retain_set_ttl", rc)) }
            Ok((had != 0).then_some(old))
        }
        /// remove_expired_messages (retain.rs:118-128): up to `cap` expired topics per call; their handles come back.
        pub fn retain_remove_expired(&self, now_ms: u64, cap: usize) -> anyhow::Result<Vec<u32>> {
            let mut out = vec![0u32; cap];
            let mut n = 0u64;
            let rc = unsafe { sys::gm_retain_remove_expired(self.0, now_ms, out.as_mut_ptr(), cap as u64, &mut n) };
            if rc != sys::GM_OK { return Err(self.err("gm_retain_remove_expired", rc)) }
            out.truncate(n as usize);
            Ok(out)
        }
        /// Removal of a list of topics as ONE call (RetainTree::retain, retain.rs:261-288).
        pub fn retain_remove_batch(&self, topics: &[&str]) -> anyhow::Result<u64> {
            let (mut blob, mut offs) = (Vec::new(), vec![0u32]);
            for t in topics { blob.extend_from_slice(t.as_bytes()); offs.push(blob.len() as u32); }
            let mut removed = 0u64;
            let rc = unsafe { sys::gm_retain_remove_batch(self.0, blob.as_ptr(), offs.as_ptr(), topics.len() as u64, std::ptr::null_mut(), &mut removed) };
            if rc != sys::GM_OK { return Err(self.err("gm_retain_remove_batch", rc)) }
            Ok(removed)
        }
        /// RetainStorage::get for a batch of SUBSCRIBE filters (a SUBSCRIBE packet carries several): blocking, call it from
        /// `spawn_blocking`.  Per filter the handles of the retained messages it matches, or Err for an invalid filter.
        pub fn retain_match(&self, filters: &[&str]) -> anyhow::Result<Vec<MatchReply>> {
            let n = filters.len();
            let (mut blob, mut offs) = (Vec::new(), vec![0u32]);
            for f in filters { blob.extend_from_slice(f.as_bytes()); offs.push(blob.len() as u32); }
            let mut spans = vec![sys::gm_span::default(); n];
            let mut status = vec![0i32; n];
            let mut cap = (n * 64).max(1024);
            loop {
                let mut ids = vec![0u32; cap];
                let mut needed = 0u64;
                let rc = unsafe {
                    sys::gm_retain_match_batch(self.0, blob.as_ptr(), offs.as_ptr(), n as u64, spans.as_mut_ptr(), ids.as_mut_ptr(), cap as u64, &mut needed, status.as_mut_ptr())
                };
                if rc == sys::GM_ERR_CAPACITY { cap = needed as usize; continue }
                if rc != sys::GM_OK { return Err(self.err("gm_retain_match_batch", rc)) }
                return Ok((0..n).map(|i| if status[i] != 0 { Err(status[i]) } else { Ok(ids[spans[i].off as usize..(spans[i].off + spans[i].cnt) as usize].to_vec()) }).collect());
            }
        }
        /// The unique matched FILTERS of a topic (descriptor mode; what `get` / `_has_matches` / `query_subscriptions` need).
        pub fn matched_handles_one_per_filter(&self, topic: &str) -> anyhow::Result<Vec<u32>> {
            let offs = [0u32, topic.len() as u32];
            let (mut span, mut status, mut needed) = (sys::gm_span::default(), 0i32, 0u64);
            let mut descs = vec![sys::gm_desc::default(); 64];
            loop {
                let rc = unsafe { sys::gm_match_batch_desc(self.0, topic.as_ptr(), offs.as_ptr(), 1, &mut span, descs.as_mut_ptr(), descs.len() as u64, &mut needed, &mut status) };
                if rc == sys::GM_ERR_CAPACITY { descs.resize(needed as usize, sys::gm_desc::default()); continue }
                if rc != sys::GM_OK { return Err(self.err("gm_match_batch_desc", rc)) }
                break;
            }
            if status != 0 { anyhow::bail!("invalid topic") }
            let mut view = sys::gm_values { values: std::ptr::null(), n_values: 0, ranges: std::ptr::null(), n_ranges: 0, epoch: 0 };
            let rc = unsafe { sys::gm_values_view(self.0, &mut view) };
            if rc != sys::GM_OK { return Err(self.err("gm_values_view", rc)) }
            // any member of a matched value set names the filter (all members of one set share it)
            Ok(descs[span.off as usize..(span.off + span.cnt) as usize].iter().map(|d| unsafe {
                if d.cnt == 1 { d.r#ref } else if d.cnt == 0xFFFF { *view.values.add((*view.ranges.add(d.r#ref as usize)).off as usize) } else { *view.values.add(d.r#ref as usize) }
            }).collect())
        }
    }
    impl Drop for Engine {
        fn drop(&mut self) { unsafe { sys::gm_destroy(self.0) } }
    }

    /// The library's MPSC micro-batcher (`gm_batcher_*`, rmqtt_b200/csrc/batcher.cpp): one `submit` per PUBLISH from any tokio
    /// worker, device batches behind it (<= 2048 topics = one CUDA-graph launch), one callback per topic on a dispatcher thread.
    pub struct Batcher { raw: *mut sys::gm_batcher, _engine: std::sync::Arc<Engine> }
    unsafe impl Send for Batcher {}
    unsafe impl Sync for Batcher {}

    extern "C" fn on_match(_user: *mut c_void, cookie: u64, status: i32, ids: *const u32, n_ids: u32) {
        // the cookie is the leaked Sender of the oneshot `submit` is waiting on; `ids` is valid during this call only
        let tx = unsafe { Box::from_raw(cookie as *mut oneshot::Sender<MatchReply>) };
        let reply = if status == sys::GM_OK { Ok(unsafe { std::slice::from_raw_parts(ids, n_ids as usize) }.to_vec()) } else { Err(status) };
        let _ = tx.send(reply);
    }

    impl Batcher {
        pub fn new(engine: std::sync::Arc<Engine>, max_batch: u32, max_wait_us: u32, dispatchers: u32) -> anyhow::Result<Self> {
            Self::create(engine, max_batch, max_wait_us, dispatchers, false)
        }
        /// The retained batcher (`gm_retain_batcher_create`): one `submit` per SUBSCRIBE filter, the reply holds the handles of
        /// the retained messages it matches.
        pub fn retained(engine: std::sync::Arc<Engine>, max_batch: u32, max_wait_us: u32, dispatchers: u32) -> anyhow::Result<Self> {
            Self::create(engine, max_batch, max_wait_us, dispatchers, true)
        }
        fn create(engine: std::sync::Arc<Engine>, max_batch: u32, max_wait_us: u32, dispatchers: u32, retained: bool) -> anyhow::Result<Self> {
            let cfg = sys::gm_batcher_config {
                struct_size: std::mem::size_of::<sys::gm_batcher_config>() as u32, max_batch, max_wait_us, dispatchers, on_match, user: std::ptr::null_mut(),
            };
            let mut raw = std::ptr::null_mut();
            let rc = unsafe { if retained { sys::gm_retain_batcher_create(engine.0, &cfg, &mut raw) } else { sys::gm_batcher_create(engine.0, &cfg, &mut raw) } };
            if rc != sys::GM_OK { return Err(engine.err(if retained { "gm_retain_batcher_create" } else { "gm_batcher_create" }, rc)) }
            Ok(Self { raw, _engine: engine })
        }
        /// Never waits for the device; the reply arrives on the returned channel.
        pub fn submit(&self, topic: &str) -> anyhow::Result<oneshot::Receiver<MatchReply>> {
            let (tx, rx) = oneshot::channel();
            let cookie = Box::into_raw(Box::new(tx)) as u64;
            let rc = unsafe { sys::gm_submit(self.raw, topic.as_ptr(), topic.len() as u32, cookie) };
            if rc != sys::GM_OK {
                drop(unsafe { Box::from_raw(cookie as *mut oneshot::Sender<MatchReply>) }); // not queued: take the Sender back
                anyhow::bail!("gm_submit: {rc}")
            }
            Ok(rx)
        }
    }
    impl Drop for Batcher {
        fn drop(&mut self) { unsafe { sys::gm_batcher_destroy(self.raw) } } // drains: every pending callback runs first
    }
}
use engine::{Batcher, Engine};

// ---- plugin ---------------------------------------------------------------------------------------------------------
#[derive(Debug, Clone, Deserialize, Serialize)]
pub struct PluginConfig {
    #[serde(default)]
    pub device: i32, // CUDA device ordinal
    #[serde(default = "PluginConfig::max_batch_default")]
    pub max_batch: u32, // dispatch when this many PUBLISH topics are queued ...
    #[serde(default = "PluginConfig::max_wait_us_default")]
    pub max_wait_us: u32, // ... or when the oldest has waited this long
    #[serde(default = "PluginConfig::dispatchers_default")]
    pub dispatchers: u32, // batches in flight
    #[serde(default)]
    pub filters_hint: u64, // expected subscriptions (pre-sizes the tables)
    #[serde(default = "PluginConfig::retain_default")]
    pub retain: bool, // also replace the retainer
}
impl PluginConfig {
    fn max_batch_default() -> u32 { 4096 }
    fn max_wait_us_default() -> u32 { 50 }
    fn dispatchers_default() -> u32 { 2 }
    fn retain_default() -> bool { true }
    fn to_json(&self) -> Result<serde_json::Value> { Ok(serde_json::to_value(self)?) }
}

register!(GpuRouterPlugin::new); // rmqtt/src/plugin.rs:75-106

#[derive(Plugin)]
struct GpuRouterPlugin {
    scx: ServerContext,
    cfg: PluginConfig,
    engine: Arc<Engine>,
    router: GpuRouter,
    retainer: Option<GpuRetainer>,
}

impl GpuRouterPlugin {
    async fn new<N: Into<String>>(scx: ServerContext, name: N) -> Result<Self> {
        let name = name.into();
        let cfg = scx.plugins.read_config_default::<PluginConfig>(&name)?;
        log::info!("{name} GpuRouterPlugin cfg: {cfg:?}");
        let engine = Arc::new(Engine::new(cfg.device, cfg.filters_hint)?);
        let router = GpuRouter::new(scx.clone(), engine.clone(), &cfg)?;
        let retainer = if cfg.retain { Some(GpuRetainer::new(engine.clone())?) } else { None };
        Ok(Self { scx, cfg, engine, router, retainer })
    }
}

#[async_trait]
impl Plugin for GpuRouterPlugin {
    async fn init(&mut self) -> Result<()> {
        if let Some(r) = self.retainer.clone() {
            tokio::spawn(async move {
                loop {
                    tokio::time::sleep(Duration::from_secs(10)).await; // rmqtt-retainer/src/lib.rs:112-124
                    let _ = r.remove_expired_messages().await;
                }
            });
        }
        Ok(())
    }
    async fn get_config(&self) -> Result<serde_json::Value> { self.cfg.to_json() }
    async fn start(&mut self) -> Result<()> {
        log::info!("{} start, {}", self.name(), self.engine.values_size()?);
        *self.scx.extends.router_mut().await = Box::new(self.router.clone()); // rmqtt/src/extend.rs:133-137
        if let Some(r) = self.retainer.clone() {
            *self.scx.extends.retain_mut().await = Box::new(r); // rmqtt-retainer/src/lib.rs:151
        }
        Ok(())
    }
    async fn stop(&mut self) -> Result<bool> {
        log::warn!("{} stop: the router cannot be swapped back while sessions hold subscriptions", self.name());
        Ok(false)
    }
}

// ---- router ---------------------------------------------------------------------------------------------------------
/// value handle <-> (filter, client): one u32 per subscription relation (`relations[filter][client]` in the reference).
#[derive(Default)]
struct Handles {
    by_key: DashMap<(TopicFilter, ClientId), u32>,
    by_id: DashMap<u32, (TopicFilter, ClientId)>,
    next: AtomicU32,
}

/// `inner` contributes `relations`, the two counters and the cold admin queries; its `topics` tree stays EMPTY — the trie
/// lives in libgpumqtt (host mirror + HBM), which serves `matches`, `get` and `topics_tree`.  One copy of the subscription set.
#[derive(Clone)]
pub struct GpuRouter {
    inner: DefaultRouter,
    engine: Arc<Engine>,
    handles: Arc<Handles>,
    batcher: Arc<Batcher>,
}

impl GpuRouter {
    fn new(scx: ServerContext, engine: Arc<Engine>, cfg: &PluginConfig) -> Result<Self> {
        let batcher = Arc::new(Batcher::new(engine.clone(), cfg.max_batch, cfg.max_wait_us, cfg.dispatchers)?);
        Ok(Self { inner: DefaultRouter::new(Some(scx)), engine, handles: Arc::new(Handles::default()), batcher })
    }
    fn scx(&self) -> &ServerContext { self.inner.context() }
}

#[async_trait]
impl Router for GpuRouter {
    /// router.rs:417-436 without the CPU trie: the filter is validated by the engine (`GM_ERR_INVALID_TOPIC` = `Topic::from_str` Err)
    async fn add(&self, topic_filter: &str, id: Id, opts: SubscriptionOptions) -> Result<()> {
        let key = (TopicFilter::from(topic_filter), id.client_id.clone());
        let h = *self.handles.by_key.entry(key.clone()).or_insert_with(|| {
            let h = self.handles.next.fetch_add(1, Ordering::Relaxed);
            self.handles.by_id.insert(h, key);
            h
        });
        self.engine.sub_add(topic_filter, h)?; // Err before any state changes, like `Topic::from_str(topic_filter)?`
        let old = self
            .inner
            .relations
            .entry(TopicFilter::from(topic_filter))
            .or_insert_with(|| { self.inner.topics_count.inc(); HashMap::default() })
            .insert(id.client_id.clone(), (id, opts));
        if old.is_none() { self.inner.relations_count.inc(); }
        Ok(())
    }

    /// router.rs:439-479: the Id-equality rule and the counters, then the relation's handle leaves the device trie
    async fn remove(&self, topic_filter: &str, id: Id) -> Result<bool> {
        let res = if let Some(mut rels) = self.inner.relations.get_mut(topic_filter) {
            let enable = rels.value().get(&id.client_id).map(|(s_id, _)| *s_id == id).unwrap_or(false);
            if enable {
                let ok = rels.value_mut().remove(&id.client_id).is_some();
                if ok { self.inner.relations_count.dec(); }
                Some((rels.is_empty(), ok))
            } else { None }
        } else { None };
        let Some((is_empty, ok)) = res else { return Ok(false) };
        if is_empty && self.inner.relations.remove(topic_filter).is_some() { self.inner.topics_count.dec(); }
        if ok {
            if let Some((_, h)) = self.handles.by_key.remove(&(TopicFilter::from(topic_filter), id.client_id.clone())) {
                self.handles.by_id.remove(&h);
                self.engine.sub_remove(topic_filter, h)?;
            }
        }
        Ok(ok)
    }

    /// router.rs:162-248 fed from the engine's handles instead of the trie iterator.
    async fn matches(&self, this_id: Id, topic: &TopicName) -> Result<SubRelationsMap> {
        let handles = match self.batcher.submit(topic)?.await? {
            Ok(h) => h,
            Err(status) => return Err(anyhow::anyhow!("invalid topic ({status})")), // router.rs:165; shared.rs:615-621 logs it and forwards nothing
        };
        let mut collector_map: SubscriptioRelationsCollectorMap = HashMap::default();
        #[allow(clippy::type_complexity)]
        let mut groups: HashMap<(TopicFilter, SharedGroup), Vec<(NodeId, ClientId, SubscriptionOptions, Option<Vec<SubscriptionIdentifier>>, Option<IsOnline>)>> =
            HashMap::default();
        for h in handles {
            let Some(kv) = self.handles.by_id.get(&h) else { continue }; // removed since the batch was flushed
            let (topic_filter, client_id) = kv.value();
            let Some(rels) = self.inner.relations.get(topic_filter) else { continue };
            let Some((id, opts)) = rels.get(client_id) else { continue };
            if let Some(true) = opts.no_local() { if &this_id == id { continue } } // router.rs:184-189
            if let Some(group) = opts.shared_group() {
                // router.rs:192-200: members are bucketed per (filter, group) ...
                let online = self.scx().extends.router().await.is_online(id.node_id, client_id).await;
                groups.entry((topic_filter.clone(), group.clone())).or_default().push((id.node_id, client_id.clone(), opts.clone(), None, Some(online)));
            } else {
                collector_map.entry(id.node_id).or_default().add(topic_filter, client_id.clone(), opts.clone(), None);
            }
        }
        // ... and ONE member per group is chosen by the broker's strategy (router.rs:224-238; random in the default)
        for ((topic_filter, group), mut s_subs) in groups.drain() {
            let group_cids = s_subs.iter().map(|(_, cid, _, _, _)| cid.clone()).collect();
            if let Some((idx, is_online)) = self.scx().extends.shared_subscription().await.choice(self.scx(), &s_subs).await {
                let (node_id, client_id, opts, _, _) = s_subs.remove(idx);
                collector_map.entry(node_id).or_default().add(&topic_filter, client_id, opts, Some((group, is_online, group_cids)));
            }
        }
        Ok(collector_map.into_iter().map(|(n, c)| (n, c.into())).collect())
    }

    /// router.rs:522-546: the unique matched filters come from the engine (descriptor mode), the node ids from `relations`
    async fn get(&self, topic: &str) -> Result<Vec<Route>> {
        let (engine, topic) = (self.engine.clone(), topic.to_string());
        let hs = tokio::task::spawn_blocking(move || engine.matched_handles_one_per_filter(&topic)).await??;
        let mut routes = Vec::new();
        for tf in hs.into_iter().filter_map(|h| self.handles.by_id.get(&h).map(|kv| kv.value().0.clone())).unique() {
            if let Some(entry) = self.inner.relations.get(&tf) {
                routes.extend(entry.iter().map(|(_, (id, _))| id.node_id).unique().map(|node_id| Route { node_id, topic: tf.clone() }));
            }
        }
        Ok(routes)
    }

    async fn topics_tree(&self) -> usize { self.engine.values_size().unwrap_or(0) } // TopicTree::values_size (trie.rs:148-151)
    async fn is_online(&self, node_id: NodeId, client_id: &str) -> bool { self.inner.is_online(node_id, client_id).await }
    async fn gets(&self, limit: usize) -> Vec<Route> { self.inner.gets(limit).await } // relations only
    // `_match_topic` queries (router.rs:315-363) would read the empty CPU trie: route them through `get`'s matched filters;
    // every other query shape reads `relations` only (router.rs:366-414)
    async fn query_subscriptions(&self, q: &SubsSearchParams) -> Vec<SubsSearchResult> { self.inner.query_subscriptions(q).await }
    fn topics(&self) -> Counter { self.inner.topics() }
    fn routes(&self) -> Counter { self.inner.routes() }
    fn merge_topics(&self, m: &HashMap<NodeId, Counter>) -> Counter { self.inner.merge_topics(m) }
    fn merge_routes(&self, m: &HashMap<NodeId, Counter>) -> Counter { self.inner.merge_routes(m) }
    async fn list_topics(&self, top: usize) -> Vec<String> { self.inner.relations.iter().take(top).map(|e| e.key().to_string()).collect() }
    async fn list_relations(&self, top: usize) -> Vec<serde_json::Value> { self.inner.list_relations(top).await }
    fn relations(&self) -> &AllRelationsMap { self.inner.relations() }
}

// ---- retainer -------------------------------------------------------------------------------------------------------
/// One slot per retained topic, indexed by the handle stored in the device tree: `get` never walks a CPU `RetainTree`.
/// The engine keeps the deadlines (gm_retain_set_ttl): its lookups return live handles only.
struct Slot { topic: TopicName, retain: Retain }

#[derive(Clone)]
pub struct GpuRetainer {
    engine: Arc<Engine>,
    batcher: Arc<Batcher>,
    slots: Arc<DashMap<u32, Slot>>,
    next: Arc<AtomicU32>,
}

impl GpuRetainer {
    /// A reconnect storm resubscribes many sessions at once: their lookups share device batches instead of queueing one by one.
    fn new(engine: Arc<Engine>) -> Result<Self> {
        let batcher = Arc::new(Batcher::retained(engine.clone(), 2048, 100, 2)?);
        Ok(Self { engine, batcher, slots: Arc::new(DashMap::default()), next: Arc::new(AtomicU32::new(0)) })
    }

    /// retain.rs:118-128 (`remove_expired_messages`): the engine's deadline queue yields the expired topics, a batch per call
    async fn remove_expired_messages(&self) -> usize {
        const CAP: usize = 65_536;
        let now = timestamp_millis() as u64;
        let mut n = 0;
        loop {
            let dead = self.engine.retain_remove_expired(now, CAP).unwrap_or_default();
            for h in &dead { self.slots.remove(h); }
            n += dead.len();
            if dead.len() < CAP { return n }
        }
    }
}

#[async_trait]
impl RetainStorage for GpuRetainer {
    fn enable(&self) -> bool { true }

    /// retain.rs:131-149: remove, then insert unless the payload is empty
    async fn set(&self, topic: &TopicName, retain: Retain, expiry_interval: Option<Duration>) -> Result<()> {
        if retain.publish.payload.is_empty() {
            if let Some(old) = self.engine.retain_remove(topic)? { self.slots.remove(&old); }
            return Ok(());
        }
        let h = self.next.fetch_add(1, Ordering::Relaxed);
        let deadline = expiry_interval.map(|d| timestamp_millis() as u64 + d.as_millis() as u64).unwrap_or(0);
        self.slots.insert(h, Slot { topic: topic.clone(), retain });
        if let Some(old) = self.engine.retain_set_ttl(topic, h, deadline)? { self.slots.remove(&old); } // Option::replace semantics
        Ok(())
    }

    /// retain.rs:152-169: the device already dropped the expired handles; the rest are cloned out
    async fn get(&self, topic_filter: &TopicFilter) -> Result<Vec<(TopicName, Retain)>> {
        let ids = self.batcher.submit(topic_filter.as_ref())?.await?.map_err(|st| anyhow::anyhow!("retained lookup failed ({st})"))?;
        Ok(ids.into_iter().filter_map(|h| self.slots.get(&h).map(|s| (s.topic.clone(), s.retain.clone()))).collect())
    }

    async fn count(&self) -> isize { self.slots.len() as isize }
    async fn max(&self) -> isize { self.slots.len() as isize }
}

// ---- message store --------------------------------------------------------------------------------------------------
/// rmqtt-message-storage's `MessageManager` with `get`'s forwarded checks and marks on the device (gm_msgstore_*).
/// The store owns the retained tree of its engine: it gets an engine of its own, with max_levels one above the listener's.
pub mod msgstore {
    #![allow(unsafe_code)]
    use super::engine::Engine;
    use dashmap::DashMap;
    use gpumqtt_sys as sys;
    use rmqtt::{timestamp_millis, From, MsgID, Publish, Result, SharedGroup, SubClientIds};
    use std::time::Duration;

    pub struct GpuMessageManager {
        engine: Engine,
        store: *mut sys::gm_msgstore,
        msgs: DashMap<MsgID, (From, Publish)>,               // payloads and senders stay on the host, by message id
        clients: DashMap<String, u32>,                       // ClientId -> client key
        shares: DashMap<(String, String), u32>,              // (topic filter, group) -> share key: equal pairs, equal keys
    }
    unsafe impl Send for GpuMessageManager {}
    unsafe impl Sync for GpuMessageManager {}               // gm_msgstore calls are serialised inside the library

    impl GpuMessageManager {
        pub fn new(engine: Engine) -> anyhow::Result<Self> {
            let mut store = std::ptr::null_mut();
            let rc = unsafe { sys::gm_msgstore_create(engine.0, std::ptr::null(), &mut store) };
            anyhow::ensure!(rc == sys::GM_OK, "gm_msgstore_create: {rc}");
            Ok(Self { engine, store, msgs: DashMap::default(), clients: DashMap::default(), shares: DashMap::default() })
        }
        fn client_key(&self, c: &str) -> u32 { let n = self.clients.len() as u32; *self.clients.entry(c.to_owned()).or_insert(n) }
        fn share_key(&self, f: &str, g: &str) -> u32 { let n = self.shares.len() as u32; *self.shares.entry((f.to_owned(), g.to_owned())).or_insert(n) }

        /// ram.rs:259-300 (`_set`): kept under topic/<msg_id> until now + expiry_interval, marked as forwarded to sub_client_ids
        pub fn store(&self, msg_id: MsgID, from: From, p: Publish, expiry_interval: Duration, sub_client_ids: SubClientIds) -> Result<()> {
            let at = timestamp_millis() as u64 + expiry_interval.as_millis() as u64;
            let (cl, sh): (Vec<u32>, Vec<u32>) = sub_client_ids.unwrap_or_default().iter()
                .map(|(c, s)| (self.client_key(c), s.as_ref().map(|(f, g)| self.share_key(f, g)).unwrap_or(sys::GM_MSGSTORE_NO_SHARE)))
                .unzip();
            let topic = p.topic.clone();
            self.msgs.insert(msg_id, (from, p));
            let rc = unsafe { sys::gm_msgstore_store(self.store, topic.as_ptr(), topic.len() as u32, msg_id as u32, at, cl.as_ptr(), sh.as_ptr(), cl.len() as u32) };
            if rc != sys::GM_OK { self.msgs.remove(&msg_id); anyhow::bail!("gm_msgstore_store: {rc}") }
            Ok(())
        }

        /// ram.rs:303-367 (`get`): the device drops what was forwarded or expired and marks what it returns
        pub fn get(&self, client_id: &str, topic_filter: &str, group: Option<&SharedGroup>) -> Result<Vec<(MsgID, From, Publish)>> {
            let cl = [self.client_key(client_id)];
            let sh = [group.map(|g| self.share_key(topic_filter, g)).unwrap_or(sys::GM_MSGSTORE_NO_SHARE)];
            let offs = [0u32, topic_filter.len() as u32];
            let (mut span, mut status, mut needed) = (sys::gm_span { off: 0, cnt: 0 }, 0i32, 0u64);
            let mut out = vec![0u32; 256];
            loop {
                let rc = unsafe { sys::gm_msgstore_get_batch(self.store, timestamp_millis() as u64, topic_filter.as_ptr(), offs.as_ptr(), 1, cl.as_ptr(),
                                                             sh.as_ptr(), &mut span, out.as_mut_ptr(), out.len() as u64, &mut needed, &mut status) };
                if rc == sys::GM_ERR_CAPACITY { out.resize(needed as usize, 0); continue }   // nothing was marked: ask again
                anyhow::ensure!(rc == sys::GM_OK, "gm_msgstore_get_batch: {rc}");
                anyhow::ensure!(status == sys::GM_OK, "invalid topic filter");
                break;
            }
            Ok(out[span.off as usize..(span.off + span.cnt) as usize].iter()
                .filter_map(|h| self.msgs.get(&(*h as MsgID)).map(|m| (*h as MsgID, m.0.clone(), m.1.clone()))).collect())
        }

        /// ram.rs:143-191: expiry_time_at <= now, earliest first; `evict` (cache_max_count / cache_capacity) takes the k earliest-expiring
        pub fn remove_expired_messages(&self, evict: Option<usize>) -> usize {
            const CAP: usize = 65_536;
            let (now, cap) = match evict { Some(k) => (u64::MAX - 1, k), None => (timestamp_millis() as u64, CAP) };
            let mut out = vec![0u32; cap.max(1)];
            let mut n = 0u64;
            if unsafe { sys::gm_msgstore_remove_expired(self.store, now, out.as_mut_ptr(), cap as u64, &mut n) } != sys::GM_OK { return 0 }
            for h in &out[..n as usize] { self.msgs.remove(&(*h as MsgID)); }
            n as usize
        }
    }

    impl Drop for GpuMessageManager {
        fn drop(&mut self) { unsafe { sys::gm_msgstore_destroy(self.store) } }
    }
}
