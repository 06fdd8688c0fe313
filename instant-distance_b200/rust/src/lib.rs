//! `instant_distance`-shaped API (Builder / Hnsw / HnswMap / Search / Point / PointId / Item / MapItem / Heuristic) for f32
//! vector points, executed by the H100 engine through the C ABI.  Mirrors instant-distance/src/lib.rs; method-level
//! citations below refer to that file.  NOT compiled in the build image (no Rust toolchain): kept in sync with the header.
use std::ffi::CStr;
use std::os::raw::c_char;

#[repr(C)]
#[derive(Clone, Copy)]
struct IdbParams {
    m: u32,
    ef_construction: u32,
    ef_search: u32,
    ml: f32,
    seed: u64,
    heuristic: i32,
    extend_candidates: i32,
    keep_pruned: i32,
    insert_batch: u32,
    device: i32,
    storage: u32,
    progress: Option<extern "C" fn(done: u64, total: u64, user: *mut std::ffi::c_void)>,
    progress_user: *mut std::ffi::c_void,
}
#[repr(C)]
struct IdbIndex {
    _private: [u8; 0],
}
extern "C" {
    fn idb_params_default(p: *mut IdbParams) -> i32;
    fn idb_build_f32(rows: *const f32, n: u64, dim: u32, p: *const IdbParams, out: *mut *mut IdbIndex, out_ids: *mut u32) -> i32;
    fn idb_build_ex(rows: *const f32, n: u64, dim: u32, p: *const IdbParams, metric: u32, out: *mut *mut IdbIndex, out_ids: *mut u32) -> i32;
    fn idb_index_from_graph_ex(points: *const f32, n: u64, dim: u32, m: u32, ef_search: u32, zero: *const u32, n_upper: u32,
                               upper: *const *const u32, upper_n: *const u64, storage: u32, metric: u32, device: i32,
                               out: *mut *mut IdbIndex) -> i32;
    fn idb_index_load_ex(path: *const c_char, dim: u32, m: u32, metric: u32, device: i32, out: *mut *mut IdbIndex, values_offset: *mut u64) -> i32;
    fn idb_index_load_storage(path: *const c_char, dim: u32, m: u32, metric: u32, storage: u32, device: i32, out: *mut *mut IdbIndex,
                              values_offset: *mut u64) -> i32;
    fn idb_normalize_f32(rows: *const f32, n: u64, dim: u32, device: i32, out: *mut f32) -> i32;
    fn idb_index_metric(ix: *const IdbIndex, out: *mut u32) -> i32;
    fn idb_search_batch_f32(ix: *mut IdbIndex, q: *const f32, nq: u64, ef: u32, k: u32, ids: *mut u32, dist: *mut f32, len: *mut u32) -> i32;
    fn idb_exact_search_batch_f32(ix: *mut IdbIndex, q: *const f32, nq: u64, k: u32, ids: *mut u32, dist: *mut f32, len: *mut u32) -> i32;
    fn idb_exact_search_batch_device_lane(ix: *mut IdbIndex, lane: u32, q: *const f32, nq: u64, k: u32, ids: *mut u32, dist: *mut f32, len: *mut u32) -> i32;
    fn idb_range_search_batch_f32(ix: *mut IdbIndex, q: *const f32, nq: u64, radius: f32, capacity: u64, offsets: *mut u64, ids: *mut u32, dist: *mut f32) -> i32;
    fn idb_range_search_batch_device_lane(ix: *mut IdbIndex, lane: u32, q: *const f32, nq: u64, radius: f32, capacity: u64, offsets: *mut u64, ids: *mut u32, dist: *mut f32, total: *mut u64) -> i32;
    fn idb_graph_range_search_batch_f32(ix: *mut IdbIndex, q: *const f32, nq: u64, ef: u32, radius: f32, capacity: u64, offsets: *mut u64, ids: *mut u32, dist: *mut f32) -> i32;
    fn idb_graph_range_search_batch_device_lane(ix: *mut IdbIndex, lane: u32, q: *const f32, nq: u64, ef: u32, radius: f32, capacity: u64, offsets: *mut u64, ids: *mut u32, dist: *mut f32, total: *mut u64) -> i32;
    fn idb_index_insert_f32(ix: *mut IdbIndex, rows: *const f32, m: u64, dim: u32, p: *const IdbParams, global_ids: *const u32, out_ids: *mut u32) -> i32;
    fn idb_index_remove(ix: *mut IdbIndex, pids: *const u32, m: u64, p: *const IdbParams, out_new_ids: *mut u32) -> i32;
    fn idb_index_free(ix: *mut IdbIndex);
    fn idb_last_error() -> *const c_char;
    // Batched / device-side / multi-GPU entry points (no counterpart in the reference; see include/instant_distance_b200.h):
    //   idb_search_batch_device_lane, idb_index_lane_stream, idb_last_search_failures   — device buffers, 4 submission lanes per index
    //   idb_comm_create, idb_index_set_id_map, idb_sharded_search_batch_f32_multi        — PointId-range shards + ONE all-gather
    //   idb_device_set_persisting_l2                                                      — opt out of the persisting-L2 reservation
}
fn last_error() -> String {
    unsafe { CStr::from_ptr(idb_last_error()).to_string_lossy().into_owned() }
}

/// types.rs:236-267
#[derive(Clone, Copy, Debug, Eq, Hash, Ord, PartialEq, PartialOrd)]
pub struct PointId(pub(crate) u32);
impl PointId {
    pub fn is_valid(self) -> bool { self.0 != u32::MAX }
    pub fn into_inner(self) -> u32 { self.0 }
}

/// lib.rs:780-782
pub trait Point: Clone + Sync {
    fn distance(&self, other: &Self) -> f32;
}
/// The f32-vector point the GPU engine serves; metric = squared L2 (instant-distance-py/src/lib.rs:378-421).
#[derive(Clone)]
pub struct F32Point(pub Vec<f32>);
impl Point for F32Point {
    fn distance(&self, o: &Self) -> f32 { self.0.iter().zip(&o.0).map(|(a, b)| (a - b) * (a - b)).sum() }
}

/// What the index reports (include/instant_distance_b200.h IDB_METRIC_*): squared L2, or 1 - cos through canonically normalised
/// points and queries (DESIGN.md §3a).  `F32Point::distance` stays squared L2.
pub const METRIC_L2SQ: u32 = 0;
pub const METRIC_COSINE: u32 = 1;

/// How an index stores its rows (include/instant_distance_b200.h IDB_STORAGE_*, the `storage` field of `IdbParams`): f32, rounded
/// to bf16 / fp16 (half the bytes; fp16 refuses values that round to infinity), or quantised to a per-row 8-bit grid (q8: a quarter
/// of the bytes plus 8 per row; refuses non-finite rows), or kept as 0/1 bits (bin: one byte per four elements; refuses any other
/// value and the cosine metric).  Distances stay fp32 on the exactly widened or dequantised rows.
pub const STORAGE_F32: u32 = 0;
pub const STORAGE_BF16: u32 = 1;
pub const STORAGE_F16: u32 = 2;
pub const STORAGE_Q8: u32 = 4;
pub const STORAGE_BIN: u32 = 8;

/// The canonical normalisation the cosine metric applies, evaluated on `device` (rows: n x dim, row-major).
pub fn normalize(rows: &[f32], dim: usize, device: i32) -> Vec<f32> {
    let mut out = vec![0f32; rows.len()];
    let rc = unsafe { idb_normalize_f32(rows.as_ptr(), (rows.len() / dim.max(1)) as u64, dim as u32, device, out.as_mut_ptr()) };
    assert_eq!(rc, 0, "{}", last_error());
    out
}

/// lib.rs:115-128
#[derive(Copy, Clone, Debug)]
pub struct Heuristic { pub extend_candidates: bool, pub keep_pruned: bool }
impl Default for Heuristic {
    fn default() -> Self { Heuristic { extend_candidates: false, keep_pruned: true } }
}

/// lib.rs:21-113
#[derive(Clone)]
pub struct Builder { ef_search: usize, ef_construction: usize, heuristic: Option<Heuristic>, ml: f32, seed: u64, metric: u32 }
impl Default for Builder {
    fn default() -> Self {
        let mut p = unsafe { std::mem::zeroed::<IdbParams>() };
        unsafe { idb_params_default(&mut p) };
        Self { ef_search: 100, ef_construction: 100, heuristic: Some(Heuristic::default()), ml: p.ml, seed: 0, metric: METRIC_L2SQ }
    }
}
impl Builder {
    /// Not in the reference: METRIC_L2SQ (default) or METRIC_COSINE.
    pub fn metric(mut self, v: u32) -> Self { self.metric = v; self }
    pub fn ef_construction(mut self, v: usize) -> Self { self.ef_construction = v; self }
    pub fn ef_search(mut self, v: usize) -> Self { self.ef_search = v; self }
    pub fn select_heuristic(mut self, h: Option<Heuristic>) -> Self { self.heuristic = h; self }
    pub fn ml(mut self, v: f32) -> Self { self.ml = v; self }
    pub fn seed(mut self, v: u64) -> Self { self.seed = v; self }
    /// lib.rs:83-85
    pub fn build_hnsw(self, points: Vec<F32Point>) -> (Hnsw, Vec<PointId>) {
        let dim = points.first().map_or(1, |p| p.0.len());
        let flat: Vec<f32> = points.iter().flat_map(|p| p.0.iter().copied()).collect();
        let mut p = unsafe { std::mem::zeroed::<IdbParams>() };
        unsafe { idb_params_default(&mut p) };
        p.ef_construction = self.ef_construction as u32;
        p.ef_search = self.ef_search as u32;
        p.ml = self.ml;
        p.seed = self.seed;
        p.heuristic = self.heuristic.is_some() as i32;
        if let Some(h) = self.heuristic { p.extend_candidates = h.extend_candidates as i32; p.keep_pruned = h.keep_pruned as i32; }
        let mut raw = std::ptr::null_mut();
        let mut ids = vec![0u32; points.len()];
        let rc = unsafe { idb_build_ex(flat.as_ptr(), points.len() as u64, dim as u32, &p, self.metric, &mut raw, ids.as_mut_ptr()) };
        assert_eq!(rc, 0, "{}", last_error()); // the reference's build is infallible
        let mut shuffled = points.clone(); // Hnsw::points is in PointId order (lib.rs:263-270)
        for (orig, pid) in ids.iter().enumerate() { shuffled[*pid as usize] = points[orig].clone(); }
        (Hnsw { raw, points: shuffled, ef_search: self.ef_search, m: p.m }, ids.into_iter().map(PointId).collect())
    }
    /// lib.rs:78-80 -> HnswMap::new (lib.rs:141-152)
    pub fn build<V: Clone>(self, points: Vec<F32Point>, values: Vec<V>) -> HnswMap<V> {
        let (hnsw, ids) = self.build_hnsw(points);
        let mut sorted = ids.into_iter().enumerate().collect::<Vec<_>>();
        sorted.sort_unstable_by_key(|id| id.1);
        let values = sorted.into_iter().map(|(src, _)| values[src].clone()).collect();
        HnswMap { hnsw, values }
    }
}

/// lib.rs:560-574 — the traversal scratch lives on the device; this holds the result list of the last search.
#[derive(Default)]
pub struct Search { nearest: Vec<(f32, PointId)> }

/// lib.rs:193-199
pub struct Hnsw { raw: *mut IdbIndex, points: Vec<F32Point>, ef_search: usize, m: u32 }
unsafe impl Send for Hnsw {}
unsafe impl Sync for Hnsw {} // lib.rs:352-356: concurrent searches each take a submission lane inside the library and overlap on the device
impl Drop for Hnsw {
    fn drop(&mut self) { unsafe { idb_index_free(self.raw) } }
}
pub struct Item<'a> { pub distance: f32, pub pid: PointId, pub point: &'a F32Point }
impl Hnsw {
    pub fn builder() -> Builder { Builder::default() }
    /// lib.rs:352-383
    pub fn search<'a, 'b: 'a>(&'b self, point: &F32Point, search: &'a mut Search) -> impl ExactSizeIterator<Item = Item<'b>> + 'a {
        let ef = self.ef_search;
        search.nearest.clear();
        if ef > 0 && !self.points.is_empty() {
            let (mut ids, mut dist, mut len) = (vec![u32::MAX; ef], vec![f32::INFINITY; ef], 0u32);
            let rc = unsafe { idb_search_batch_f32(self.raw, point.0.as_ptr(), 1, ef as u32, ef as u32, ids.as_mut_ptr(), dist.as_mut_ptr(), &mut len) };
            assert_eq!(rc, 0, "{}", last_error());
            search.nearest.extend((0..len as usize).map(|i| (dist[i], PointId(ids[i]))));
        }
        search.nearest.iter().map(move |&(distance, pid)| Item { distance, pid, point: &self.points[pid.0 as usize] })
    }
    /// Not in the reference: the exact k nearest points (every point scanned; ties by lower PointId), as (distance, PointId).
    pub fn search_exact(&self, point: &F32Point, k: usize) -> Vec<(f32, PointId)> {
        if k == 0 { return Vec::new(); }
        let (mut ids, mut dist, mut len) = (vec![u32::MAX; k], vec![f32::INFINITY; k], 0u32);
        let rc = unsafe { idb_exact_search_batch_f32(self.raw, point.0.as_ptr(), 1, k as u32, ids.as_mut_ptr(), dist.as_mut_ptr(), &mut len) };
        assert_eq!(rc, 0, "{}", last_error());
        (0..len as usize).map(|i| (dist[i], PointId(ids[i]))).collect()
    }
    /// Not in the reference: every point within `radius` of `point` (distance <= radius; exact, every point scanned), nearest first,
    /// ties by lower PointId, as (distance, PointId).
    pub fn search_range(&self, point: &F32Point, radius: f32) -> Vec<(f32, PointId)> {
        let mut offsets = [0u64; 2];
        let mut cap = 1024usize;
        loop {
            let (mut ids, mut dist) = (vec![u32::MAX; cap], vec![f32::INFINITY; cap]);
            let rc = unsafe {
                idb_range_search_batch_f32(self.raw, point.0.as_ptr(), 1, radius, cap as u64, offsets.as_mut_ptr(), ids.as_mut_ptr(), dist.as_mut_ptr())
            };
            if rc == 7 && offsets[1] as usize > cap { cap = offsets[1] as usize; continue; } // IDB_ERR_CAPACITY: once more, sized exactly
            assert_eq!(rc, 0, "{}", last_error());
            return (0..offsets[1] as usize).map(|i| (dist[i], PointId(ids[i]))).collect();
        }
    }
    /// Not in the reference: the points within `radius` of `point` that layer 0 reaches from its `ef_search` approximate nearest
    /// neighbours through points within `radius` (0: the index's ef_search), nearest first, ties by lower PointId, as (distance,
    /// PointId).  A subset of search_range's result, at a cost that follows the hits rather than the number of points.
    pub fn search_range_graph(&self, point: &F32Point, radius: f32, ef_search: u32) -> Vec<(f32, PointId)> {
        let mut offsets = [0u64; 2];
        let mut cap = 1024usize;
        loop {
            let (mut ids, mut dist) = (vec![u32::MAX; cap], vec![f32::INFINITY; cap]);
            let rc = unsafe {
                idb_graph_range_search_batch_f32(self.raw, point.0.as_ptr(), 1, ef_search, radius, cap as u64, offsets.as_mut_ptr(),
                                                 ids.as_mut_ptr(), dist.as_mut_ptr())
            };
            if rc == 7 && offsets[1] as usize > cap { cap = offsets[1] as usize; continue; } // IDB_ERR_CAPACITY: once more, sized exactly
            assert_eq!(rc, 0, "{}", last_error());
            return (0..offsets[1] as usize).map(|i| (dist[i], PointId(ids[i]))).collect();
        }
    }
    /// Not in the reference: removes the points `pids` (distinct PointIds).  The rows that listed a removed point are selected again
    /// with `ef_construction` and `heuristic` (None: the simple selection); the other points keep their order and are renumbered
    /// without gaps.  Returns, for each point the index had, its PointId afterwards, or None for a removed one.
    pub fn remove(&mut self, pids: &[PointId], ef_construction: usize, heuristic: Option<Heuristic>) -> Vec<Option<PointId>> {
        let mut p = unsafe { std::mem::zeroed::<IdbParams>() };
        unsafe { idb_params_default(&mut p) };
        p.m = self.m;
        p.ef_construction = ef_construction as u32;
        p.heuristic = heuristic.is_some() as i32;
        if let Some(h) = heuristic { p.extend_candidates = h.extend_candidates as i32; p.keep_pruned = h.keep_pruned as i32; }
        let raw: Vec<u32> = pids.iter().map(|pid| pid.0).collect();
        let mut new_ids = vec![u32::MAX; self.points.len()];
        let rc = unsafe { idb_index_remove(self.raw, raw.as_ptr(), raw.len() as u64, &p, new_ids.as_mut_ptr()) };
        assert_eq!(rc, 0, "{}", last_error());
        let old = std::mem::take(&mut self.points);
        self.points = old.into_iter().zip(&new_ids).filter(|(_, y)| **y != u32::MAX).map(|(pt, _)| pt).collect();
        new_ids.into_iter().map(|y| if y == u32::MAX { None } else { Some(PointId(y)) }).collect()
    }
    pub fn iter(&self) -> impl Iterator<Item = (PointId, &F32Point)> { self.points.iter().enumerate().map(|(i, p)| (PointId(i as u32), p)) }
}
impl std::ops::Index<PointId> for Hnsw {
    type Output = F32Point;
    fn index(&self, i: PointId) -> &F32Point { &self.points[i.0 as usize] }
}

/// lib.rs:130-173
pub struct HnswMap<V> { hnsw: Hnsw, pub values: Vec<V> }
pub struct MapItem<'a, V> { pub distance: f32, pub pid: PointId, pub point: &'a F32Point, pub value: &'a V }
impl<V: Clone> HnswMap<V> {
    pub fn search<'a>(&'a self, point: &F32Point, search: &'a mut Search) -> impl ExactSizeIterator<Item = MapItem<'a, V>> + 'a {
        self.hnsw.search(point, search).map(move |it| MapItem { distance: it.distance, pid: it.pid, point: it.point, value: &self.values[it.pid.0 as usize] })
    }
    pub fn iter(&self) -> impl Iterator<Item = (PointId, &F32Point)> { self.hnsw.iter() }
    /// Hnsw::remove; the values of the removed points are dropped, the others follow their points' new PointIds.
    pub fn remove(&mut self, pids: &[PointId], ef_construction: usize, heuristic: Option<Heuristic>) -> Vec<Option<PointId>> {
        let new_ids = self.hnsw.remove(pids, ef_construction, heuristic);
        let old = std::mem::take(&mut self.values);
        self.values = old.into_iter().zip(&new_ids).filter(|(_, y)| y.is_some()).map(|(v, _)| v).collect();
        new_ids
    }
}
