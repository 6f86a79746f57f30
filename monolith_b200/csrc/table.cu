// table.cu — storage management of the collisionless table: creation, growth (row slabs and
// bucket array), TTL eviction, export.  The probe / insert primitives are in common.cuh.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "engine.h"

namespace mono {

std::atomic<int64_t> g_launches{0};
std::atomic<int> g_opt_lookup_tma{1};  // TMA-staged single-table lookup: the faster forward on H100 (A/B below)

namespace {
struct KnobDef { const char* name; int dflt; };
// claim_pf  : the claim kernel prefetches (L2) the NEXT occurrence's scratch-set slot and table bucket
// seg_vpl   : 16-byte vectors of a gradient row per lane in seg_reduce_kernel (1 | 2)
// apply_pf  : runs_apply_kernel prefetches (L2) the next run's weight / optimizer-state rows
// lookup_pf : the lookup kernels prefetch (L2) the next occurrence's table bucket
// seg_ahead : seg_reduce_kernel loads the positions of the two following pieces up front (no dependent position load)
// claim_dual / lookup_dual : both candidate buckets of a key are requested together (rowops.cuh probe_lane<DUAL>)
// Measured on one H100 SXM 80 GB (400 W) with bench.py --ab, C2 step, defaults 0.780 / 0.785 ms: every variant loses
// (claim_pf 0.821, apply_pf 0.796, lookup_pf 0.815, claim_dual 0.800, lookup_dual 0.795, seg_vpl = 2 0.811,
// seg_ahead = 0 0.792 ms) except the TMA-staged lookup (lookup_tma = 1: 0.770 ms), which is therefore the default.
const KnobDef kKnobs[KNOB_COUNT] = {{"claim_pf", 0}, {"seg_vpl", 1}, {"apply_pf", 0}, {"lookup_pf", 0},
                                    {"claim_dual", 0}, {"lookup_dual", 0}, {"seg_ahead", 1}};
std::atomic<int> g_knob[KNOB_COUNT];
std::once_flag g_knob_once;
void knob_init() {
  for (int i = 0; i < KNOB_COUNT; ++i) g_knob[i].store(kKnobs[i].dflt);
  const char* e = std::getenv("MONO_KNOBS");
  if (!e) return;
  std::string str(e);
  size_t pos = 0;
  while (pos < str.size()) {
    size_t end = str.find(',', pos);
    if (end == std::string::npos) end = str.size();
    const std::string kv = str.substr(pos, end - pos);
    const size_t eq = kv.find('=');
    if (eq != std::string::npos) {
      const int id = knob_id(kv.substr(0, eq).c_str());
      if (id >= 0) g_knob[id].store(std::atoi(kv.c_str() + eq + 1));
    }
    pos = end + 1;
  }
}
}  // namespace
int knob_id(const char* name) {
  for (int i = 0; i < KNOB_COUNT; ++i)
    if (name && std::strcmp(name, kKnobs[i].name) == 0) return i;
  return -1;
}
int knob(int id) {
  std::call_once(g_knob_once, knob_init);
  return g_knob[id].load(std::memory_order_relaxed);
}
void knob_set(int id, int value) {
  std::call_once(g_knob_once, knob_init);
  g_knob[id].store(value);
}

// ------------------------------------------------------------------------------------------
// StageRing
// ------------------------------------------------------------------------------------------
void StageRing::init() {
  MONO_CUDA(cudaHostAlloc((void**)&host, kBlocks * kBlockBytes, cudaHostAllocDefault));
  MONO_CUDA(cudaMalloc((void**)&dev, kBlocks * kBlockBytes));
  for (int i = 0; i < kBlocks; ++i) {
    MONO_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    used[i] = false;
  }
}
void StageRing::destroy() {
  if (host) cudaFreeHost(host);
  if (dev) cudaFree(dev);
  for (int i = 0; i < kBlocks; ++i) cudaEventDestroy(ev[i]);
  host = dev = nullptr;
}
int StageRing::acquire() {
  int idx = next;
  next = (next + 1) % kBlocks;
  if (used[idx]) MONO_CUDA(cudaEventSynchronize(ev[idx]));
  used[idx] = true;
  return idx;
}
void StageRing::commit(int idx, size_t bytes, cudaStream_t s) {
  if (bytes > kBlockBytes) throw ArgError("call descriptor larger than staging block");
  MONO_CUDA(cudaMemcpyAsync(d(idx), h(idx), bytes, cudaMemcpyHostToDevice, s));
  MONO_CUDA(cudaEventRecord(ev[idx], s));
}

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
rehash_kernel(const Entry* __restrict__ old_buckets, uint64_t old_slots,
              const Entry* __restrict__ old_stash, uint32_t old_stash_cap,
              const TableDev* __restrict__ nt) {
  uint64_t total = old_slots + old_stash_cap;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total;
       i += (uint64_t)gridDim.x * blockDim.x) {
    Entry e = i < old_slots ? ld_entry_nc(old_buckets + i) : ld_entry_nc(old_stash + (i - old_slots));
    if (e.row < kTombRow) {
      e.row &= kRowMask;  // (no entry can be mid-move here: growth is stream-ordered with the inserts)
      cuckoo_insert(nt, e);
    }
  }
}

// ref: CuckooEmbeddingHashTable::Evict (cuckoo_embedding_hash_table.cc:251-264) via
// cuckoohash_map::evict (cuckoohash_map.hpp:775-800): a full scan, here one coalesced stream over
// the 16-byte entries.  Freed rows go to the free list.
__global__ void __launch_bounds__(kThreads)
evict_kernel(const TableDev* __restrict__ t, int64_t max_update_time) {
  extern __shared__ uint32_t s_pairs[];
  const int np = t->n_slot_expire;
  for (int i = threadIdx.x; i < 2 * np; i += blockDim.x) s_pairs[i] = t->slot_expire[i];
  __syncthreads();
  const uint64_t slots = (uint64_t)t->num_buckets * kBucketSlots;
  const uint64_t total = slots + t->stash_cap;
  const Entry empty = empty_entry();
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total;
       i += (uint64_t)gridDim.x * blockDim.x) {
    Entry* p = i < slots ? t->buckets + i : t->stash + (i - slots);
    Entry e = ld_entry(p);
    if (e.row >= kTombRow) continue;
    int64_t expire = t->default_expire_days;
    uint32_t slot = slot_id_v2(e.key);
    for (int j = 0; j < np; ++j)
      if (s_pairs[2 * j] == slot) { expire = s_pairs[2 * j + 1]; break; }
    if (max_update_time - (int64_t)e.ts >= expire * 86400LL) {
      Entry dead = empty;
      if (i >= slots) dead.row = kTombRow;  // keep stash probe chains intact
      *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&dead);
      uint32_t idx = atomicAdd(t->ctrs + kCtrFree, 1u);
      t->free_list[idx] = e.row & kRowMask;
      atomicSub(t->ctrs + kCtrSize, 1u);
    }
  }
}

// Export live rows of buckets [b0, b1): flat entry = [emb | state | found=1 | ts].
__global__ void __launch_bounds__(kThreads)
export_kernel(const TableDev* __restrict__ t, uint64_t slot0, uint64_t slot1, int64_t* ids_out,
              float* entry_out, uint32_t* n_out) {
  const int W = t->dim + t->state_dim + 2;
  for (uint64_t i = slot0 + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < slot1;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t slots = (uint64_t)t->num_buckets * kBucketSlots;
    const Entry* p = i < slots ? t->buckets + i : t->stash + (i - slots);
    Entry e = ld_entry_nc(p);
    if (e.row >= kTombRow) continue;
    uint32_t o = atomicAdd(n_out, 1u);
    ids_out[o] = e.key;
    float* dst = entry_out + (size_t)o * W;
    const float* src = t->emb + (size_t)(e.row & kRowMask) * t->emb_stride;
    for (int j = 0; j < t->dim; ++j) dst[j] = src[j];
    const float* st = t->state + (size_t)(e.row & kRowMask) * t->state_stride;
    for (int j = 0; j < t->state_dim; ++j) dst[t->dim + j] = st[j];
    dst[t->dim + t->state_dim] = __uint_as_float(1u);
    dst[t->dim + t->state_dim + 1] = __uint_as_float(e.ts);
  }
}

// ------------------------------------------------------------------------------------------
// host
// ------------------------------------------------------------------------------------------
static int state_floats(const mono_segment_cfg& s) {
  switch (s.opt_type) {
    case MONO_OPT_SGD: case MONO_OPT_MOVING_AVERAGE: return 0;
    case MONO_OPT_ADAGRAD: return s.dim;
    case MONO_OPT_FTRL: return 2 * s.dim;
    case MONO_OPT_ADAM: return 2 * s.dim + 2;
    case MONO_OPT_MOMENTUM: case MONO_OPT_RMSPROP: case MONO_OPT_RMSPROPV2: return s.dim;
    case MONO_OPT_ADADELTA: return 2 * s.dim;
    case MONO_OPT_AMSGRAD: return 3 * s.dim + 2;
    case MONO_OPT_GROUP_ADAGRAD: return 1;
  }
  throw ArgError("unknown optimizer type");
}

static uint32_t round_up4(uint32_t x) { return (x + 3u) & ~3u; }

static uint32_t buckets_for(uint64_t keys) {
  // sized so that `keys` keys sit at load factor 0.5 (4 slots per bucket)
  uint64_t nb = (keys + 1) / 2 + 1;
  if (nb < 64) nb = 64;
  if (nb > 0xFFFFFFF0ull) throw ArgError("table too large for 32-bit bucket index");
  return (uint32_t)nb;
}

void table_init(mono_mtable* mt, HostTable& t, const mono_table_cfg& cfg, cudaStream_t s) {
  (void)mt;
  if (cfg.n_segments <= 0 || cfg.n_segments > kMaxSegs)
    throw ArgError("n_segments must be in [1, 8]");
  t.name = cfg.name ? cfg.name : "";
  TableDev& d = t.dev;
  std::memset(&d, 0, sizeof(d));
  int col = 0, st = 0;
  for (int i = 0; i < cfg.n_segments; ++i) {
    const mono_segment_cfg& sc = cfg.segments[i];
    if (sc.dim <= 0) throw ArgError("segment dim must be positive");
    if (sc.init_type < 0 || sc.init_type > 3) throw ArgError("unknown initializer type");
    if (sc.opt_type < MONO_OPT_SGD || sc.opt_type > MONO_OPT_GROUP_ADAGRAD)
      throw ArgError("unknown optimizer type (built: sgd, adagrad, ftrl, adam, momentum, rmsprop, rmspropv2, adadelta, amsgrad, moving_average, group_adagrad)");
    t.segs.push_back(sc);
    SegDev& sd = d.segs[i];
    sd.col_begin = col;
    sd.dim = sc.dim;
    sd.state_off = st;
    sd.opt_type = sc.opt_type;
    sd.init_type = sc.init_type;
    sd.init_a = sc.init_a;
    sd.init_b = sc.init_b;
    for (int j = 0; j < 6; ++j) sd.p[j] = sc.opt_p[j];
    col += sc.dim;
    st += state_floats(sc);
  }
  t.dim = col;
  t.state_dim = st;
  t.slices = cfg.n_segments;  // every supported optimizer has SliceSize()==1
  d.dim = col;
  d.state_dim = st;
  d.num_segs = cfg.n_segments;
  d.emb_stride = round_up4(col);
  d.state_stride = round_up4(st);
  d.seed = cfg.init_seed;
  d.default_expire_days = cfg.default_expire_days;
  d.n_slot_expire = cfg.n_slot_expire;
  for (int i = 0; i < cfg.n_slot_expire; ++i) {
    t.slot_expire_pairs.push_back(cfg.slot_ids[i]);
    t.slot_expire_pairs.push_back(cfg.slot_expire_days[i]);
  }
  uint64_t rows = std::max<uint64_t>(cfg.initial_capacity, 1024);
  if (rows > 0x7FFFFFF0ull) throw ArgError("initial_capacity too large (row indices are 31 bits)");
  d.row_cap = (uint32_t)rows;
  d.num_buckets = buckets_for(rows);
  d.stash_cap = 4096;

  MONO_CUDA(cudaMalloc((void**)&d.ctrs, kNumCtrs * sizeof(uint32_t)));
  MONO_CUDA(cudaMemsetAsync(d.ctrs, 0, kNumCtrs * sizeof(uint32_t), s));
  size_t bbytes = (size_t)d.num_buckets * kBucketSlots * sizeof(Entry);
  MONO_CUDA(cudaMalloc((void**)&d.buckets, bbytes));
  MONO_CUDA(cudaMemsetAsync(d.buckets, 0xFF, bbytes, s));
  MONO_CUDA(cudaMalloc((void**)&d.stash, (size_t)d.stash_cap * sizeof(Entry)));
  MONO_CUDA(cudaMemsetAsync(d.stash, 0xFF, (size_t)d.stash_cap * sizeof(Entry), s));
  MONO_CUDA(cudaMalloc((void**)&d.free_list, (size_t)d.row_cap * sizeof(uint32_t)));
  MONO_CUDA(cudaMalloc((void**)&d.emb, (size_t)d.row_cap * d.emb_stride * sizeof(float)));
  if (d.state_stride)
    MONO_CUDA(cudaMalloc((void**)&d.state, (size_t)d.row_cap * d.state_stride * sizeof(float)));
  if (!t.slot_expire_pairs.empty()) {
    uint32_t* p = nullptr;
    MONO_CUDA(cudaMalloc((void**)&p, t.slot_expire_pairs.size() * sizeof(uint32_t)));
    MONO_CUDA(cudaMemcpy(p, t.slot_expire_pairs.data(), t.slot_expire_pairs.size() * sizeof(uint32_t),
                         cudaMemcpyHostToDevice));
    d.slot_expire = p;
  }
  MONO_CUDA(cudaHostAlloc((void**)&t.h_snap, kNumCtrs * sizeof(uint32_t), cudaHostAllocDefault));
  std::memset(t.h_snap, 0, kNumCtrs * sizeof(uint32_t));
  MONO_CUDA(cudaEventCreateWithFlags(&t.snap_ev, cudaEventDisableTiming));
}

// ref: hash_filter_ops.create_hash_filters + SlotOccurrenceThresholdConfig (embedding_hash_table.proto:100-110):
// a counting filter of `capacity` FIDs with a default and per-slot occurrence thresholds (0 = never filter).
void table_set_filter(mono_mtable* mt, int k, uint64_t capacity, uint32_t default_thr, const uint32_t* slots,
                      const uint32_t* thrs, int n_slots, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  TableDev& d = t.dev;
  MONO_CUDA(cudaStreamSynchronize(s));
  if (d.flt_cells) MONO_CUDA(cudaFree(d.flt_cells));
  if (d.slot_thr) MONO_CUDA(cudaFree((void*)d.slot_thr));
  d.flt_cells = nullptr;
  d.slot_thr = nullptr;
  d.n_slot_thr = 0;
  uint64_t total = (uint64_t)(capacity * 1.5);  // hash_filter.h: total_size_ = capacity * 1.5
  if (total == 0) total = 1;
  if (total > 0xFFFFFF00ull) throw ArgError("hash filter capacity too large");
  const size_t words = (size_t)((total + 64 + 1) / 2);
  MONO_CUDA(cudaMalloc((void**)&d.flt_cells, words * sizeof(uint32_t)));
  MONO_CUDA(cudaMemset(d.flt_cells, 0, words * sizeof(uint32_t)));
  d.flt_total = (uint32_t)total;
  d.flt_default_thr = default_thr;
  if (n_slots > 0) {
    std::vector<uint32_t> pairs;
    for (int i = 0; i < n_slots; ++i) {
      pairs.push_back(slots[i]);
      pairs.push_back(thrs[i]);
    }
    uint32_t* p = nullptr;
    MONO_CUDA(cudaMalloc((void**)&p, pairs.size() * sizeof(uint32_t)));
    MONO_CUDA(cudaMemcpy(p, pairs.data(), pairs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    d.slot_thr = p;
    d.n_slot_thr = n_slots;
  }
  mt->tables_dirty = true;
}

void table_free(HostTable& t) {
  TableDev& d = t.dev;
  cudaFree(d.ctrs);
  cudaFree(d.buckets);
  cudaFree(d.stash);
  cudaFree(d.free_list);
  cudaFree(d.emb);
  if (d.state) cudaFree(d.state);
  if (d.slot_expire) cudaFree((void*)d.slot_expire);
  if (d.flt_cells) cudaFree(d.flt_cells);
  if (d.slot_thr) cudaFree((void*)d.slot_thr);
  if (t.h_snap) cudaFreeHost(t.h_snap);
  if (t.snap_ev) cudaEventDestroy(t.snap_ev);
  std::memset(&d, 0, sizeof(d));
}

void upload_tables(mono_mtable* mt, cudaStream_t s) {
  if (!mt->tables_dirty) return;
  size_t K = mt->tables.size();
  size_t bytes = K * sizeof(TableDev);
  if (bytes <= StageRing::kBlockBytes) {
    int b = mt->ring.acquire();
    for (size_t k = 0; k < K; ++k)
      std::memcpy(mt->ring.h(b) + k * sizeof(TableDev), &mt->tables[k].dev, sizeof(TableDev));
    MONO_CUDA(cudaMemcpyAsync(mt->d_tables, mt->ring.h(b), bytes, cudaMemcpyHostToDevice, s));
    MONO_CUDA(cudaEventRecord(mt->ring.ev[b], s));
  } else {
    std::vector<TableDev> tmp(K);
    for (size_t k = 0; k < K; ++k) tmp[k] = mt->tables[k].dev;
    MONO_CUDA(cudaStreamSynchronize(s));
    MONO_CUDA(cudaMemcpy(mt->d_tables, tmp.data(), bytes, cudaMemcpyHostToDevice));
  }
  mt->tables_dirty = false;
}

void copy_counters_sync(mono_mtable* mt, int k, cudaStream_t s, uint32_t* out) {
  HostTable& t = mt->tables[k];
  MONO_CUDA(cudaMemcpyAsync(mt->h_flag, t.dev.ctrs, kNumCtrs * sizeof(uint32_t),
                            cudaMemcpyDeviceToHost, s));
  MONO_CUDA(cudaStreamSynchronize(s));
  std::memcpy(out, mt->h_flag, kNumCtrs * sizeof(uint32_t));
}

void read_counters_sync(mono_mtable* mt, int k, cudaStream_t s, uint32_t* out) {
  copy_counters_sync(mt, k, s, out);
  const std::string& name = mt->tables[k].name;
  if (out[kCtrError] & 1u) throw CudaError("table '" + name + "': stash overflow (insert failed)");
  if (out[kCtrError] & 2u) throw CudaError("table '" + name + "': row slab overflow");
  if (out[kCtrError] & 4u)
    throw CudaError("table '" + name + "': cuckoo displacement lost a marked slot (table changed under an insert)");
}

void request_snapshot(mono_mtable* mt, int k, cudaStream_t s) {
  (void)mt;
  HostTable& t = mt->tables[k];
  if (t.snapshot_pending) return;
  MONO_CUDA(cudaMemcpyAsync(t.h_snap, t.dev.ctrs, kNumCtrs * sizeof(uint32_t),
                            cudaMemcpyDeviceToHost, s));
  MONO_CUDA(cudaEventRecord(t.snap_ev, s));
  t.issued_at_pending = t.issued_total;
  t.snapshot_pending = true;
}

static void adopt_snapshot(HostTable& t, const uint32_t* c, uint64_t issued_at) {
  t.snap_bump = c[kCtrBump];
  t.snap_free = c[kCtrFree];
  t.snap_size = c[kCtrSize];
  t.snap_stash = c[kCtrStash];
  t.issued_at_snapshot = issued_at;
}

static void grow_rows(mono_mtable* mt, int k, uint64_t need_total, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  TableDev& d = t.dev;
  uint64_t ncap = std::max<uint64_t>((uint64_t)d.row_cap * 2, need_total + need_total / 8);
  if (ncap > 0x7FFFFFF0ull) {  // row indices are 31 bits (bit 31 of an entry's row marks a displacement in progress)
    ncap = 0x7FFFFFF0ull;
    if (ncap < need_total) throw ArgError("row capacity exceeds the 31-bit row index");
  }
  float* nemb = nullptr;
  float* nstate = nullptr;
  uint32_t* nfree = nullptr;
  MONO_CUDA(cudaMallocAsync((void**)&nemb, ncap * d.emb_stride * sizeof(float), s));
  MONO_CUDA(cudaMemcpyAsync(nemb, d.emb, (size_t)d.row_cap * d.emb_stride * sizeof(float),
                            cudaMemcpyDeviceToDevice, s));
  if (d.state_stride) {
    MONO_CUDA(cudaMallocAsync((void**)&nstate, ncap * d.state_stride * sizeof(float), s));
    MONO_CUDA(cudaMemcpyAsync(nstate, d.state, (size_t)d.row_cap * d.state_stride * sizeof(float),
                              cudaMemcpyDeviceToDevice, s));
  }
  MONO_CUDA(cudaMallocAsync((void**)&nfree, ncap * sizeof(uint32_t), s));
  MONO_CUDA(cudaMemcpyAsync(nfree, d.free_list, (size_t)d.row_cap * sizeof(uint32_t),
                            cudaMemcpyDeviceToDevice, s));
  MONO_CUDA(cudaFreeAsync(d.emb, s));
  if (d.state) MONO_CUDA(cudaFreeAsync(d.state, s));
  MONO_CUDA(cudaFreeAsync(d.free_list, s));
  d.emb = nemb;
  d.state = nstate;
  d.free_list = nfree;
  d.row_cap = (uint32_t)ncap;
  mt->tables_dirty = true;
}

static void rehash(mono_mtable* mt, int k, uint64_t keys_target, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  TableDev& d = t.dev;
  uint32_t nnb = std::max<uint64_t>((uint64_t)d.num_buckets * 2, buckets_for(keys_target));
  Entry* ob = d.buckets;
  Entry* os = d.stash;
  uint32_t onb = d.num_buckets;
  Entry* nbk = nullptr;
  Entry* nst = nullptr;
  size_t bbytes = (size_t)nnb * kBucketSlots * sizeof(Entry);
  MONO_CUDA(cudaMallocAsync((void**)&nbk, bbytes, s));
  MONO_CUDA(cudaMemsetAsync(nbk, 0xFF, bbytes, s));
  MONO_CUDA(cudaMallocAsync((void**)&nst, (size_t)d.stash_cap * sizeof(Entry), s));
  MONO_CUDA(cudaMemsetAsync(nst, 0xFF, (size_t)d.stash_cap * sizeof(Entry), s));
  MONO_CUDA(cudaMemsetAsync(d.ctrs + kCtrStash, 0, sizeof(uint32_t), s));
  d.buckets = nbk;
  d.stash = nst;
  d.num_buckets = nnb;
  mt->tables_dirty = true;
  upload_tables(mt, s);
  uint64_t old_slots = (uint64_t)onb * kBucketSlots;
  rehash_kernel<<<grid_for(old_slots + d.stash_cap, kThreads), kThreads, 0, s>>>(
      ob, old_slots, os, d.stash_cap, mt->d_tables + k);
  MONO_CHECK_LAUNCH();
  MONO_CUDA(cudaFreeAsync(ob, s));
  MONO_CUDA(cudaFreeAsync(os, s));
}

void ensure_capacity(mono_mtable* mt, int k, uint64_t n_new, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  TableDev& d = t.dev;
  if (t.snapshot_pending && cudaEventQuery(t.snap_ev) == cudaSuccess) {
    if (t.h_snap[kCtrError]) {
      uint32_t tmp[kNumCtrs];
      read_counters_sync(mt, k, s, tmp);  // throws with the right message
    }
    adopt_snapshot(t, t.h_snap, t.issued_at_pending);
    t.snapshot_pending = false;
  }
  auto needs = [&](bool& rows, bool& buckets) {
    uint64_t slack = t.issued_total - t.issued_at_snapshot;
    uint64_t avail = (uint64_t)d.row_cap - t.snap_bump + t.snap_free;
    rows = n_new + slack > avail;
    uint64_t size_ub = t.snap_size + slack + n_new;
    buckets = (double)size_ub > 0.75 * (double)d.num_buckets * kBucketSlots || t.snap_stash > 0;
  };
  bool nr, nbk;
  needs(nr, nbk);
  if (!nr && !nbk) return;
  if (t.snapshot_pending) {
    // the host ran ahead of the device: wait for the (older) in-flight snapshot only, not for the
    // whole stream, and re-evaluate with its counters
    MONO_CUDA(cudaEventSynchronize(t.snap_ev));
    if (t.h_snap[kCtrError]) {
      uint32_t tmp[kNumCtrs];
      read_counters_sync(mt, k, s, tmp);
    }
    adopt_snapshot(t, t.h_snap, t.issued_at_pending);
    t.snapshot_pending = false;
    needs(nr, nbk);
    if (!nr && !nbk) return;
  }
  // exact path (SYNC): read the true counters, then decide
  uint32_t c[kNumCtrs];
  read_counters_sync(mt, k, s, c);
  t.snapshot_pending = false;  // any in-flight snapshot is older than this read
  adopt_snapshot(t, c, t.issued_total);
  needs(nr, nbk);
  if (nr) grow_rows(mt, k, t.snap_bump - t.snap_free + n_new, s);
  if (nbk) rehash(mt, k, t.snap_size + n_new, s);
}

void evict_table(mono_mtable* mt, int k, int64_t max_update_time, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  upload_tables(mt, s);
  uint64_t total = (uint64_t)t.dev.num_buckets * kBucketSlots + t.dev.stash_cap;
  size_t smem = t.slot_expire_pairs.size() * sizeof(uint32_t);
  evict_kernel<<<grid_for(total, kThreads * 4), kThreads, smem, s>>>(mt->d_tables + k,
                                                                      max_update_time);
  MONO_CHECK_LAUNCH();
}

int64_t export_rows(mono_mtable* mt, int k, int64_t* cursor, int64_t max_n, int64_t* ids_out,
                    float* entry_out, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  upload_tables(mt, s);
  const uint64_t total = (uint64_t)t.dev.num_buckets * kBucketSlots + t.dev.stash_cap;
  if (*cursor < 0 || (uint64_t)*cursor >= total) { *cursor = -1; return 0; }
  uint64_t s0 = (uint64_t)*cursor;
  uint64_t s1 = std::min<uint64_t>(total, s0 + (uint64_t)max_n);  // <= max_n live rows in range
  uint32_t* n_dev = t.dev.ctrs + kCtrAux;
  MONO_CUDA(cudaMemsetAsync(n_dev, 0, sizeof(uint32_t), s));
  export_kernel<<<grid_for(s1 - s0, kThreads), kThreads, 0, s>>>(mt->d_tables + k, s0, s1, ids_out,
                                                                  entry_out, n_dev);
  MONO_CHECK_LAUNCH();
  MONO_CUDA(cudaMemcpyAsync(mt->h_flag, n_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  MONO_CUDA(cudaStreamSynchronize(s));
  *cursor = s1 >= total ? -1 : (int64_t)s1;
  return (int64_t)mt->h_flag[0];
}

}  // namespace mono
