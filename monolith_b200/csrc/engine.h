// engine.h — host-side state of the engine (one mono_mtable = K tables on one device).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <map>
#include <mutex>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace mono {

extern std::atomic<int64_t> g_launches;  // kernels launched by this library
extern std::atomic<int> g_opt_lookup_tma; // mono_set_option("lookup_tma")
// Tuning knobs (mono_set_option(name) / env MONO_KNOBS="name=value,..."): each selects between two implementations of
// the same result, kept switchable so that a bench run can A/B them in one session.
enum Knob { KNOB_CLAIM_PF = 0, KNOB_SEG_VPL, KNOB_APPLY_PF, KNOB_LOOKUP_PF, KNOB_CLAIM_DUAL, KNOB_LOOKUP_DUAL, KNOB_SEG_AHEAD, KNOB_COUNT };
int knob(int id);
int knob_id(const char* name);            // -1: unknown
void knob_set(int id, int value);

// tower.cu: the e2e bench's stand-in dense tower (64-64-1 bf16 MLP + logistic loss), forward + input gradient in one kernel
int tower_scratch_floats();
void tower_grad(const float* x, int64_t batch, const float* labels, const void* w1_bf16, const void* w2_bf16, float* dx,
                float* loss, float* scratch, cudaStream_t s);
#define MONO_COUNT_LAUNCH() (::mono::g_launches.fetch_add(1, std::memory_order_relaxed))

struct CudaError : std::runtime_error {
  using std::runtime_error::runtime_error;
};
struct ArgError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

#define MONO_CUDA(expr)                                                                    \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess)                                                                 \
      throw ::mono::CudaError(std::string(#expr) + ": " + cudaGetErrorString(_e));         \
  } while (0)

#define MONO_CHECK_LAUNCH()                                                                \
  do {                                                                                     \
    MONO_COUNT_LAUNCH();                                                                   \
    cudaError_t _e = cudaGetLastError();                                                   \
    if (_e != cudaSuccess)                                                                 \
      throw ::mono::CudaError(std::string("kernel launch: ") + cudaGetErrorString(_e));    \
  } while (0)

// Lane-group width for rows of up to max_dim floats: one 4-float vector per lane, 4 to 32 lanes.
int pick_group(int max_dim);

template <int N>
using Int = std::integral_constant<int, N>;

// Calls f(Int<G>{}) with the lane-group width G as a constant: 4, 8, 16, and 32 for anything else.
template <class F>
inline void by_group(int G, F&& f) {
  switch (G) {
    case 4: f(Int<4>{}); break;
    case 8: f(Int<8>{}); break;
    case 16: f(Int<16>{}); break;
    default: f(Int<32>{}); break;
  }
}

// Raises Kernel's dynamic shared memory limit to `bytes`, once per device: the attribute is set on the current
// device only, so a process that launches the kernel on several devices sets it on each.
constexpr int kMaxDevices = 64;
template <auto Kernel>
inline void set_max_dynamic_smem(size_t bytes) {
  static std::atomic<bool> done[kMaxDevices];
  int dev = 0;
  MONO_CUDA(cudaGetDevice(&dev));
  const bool keep = dev >= 0 && dev < kMaxDevices;
  if (keep && done[dev].load(std::memory_order_relaxed)) return;
  MONO_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  if (keep) done[dev].store(true, std::memory_order_relaxed);
}

// Streaming multiprocessors of the current device (132 on an H100 SXM): grid caps are multiples of it.
inline int device_sms() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return std::max(1, sms);
}

// max_blocks = 0: eight blocks per SM
inline int grid_for(int64_t work_items, int items_per_block, int max_blocks = 0) {
  if (max_blocks <= 0) max_blocks = device_sms() * 8;
  int64_t b = (work_items + items_per_block - 1) / items_per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return (int)b;
}

// Persistent-style grid: exactly one resident wave (SMs x occupancy), never a partial second wave;
// the kernels are grid-stride loops.  The occupancy query is cached per kernel.
template <class Kernel>
inline int resident_grid(Kernel kernel, int64_t work_items, int items_per_block, int threads = kThreads,
                         size_t smem = 0) {
  static std::mutex mu;
  static std::map<const void*, int> cache;  // keyed by kernel address
  int cached_blocks = 0;
  {
    std::lock_guard<std::mutex> lk(mu);
    auto it = cache.find(reinterpret_cast<const void*>(kernel));
    if (it != cache.end()) cached_blocks = it->second;
  }
  if (cached_blocks == 0) {
    int per_sm = 0, sms = 0, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem) != cudaSuccess ||
        per_sm < 1)
      per_sm = 1;
    cached_blocks = std::max(1, sms) * per_sm;
    std::lock_guard<std::mutex> lk(mu);
    cache[reinterpret_cast<const void*>(kernel)] = cached_blocks;
  }
  int64_t b = (work_items + items_per_block - 1) / items_per_block;
  if (b < 1) b = 1;
  return (int)std::min<int64_t>(b, cached_blocks);
}

// growable device scratch buffer (stream-ordered allocation)
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  void* get(size_t bytes, cudaStream_t s) {
    if (bytes > cap) {
      if (p) MONO_CUDA(cudaFreeAsync(p, s));
      size_t ncap = bytes + bytes / 2 + 256;
      MONO_CUDA(cudaMallocAsync(&p, ncap, s));
      cap = ncap;
    }
    return p;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
};

// Scratch open-addressing set of the claim kernels, versioned by an epoch in every entry: an entry whose
// epoch differs from the current call's is EMPTY, so the set is never cleared between calls (clearing 16 B
// x 2 x occurrences is a full extra memset pass per step); it is zero-filled once per (re)allocation and when the epoch wraps.
// The entry layout and the one claim loop: common.cuh claim_epoch_slot.
struct ClaimSet {
  DevBuf buf;
  void* init_ptr = nullptr;
  size_t init_bytes = 0;
  uint32_t epoch = 0;
  // returns the set (>= bytes) and the epoch to claim with
  void* get(size_t bytes, cudaStream_t s, uint32_t* epoch_out) {
    void* p = buf.get(bytes, s);
    if (p != init_ptr || buf.cap > init_bytes || epoch >= 0xFFFFFFF0u) {
      MONO_CUDA(cudaMemsetAsync(p, 0, buf.cap, s));
      init_ptr = p;
      init_bytes = buf.cap;
      epoch = 0;
    }
    *epoch_out = ++epoch;
    return p;
  }
  void release() {
    buf.release();
    init_ptr = nullptr;
    init_bytes = 0;
    epoch = 0;
  }
};

// Slots of a claim set for n keys (n <= 2^30): the smallest power of two >= max(1024, 2n), so the set is at most
// half full.
inline uint32_t claim_set_slots(int64_t n) {
  uint32_t cap = 1024;
  while ((uint64_t)cap < 2 * (uint64_t)n) cap <<= 1;
  return cap;
}

// Ring of pinned host blocks mirrored by device blocks: small per-call descriptors (segments,
// learning rates) are written to a pinned block and copied H2D on the call's stream.
struct StageRing {
  static constexpr int kBlocks = 32;
  static constexpr size_t kBlockBytes = 128 * 1024;
  char* host = nullptr;
  char* dev = nullptr;
  cudaEvent_t ev[kBlocks];
  bool used[kBlocks];
  int next = 0;
  void init();
  void destroy();
  // returns block index; host pointer = host + idx*kBlockBytes
  int acquire();
  char* h(int idx) { return host + (size_t)idx * kBlockBytes; }
  char* d(int idx) { return dev + (size_t)idx * kBlockBytes; }
  void commit(int idx, size_t bytes, cudaStream_t s);  // H2D + event
};

struct HostTable {
  std::string name;
  std::vector<mono_segment_cfg> segs;
  int dim = 0, state_dim = 0, slices = 0;
  TableDev dev{};  // host mirror of the device descriptor
  std::vector<uint32_t> slot_expire_pairs;
  int64_t max_update_ts = 0;
  // conservative host-side bounds (exact values live in dev.ctrs)
  uint64_t snap_size = 0, snap_bump = 0, snap_free = 0, snap_stash = 0;
  uint64_t issued_total = 0;        // ids submitted to insert-capable calls so far
  uint64_t issued_at_snapshot = 0;  // issued_total when the last completed snapshot was requested
  uint64_t issued_at_pending = 0;
  bool snapshot_pending = false;
  uint32_t* h_snap = nullptr;  // pinned [kNumCtrs]
  cudaEvent_t snap_ev = nullptr;
};

// ---- scratch of the backward's claim -> sort -> run list -> reduce pipeline (bwd.cu scratch_plan) ----
// Counters block at the head of the scratch (one memset clears it every call), word offsets:
constexpr int kCtrRuns = 0;       // runs of the sorted list (= distinct keys)
constexpr int kCtrMisses = 8;     // FIDs the claim found absent from the table
constexpr int kCtrOwners = 512;   // distinct FIDs per owner [256], then the claim set's region-overflow flag
constexpr size_t kCtrBytes = 4096;

struct SortWs {                 // the sort's and the run list's regions
  uint2 *a, *b;                 // ping-pong item buffers [M]
  uint32_t* cnt;                // [radix blocks][2048]
  uint32_t* dtot;               // [passes][2048]
  uint32_t* blk_runs;           // [run blocks]
  uint32_t* run_start;          // [M + 1]
  uint32_t* run_first_pos;      // [M]
  uint32_t* piece_run_base;     // [ceil(M / 32)]
  uint32_t* n_runs;             // device counter
  uint32_t* run_of_sorted;      // optional [M]: run index of every sorted element
  uint32_t* rowidx;             // optional [M]: each run's resolved row, gathered from the claim set
};

struct SegMeta;  // bwd.cu

// Typed views into one scratch buffer; the optional parts a caller did not ask for are null.
struct BwdScratch {
  size_t bytes;
  uint32_t* ctr;                // counters block (kCtr*)
  uint32_t* k0;                 // optional [M]: claim keys (the claim-set slot of every occurrence)
  uint32_t* miss;               // optional [M]: slots of the FIDs the claim found absent
  uint32_t* occ;                // optional [M]: occurrence -> pooled row (CSR gradient source)
  SortWs sort;
  float* part;                  // [2 * n_pieces][D] long-run block sums
  SegMeta* meta;                // [2 * n_pieces]
  float* ugrad;                 // optional [M][D]: summed gradient of every run
  int64_t* fids;                // optional [M]: a parts call's FIDs, table-major
  const float** occ_src;        // optional [M]: its gradient row (column included) of every occurrence
  float* occ_div;               // optional [M]: its MEAN divisor of every occurrence (0 = none)
  int64_t n_pieces;
  const uint2* sorted;          // the sorted {key, position} list, once the sort has run
};

}  // namespace mono

struct mono_mtable {
  mutable std::recursive_mutex mu;  // serialises host threads on this handle (capi.cu HandleGuard)
  int device = 0;
  std::vector<mono::HostTable> tables;
  mono::TableDev* d_tables = nullptr;  // device array [K]
  bool tables_dirty = true;
  mono::StageRing ring;
  mono::DevBuf ws_miss, ws_a, ws_b, ws_c, ws_d, ws_e, ws_host_in, ws_host_out;
  mono::ClaimSet claim_set;  // pool_backward's FID grouping set
  float* zero_row = nullptr;  // 128 floats of +0.0: the gradient row of a FIRSTN occurrence beyond its sequence length
  void* pinned_in = nullptr;
  size_t pinned_in_cap = 0;
  void* pinned_out = nullptr;
  size_t pinned_out_cap = 0;
  cudaStream_t own_stream = nullptr;  // used by the *_host entry points
  uint32_t* h_flag = nullptr;         // pinned scratch for small D2H reads
  // Which stream inserts come from.  A lookup launched on the SAME stream is ordered behind them; one launched on another
  // stream may run beside an insert and must confirm its misses (rowops.cuh probe_lane_confirm_miss).  Sticky once two
  // different streams have been seen.
  cudaStream_t insert_stream = nullptr;
  bool any_insert = false, confirm_always = false;
  void note_insert(cudaStream_t s) {
    if (any_insert && insert_stream != s) confirm_always = true;
    insert_stream = s;
    any_insert = true;
  }
  bool lookup_must_confirm(cudaStream_t s) const { return confirm_always || (any_insert && insert_stream != s); }
};

// one reusable grouping of a batch (see bwd.cu "Owner grouping")
struct mono_grouping {
  int device = 0;
  mono::DevBuf ws;
  mono::ClaimSet claim_set;
  int64_t M = 0;
  int dim = 0;
  mono::BwdScratch plan{};       // views into ws, valid after build() (plan.sorted != nullptr)
  uint32_t* h_counts = nullptr;  // pinned: per-owner distinct counts [256] + overflow flag
  cudaStream_t side = nullptr;   // carries the early counts copy while the sort runs on the caller's stream
  cudaEvent_t ev_claimed = nullptr, ev_copied = nullptr;
  // the sharded step over parts: the concatenated FIDs of the parts, and the occurrence map of their gradient rows
  mono::DevBuf fids_cat, occ_map;
};

// ---- NVLink peer window (peer.cu) ----------------------------------------------------------------
namespace mono {
constexpr int kMaxPeers = 16;
constexpr size_t kPeerFlagBytes = 4096;  // head of every window: arrival flags written by the peers

// By-value kernel argument of the push kernels: item i of a list partitioned into `n` consecutive
// parts goes to base[r] + (i - start[r]) * item_bytes, r = the part holding i.  base[r] points into
// rank r's window (a peer mapping of it), already offset to where this rank's items begin there.
struct PeerOut {
  char* base[kMaxPeers];
  int64_t start[kMaxPeers + 1];
  int n;
  const uint32_t* cnt_dev;  // optional: the part sizes live on the device (start[] is then ignored)
};
#ifdef __CUDACC__
// Part boundaries (from the host-side start[] or as the prefix of the device counts) and part bases into shared
// memory; every thread of the block must call it (it ends with a barrier).  s_start[kMaxPeers + 1], s_base[kMaxPeers].
__device__ __forceinline__ void peer_starts(const PeerOut& po, int64_t* s_start, char** s_base = nullptr) {
  if (po.n == 0) return;  // uniform: no peer output
  if (threadIdx.x == 0) {
    int64_t run = 0;
    for (int r = 0; r <= kMaxPeers; ++r) {
      s_start[r] = po.cnt_dev ? run : po.start[r];
      if (po.cnt_dev && r < po.n) run += po.cnt_dev[r];
    }
  }
  if (s_base && threadIdx.x < kMaxPeers) s_base[threadIdx.x] = po.base[threadIdx.x];
  __syncthreads();
}
__device__ __forceinline__ int peer_part(const int64_t* __restrict__ start, int n, int64_t i) {
  int r = 0;
#pragma unroll
  for (int q = 1; q < kMaxPeers; ++q)
    if (q < n && i >= start[q]) r = q;
  return r;
}
#endif
}  // namespace mono

struct mono_peer {
  int device = 0, world = 1, rank = 0;
  size_t bytes = 0;                      // data bytes of every rank's window (after the flag page)
  char* local = nullptr;                 // this rank's window (cudaMalloc: flag page + data)
  char* base[mono::kMaxPeers] = {};      // base[r]: rank r's window as mapped into this process
  bool attached = false;
  uint64_t seq = 0;                      // barrier sequence number (same on every rank)
  uint64_t phase_seq[4] = {0, 0, 0, 0};  // sequence numbers of the directional flags (peer_signal / peer_wait)
};

namespace mono {
struct XWin {  // the exchange as the kernels see it (by value)
  char* base[kMaxPeers];   // base[r]: rank r's window as mapped here (flag page first)
  int N, me, D;
  int64_t C;               // capacity of one (owner, source) sub-region, in items
  int64_t off_ids[2], off_rows, off_grads;  // byte offsets of the regions behind the flag page
  __device__ __forceinline__ uint64_t* flags(int r) const { return reinterpret_cast<uint64_t*>(base[r]); }
  __device__ __forceinline__ int64_t* ids_in(int r, int par, int src) const {
    return reinterpret_cast<int64_t*>(base[r] + kPeerFlagBytes + off_ids[par]) + (int64_t)src * C;
  }
  __device__ __forceinline__ float* rows_in(int r) const {
    return reinterpret_cast<float*>(base[r] + kPeerFlagBytes + off_rows);
  }
  __device__ __forceinline__ float* grads_in(int r, int src) const {
    return reinterpret_cast<float*>(base[r] + kPeerFlagBytes + off_grads) + (int64_t)src * C * D;
  }
};

}  // namespace mono

struct mono_xstep {
  mono_mtable* mt = nullptr;
  int k = 0;
  mono_peer* win = nullptr;
  // two groupings (by step parity): while step e runs, the grouping of batch e + 1 can be built on another stream
  // (mono_xstep_prepare) — it does not depend on the table
  mono_grouping* grouping[2] = {nullptr, nullptr};  // owned
  mono::DevBuf uniq[2], offs[2];                     // bucketed unique list, per-occurrence row offsets
  mono::DevBuf fids_cat;                             // forward over parts: the parts' concatenated FIDs
  cudaEvent_t ev_prep[2] = {nullptr, nullptr};       // grouping [slot] built (recorded on the prepare stream)
  cudaEvent_t ev_bwd[2] = {nullptr, nullptr};        // backward of the step that used grouping [slot] enqueued
  bool bwd_recorded[2] = {false, false};
  uint64_t prep_seq = 0;                             // step the prepared grouping belongs to (0 = none)
  const int64_t* prep_fids = nullptr;
  int64_t prep_m = 0;
  int64_t C = 0;
  int N = 1, me = 0, D = 0;
  mono::XWin w{};
  uint64_t step = 0;               // steps started (forward calls)
  uint64_t timeout_ns = 0;
  mono::DevBuf ws;                 // owner-side scratch
  mono::ClaimSet miss_set;
  int64_t last_m = 0, last_rows = 0;
  bool fwd_done = false;
};


namespace mono {

mono_peer* peer_create(int device, int world, int rank, size_t bytes);
void peer_destroy(mono_peer* p);
void peer_detach(mono_peer* p);
void peer_handle(mono_peer* p, void* out64);
void peer_attach(mono_peer* p, const void* handles);
void peer_barrier(mono_peer* p, cudaStream_t s);
void peer_put(mono_peer* p, int64_t region_off, const int64_t* dst_off, const void* src,
              const int64_t* src_off, const int64_t* nbytes, cudaStream_t s);
void peer_get(mono_peer* p, int64_t region_off, const int64_t* src_off, void* dst, const int64_t* dst_off,
              const int64_t* nbytes, cudaStream_t s);
PeerOut peer_out(mono_peer* p, int64_t region_off, const int64_t* dst_item_off, const int64_t* counts,
                 int64_t item_bytes);
void launch_lookup_push(mono_mtable* mt, int k, const int64_t* ids_dev, int64_t n_total, const PeerOut& po,
                        cudaStream_t s);
// grad_scale (here and in grouping_reduce, xstep_backward): device float, or null; every pooled gradient element is
// multiplied by it in fp32 where the reduce loads it (the scaled_ reduce kernels)
void grouping_reduce_push(mono_grouping* g, const float* pooled_grad, int64_t grad_stride, int grad_col,
                          const int32_t* row_offsets, int64_t n_rows, int pooling, const PeerOut& po,
                          cudaStream_t s, const float* grad_scale = nullptr);

mono_grouping* grouping_create(int device);
void grouping_destroy(mono_grouping* g);  // synchronises the device first
void grouping_build(mono_grouping* g, const int64_t* fids_dev, int64_t M, int N, int dim,
                    int64_t* uniq_out, int32_t* occ_offset_out, int32_t* shard_counts_host,
                    int64_t* n_unique_host, cudaStream_t s);
void grouping_reduce(mono_grouping* g, const float* pooled_grad, int64_t grad_stride, int grad_col,
                     const int32_t* row_offsets, int64_t n_rows, int pooling, float* out_rows, cudaStream_t s,
                     const float* grad_scale = nullptr);

// The sharded step over parts of ONE table k (bwd.cu): the occurrences of all parts are one batch, part order then
// occurrence order.  check_shard_parts checks the parts before any device work (grads: their rows are gradient rows
// the reduce reads, bf16 ones when bf16) and returns the occurrence count.
int64_t check_shard_parts(const char* who, mono_mtable* mt, int k, const mono_pool_part* parts, int n_parts,
                          bool grads, bool bf16);
// the concatenated FIDs of the parts: one part's FIDs as they are, else written into buf (one launch)
const int64_t* shard_parts_fids(mono_mtable* mt, int k, const mono_pool_part* parts, int n_parts, int64_t M,
                                DevBuf& buf, cudaStream_t s);
// grouping_build over the concatenated FIDs of the parts
void grouping_build_parts(mono_grouping* g, mono_mtable* mt, int k, const mono_pool_part* parts, int n_parts, int N,
                          int64_t* uniq_out, int32_t* occ_offset_out, int32_t* shard_counts_host,
                          int64_t* n_unique_host, cudaStream_t s);
// grouping_reduce (po.n == 0: into out_rows) or grouping_reduce_push (po.n > 0) with the parts' rows as the gradient
// source (bf16: bf16 rows), through the parts occurrence map: one more launch than the reduce itself
void grouping_reduce_parts(mono_grouping* g, mono_mtable* mt, int k, const mono_pool_part* parts, int n_parts,
                           bool bf16, float* out_rows, const PeerOut& po, cudaStream_t s,
                           const float* grad_scale = nullptr);

// xstep.cu
int64_t xstep_window_bytes(int N, int64_t C, int D);
mono_xstep* xstep_create(mono_mtable* mt, int k, mono_peer* win, int64_t cap_pair);
void xstep_destroy(mono_xstep* x);
void xstep_prepare(mono_xstep* x, const int64_t* fids_next_dev, int64_t M, cudaStream_t s2);
void xstep_forward(mono_xstep* x, const int64_t* fids_dev, int64_t M, const int32_t* row_offsets, int64_t n_rows,
                   int pooling, float* out, int64_t out_stride, int out_col, cudaStream_t s);
void xstep_backward(mono_xstep* x, const float* pooled_grad, int64_t grad_stride, int grad_col,
                    const int32_t* row_offsets, int pooling, const float* lr_host, int64_t update_time, cudaStream_t s,
                    const float* grad_scale = nullptr);
// the step over parts of the xstep's table (bf16: the parts' rows are bf16; forward: output rows, backward: gradients)
void xstep_forward_parts(mono_xstep* x, const mono_pool_part* parts, int n_parts, bool bf16, cudaStream_t s);
void xstep_backward_parts(mono_xstep* x, const mono_pool_part* parts, int n_parts, bool bf16, const float* lr_host,
                          int64_t update_time, cudaStream_t s, const float* grad_scale = nullptr);

// table.cu
void table_init(mono_mtable* mt, HostTable& t, const mono_table_cfg& cfg, cudaStream_t s);
void table_free(HostTable& t);
void table_set_filter(mono_mtable* mt, int k, uint64_t capacity, uint32_t default_thr, const uint32_t* slots,
                      const uint32_t* thrs, int n_slots, cudaStream_t s);
void upload_tables(mono_mtable* mt, cudaStream_t s);
// make room for n_new more keys in table k (grows row slabs / rehashes buckets when needed)
void ensure_capacity(mono_mtable* mt, int k, uint64_t n_new, cudaStream_t s);
void request_snapshot(mono_mtable* mt, int k, cudaStream_t s);
// the table's counter words as they are (no error check); read_counters_sync also raises on every error bit
void copy_counters_sync(mono_mtable* mt, int k, cudaStream_t s, uint32_t* out /*kNumCtrs*/);
void read_counters_sync(mono_mtable* mt, int k, cudaStream_t s, uint32_t* out /*kNumCtrs*/);
void evict_table(mono_mtable* mt, int k, int64_t max_update_time, cudaStream_t s);
int64_t export_rows(mono_mtable* mt, int k, int64_t* cursor, int64_t max_n, int64_t* ids_out,
                    float* entry_out, cudaStream_t s);

// ops.cu
enum UpsertOp { kOpOptimize = 0, kOpAssign = 1, kOpAssignAdd = 2, kOpReinit = 3, kOpRestore = 4 };
// T: element type of the output rows, float or __half (mono_mtable_lookup_f16: each element rounded once to fp16)
template <typename T>
void launch_lookup(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const int64_t* ids_dev,
                   int64_t n_total, T* out_dev, cudaStream_t s);
void launch_lookup_pool(mono_mtable* mt, int k, const int64_t* fids_dev, const int32_t* row_offsets,
                        int64_t n_rows, int pooling, float* out, int64_t out_stride, int out_col,
                        cudaStream_t s);
void launch_contains(mono_mtable* mt, int k, const int64_t* ids, int64_t n, uint8_t* out,
                     cudaStream_t s);
void launch_lookup_entry(mono_mtable* mt, int k, const int64_t* ids, int64_t n, float* out,
                         cudaStream_t s);
// generic find-or-insert + apply over segments.  ids may contain duplicates unless `unique`.
void run_upsert(mono_mtable* mt, UpsertOp op, const CallSeg* h_segs, int nsegs,
                const int64_t* ids_dev, int64_t n_total, const float* vals_dev,
                const float* lr_host, int n_lr, int64_t update_time, bool unique, bool dedup_sum,
                int32_t* status_dev, cudaStream_t s);

// optimize over `ngroups` groups of segments; ids unique inside a group, groups applied in order
void run_upsert_groups(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const int64_t* group_begin,
                       int ngroups, const int64_t* ids_dev, const float* vals_dev, const float* lr_host,
                       int n_lr, int64_t update_time, cudaStream_t s);

// grad_scale: as run_pool_backward_parts' (the one table has no FIRSTN rows)
void run_pool_backward(mono_mtable* mt, int k, const int64_t* fids_dev, int64_t n_fids,
                       const int32_t* row_offsets, int64_t n_rows, int pooling,
                       const float* pooled_grad, int64_t grad_stride, int grad_col,
                       const float* lr_host, int64_t update_time, cudaStream_t s,
                       const float* grad_scale = nullptr);

// A FIRSTN part's sequence length (max_seq_len is read for FIRSTN parts only): L >= 1 and n_rows * L <= 2^31
inline void check_firstn(const char* who, const mono_pool_part& p) {
  if (p.pooling != MONO_POOL_FIRSTN) return;
  if (p.max_seq_len < 1) throw ArgError(std::string(who) + ": FIRSTN needs max_seq_len >= 1");
  if (p.n_rows > ((int64_t)1 << 31) / p.max_seq_len) throw ArgError(std::string(who) + ": n_rows * max_seq_len over 2^31");
}

// bf16: the parts' rows are bfloat16 (the *_parts_bf16 calls)
void run_lookup_pool_parts(mono_mtable* mt, const mono_pool_part* parts, int n_parts, cudaStream_t s, bool bf16);
// grad_scale (device float, or null): every gradient row is multiplied by it in fp32 where it is loaded (the scaled_
// kernels; null runs the unscaled kernels)
void run_pool_backward_parts(mono_mtable* mt, const mono_pool_part* parts, int n_parts, const float* lr_host,
                             int64_t update_time, cudaStream_t s, bool bf16, const float* grad_scale = nullptr);

void run_scatter_rows(int device, const int32_t* offs_dev, int64_t M, int dim, const int32_t* row_offsets,
                      int64_t n_rows, int pooling, const float* pooled_grad, int64_t grad_stride,
                      int grad_col, float* out_rows, int64_t total_floats, cudaStream_t s, bool bf16 = false,
                      const float* grad_scale = nullptr);

// bwd.cu: the backward's stable LSD radix sort of (keys[i], i) over `bits` key bits (keys < 2^bits), stand-alone in
// key_sort_bytes(M, bits) bytes of scratch at ws; runs: also the ordered run list (the returned regions' run_start
// [n_runs + 1] and *n_runs).  *sorted receives the sorted {key, position} pairs.
size_t key_sort_bytes(int64_t M, int bits);
SortWs key_sort(char* ws, const uint32_t* keys, int64_t M, int bits, bool runs, const uint2** sorted, cudaStream_t s);

// dedup.cu
void run_reorder(int device, const int64_t* ids_dev, const int64_t* id_split_host, int K, int N,
                 const int32_t* dims_host, int rank0_empty, int64_t* output_dev, int32_t* sizes_dev,
                 int32_t* fused_emb_offset_dev, int32_t* shard_sizes_host,
                 int32_t* sharded_slot_sizes_host, int64_t* n_unique_host, int32_t* n_unique_dev,
                 cudaStream_t s);
// The version-5 outputs of mono_sharding_sparse_fids_v5, written on the device after the v3/v4 outputs:
// row_splits_size[k * N + n] = features of table k + 1, emb_size[k * N + n] = floats of list (table k, shard n) and
// sizes = {nfl_size, feature_size, fid_size, batch_size}.
struct ShardingV5 {
  int32_t batch_size;
  int32_t* row_splits_size;
  int32_t* emb_size;
  int32_t* sizes;
};
void run_sharding(int device, const int64_t* fids_dev, const int64_t* row_splits_dev,
                  const mono_sharding_feature* feats, int F, int K, int N, int unique, int64_t* fid_list_dev,
                  uint64_t* fid_offset_dev, int32_t* feature_offset_dev, uint32_t* nfl_offset_dev,
                  int64_t* row_splits_out_dev, int32_t* table_len_dev, int32_t* shard_len_dev, int32_t* emb_len_dev,
                  int32_t* bad_row_splits_dev, int32_t* table_len_host, cudaStream_t s,
                  const ShardingV5* v5 = nullptr);
// mono_normalize_merged_split: merge_num row splits laid end to end, each restarting at 0, joined into one
void run_normalize_merged_split(int device, const int64_t* row_split_dev, int64_t split_num,
                                const int32_t* row_split_size_dev, int64_t merge_num, int64_t* out_dev,
                                int32_t* bad_dev, cudaStream_t s);

// the async parameter-server worker path (mono_unique_key_with_value_and_offset, mono_ragged_split_by_indices)
void run_unique_offset(int device, const int64_t* key_dev, const int64_t* key_split_host, int K,
                       const int32_t* dims_host, int64_t* unique_key_dev, int64_t* unique_key_split_dev,
                       int64_t* value_offset_dev, int64_t* value_offset_split_dev, int64_t* value_len_host,
                       int64_t* unique_key_split_host, cudaStream_t s);
void run_ragged_split(int device, const int64_t* indices_dev, const int64_t* values_dev, int64_t cap,
                      const int64_t* num_split_dev, int K, int S, int64_t* values_out_dev, int64_t* pos_out_dev,
                      int64_t* row_splits_out_dev, int64_t* split_offsets_dev, int32_t* bad_dev,
                      int64_t* row_splits_host, cudaStream_t s);

// layout.cu; T: element type of the pooled rows, float or __nv_bfloat16
template <typename T>
void launch_gather_pool(const float* fused_emb, const int32_t* emb_offset, const int32_t* row_offsets,
                        int64_t n_rows, int dim, int pooling, T* out, int64_t out_stride, int out_col,
                        cudaStream_t s);
// the pooling of received rows over the parts of table k of a sharded step (occ_offset: the grouping's row offset of
// every occurrence of the concatenated parts): one launch per distinct kernel among the parts
template <typename T>
void launch_gather_pool_parts(mono_mtable* mt, int k, const float* rows_in, const int32_t* occ_offset,
                              const mono_pool_part* parts, int n_parts, cudaStream_t s);
template <typename T>
void launch_gather_pool_grad(const T* pooled_grad, int64_t grad_stride, int grad_col, const int32_t* emb_offset,
                             const int32_t* row_offsets, int64_t n_rows, int dim, int pooling, float* grad_fused,
                             cudaStream_t s, const float* grad_scale = nullptr);
void check_layout_tasks(const mono_slice_task* tasks, int n_tasks, int total_nfl);
void launch_layout(bool backward, float* const* emb_ptrs_dev, const int32_t* emb_strides_dev,
                   int n_emb, const uint64_t* fid_offset, int64_t total_fid,
                   const int32_t* feature_offset, int total_feature, const uint32_t* nfl_offset,
                   int total_nfl, int batch_size, const mono_slice_task* tasks_host, int n_tasks,
                   float* const* out_ptrs_dev, cudaStream_t s, bool bf16 = false, const float* grad_scale = nullptr,
                   bool f16_in = false);
// f16_in (forward only): emb_ptrs_dev point at __half rows, widened exactly where they are loaded (the f16in_ kernels)
// mono_round_to_f16: dst[i] = fp16 round-to-nearest-even of src[i]
void launch_round_to_f16(const float* src, int64_t n, __half* dst, cudaStream_t s);
// mono_reduce_and_split[_grad]; T: element type of the slice rows.  grad_scale (backward only; device float, or
// null): every slice gradient element is multiplied by it in fp32 where it is loaded (the scaled_ kernels)
void check_reduce_split(const mono_reduce_feature* feats, int n_features);
template <typename T>
void launch_reduce_split(bool backward, const mono_reduce_feature* feats, int n_features, int32_t* bad_splits_dev,
                         cudaStream_t s, const float* grad_scale = nullptr);

// mono_fill_with_offset_map (grad = false: src = the server's rows, dst = the value buffer) and
// mono_fill_with_offset_map_grad (grad = true: src = the value buffer's gradient, dst = the server's row gradients).
// f16: the server's rows (src, or dst with grad) are __half behind the float pointer (the _f16 calls); src_len then
// counts fp16 elements.
void run_fill_offset_map(bool grad, int device, const int64_t* pos_dev, const int64_t* pos_split_host, int K,
                         const int32_t* dims_host, const float* src_dev, int64_t src_len,
                         const int64_t* value_offset_dev, const int64_t* value_offset_split_dev, int64_t num_unique,
                         float* dst_dev, int32_t* bad_dev, cudaStream_t s, bool f16 = false);

// clip.cu
void check_global_norm(const mono_norm_tensor* tensors, int n_tensors, float clip_norm, const float* norm_dev,
                       const float* scale_dev);
void launch_global_norm(const mono_norm_tensor* tensors, int n_tensors, float clip_norm, float* norm_dev,
                        float* scale_dev, cudaStream_t s);

}  // namespace mono
