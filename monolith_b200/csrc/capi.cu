// capi.cu — the C ABI declared in include/mono_emb.h.  Thin glue: argument checks, segment
// descriptors, error translation.  No exception crosses the boundary.
#include <algorithm>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include "engine.h"

using namespace mono;

namespace {
thread_local std::string g_last_error;

template <class F>
int guarded(F f) {
  try {
    f();
    return MONO_OK;
  } catch (const ArgError& e) {
    g_last_error = e.what();
    return MONO_ERR_INVALID_ARGUMENT;
  } catch (const CudaError& e) {
    g_last_error = e.what();
    return MONO_ERR_CUDA;
  } catch (const std::bad_alloc& e) {
    g_last_error = e.what();
    return MONO_ERR_RESOURCE_EXHAUSTED;
  } catch (const std::exception& e) {
    g_last_error = e.what();
    return MONO_ERR_INTERNAL;
  }
}

void require(bool c, const char* msg) {
  if (!c) throw ArgError(msg);
}

// Every entry point that touches a table's device state or scratch takes the handle's lock for the duration of
// the (asynchronous) enqueue and selects its device: host threads may share one handle, as the reference's
// interface allows (embedding_hash_table_interface.h:32-33); recursive because the *_host variants nest.
struct HandleGuard {
  std::unique_lock<std::recursive_mutex> lk;
  explicit HandleGuard(const mono_mtable_t* t) : lk(t->mu) { MONO_CUDA(cudaSetDevice(t->device)); }
};

// segments of a per-table call (id_split over K tables; values laid out table after table)
std::vector<CallSeg> table_segs(const mono_mtable_t* t, const int64_t* id_split, int width_extra,
                                int64_t* n_total, int* n_lr) {
  const int K = (int)t->tables.size();
  require(id_split != nullptr, "id_split is null");
  require(id_split[0] == 0, "id_split must start at 0");
  std::vector<CallSeg> segs;
  int64_t voff = 0;
  int lroff = 0;
  for (int k = 0; k < K; ++k) {
    // ref: MismatchLength / ordering checks, multi_hash_table_update_op.cc:34-45
    require(id_split[k + 1] >= id_split[k], "id_split must be non-decreasing");
    const int64_t n = id_split[k + 1] - id_split[k];
    const int width = width_extra ? t->tables[k].dim + t->tables[k].state_dim + 2 : t->tables[k].dim;
    if (n > 0) {
      CallSeg s;
      s.id_begin = id_split[k];
      s.id_end = id_split[k + 1];
      s.val_off = voff;
      s.table = k;
      s.lr_off = lroff;
      segs.push_back(s);
    }
    voff += n * width;
    lroff += t->tables[k].slices;
  }
  *n_total = id_split[K];
  if (n_lr) *n_lr = lroff;
  return segs;
}

void fused_offsets(const mono_mtable_t* t, const int32_t* slot_size, int N, int32_t* emb_splits,
                   int32_t* key_offsets, int32_t* emb_offsets) {
  // ref: ComputeFusedOffsets<false>, RT/hash_table/utils.h:28-61
  const int K = (int)t->tables.size();
  int total_embs = 0, prev = 0;
  key_offsets[0] = emb_offsets[0] = 0;
  for (int s = 0; s < N; ++s) {
    for (int k = 0; k < K; ++k) {
      const int idx = K * s + k;
      require(slot_size[idx] >= 0, "negative fused_slot_size");
      const int seg = t->tables[k].dim * slot_size[idx];
      total_embs += seg;
      key_offsets[idx + 1] = key_offsets[idx] + slot_size[idx];
      emb_offsets[idx + 1] = emb_offsets[idx] + seg;
    }
    if (emb_splits) emb_splits[s] = total_embs - prev;
    prev = total_embs;
  }
}

void ensure_pinned(void** p, size_t* cap, size_t bytes) {
  if (bytes <= *cap) return;
  if (*p) cudaFreeHost(*p);
  *p = nullptr;
  size_t ncap = bytes + bytes / 4 + 4096;
  MONO_CUDA(cudaHostAlloc(p, ncap, cudaHostAllocDefault));
  *cap = ncap;
}
}  // namespace

extern "C" {

const char* mono_last_error(void) { return g_last_error.c_str(); }
int32_t mono_abi_version(void) { return MONO_EMB_ABI_VERSION; }
int64_t mono_kernel_launch_count(void) { return g_launches.load(); }

int mono_set_option(const char* name, int64_t value) {
  return guarded([&] {
    require(name != nullptr, "set_option: null name");
    if (std::strcmp(name, "lookup_tma") == 0) g_opt_lookup_tma.store(value != 0 ? 1 : 0);
    else if (knob_id(name) >= 0) knob_set(knob_id(name), (int)value);
    else throw ArgError(std::string("unknown option: ") + name);
  });
}
int64_t mono_get_option(const char* name) {
  if (name && std::strcmp(name, "lookup_tma") == 0) return g_opt_lookup_tma.load();
  if (knob_id(name) >= 0) return knob(knob_id(name));
  return -1;
}

int64_t mono_bench_tower_scratch_floats(void) { return tower_scratch_floats(); }
int mono_bench_tower_grad(const float* pooled, int64_t batch, const float* labels, const void* w1_bf16,
                          const void* w2_bf16, float* grad_out, float* loss_out, float* scratch,
                          int64_t scratch_floats, void* stream) {
  return guarded([&] {
    require(pooled && labels && w1_bf16 && w2_bf16 && grad_out && loss_out && scratch, "bench_tower_grad: null argument");
    require(batch >= 0 && scratch_floats >= tower_scratch_floats(), "bench_tower_grad: scratch too small");
    tower_grad(pooled, batch, labels, w1_bf16, w2_bf16, grad_out, loss_out, scratch, (cudaStream_t)stream);
  });
}

int mono_mtable_create(const mono_table_cfg* cfgs, int32_t n_tables, int32_t device,
                       mono_mtable_t** out) {
  return guarded([&] {
    require(cfgs && out && n_tables > 0, "mono_mtable_create: bad arguments");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
      throw CudaError("no CUDA device: this engine has no CPU fallback");
    require(device >= 0 && device < ndev, "mono_mtable_create: bad device ordinal");
    MONO_CUDA(cudaSetDevice(device));
    // stream-ordered allocations keep their memory (tables live for the whole job)
    cudaMemPool_t pool;
    MONO_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thr = UINT64_MAX;
    MONO_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr));
    auto mt = new mono_mtable();
    try {
      mt->device = device;
      std::vector<int> order(n_tables);
      std::iota(order.begin(), order.end(), 0);
      for (int i = 0; i < n_tables; ++i) require(cfgs[i].name != nullptr, "table name is null");
      std::sort(order.begin(), order.end(), [&](int a, int b) {
        return std::string(cfgs[a].name) < std::string(cfgs[b].name);
      });
      for (int i = 1; i < n_tables; ++i)
        require(std::string(cfgs[order[i]].name) != cfgs[order[i - 1]].name, "duplicate table name");
      mt->ring.init();
      MONO_CUDA(cudaStreamCreateWithFlags(&mt->own_stream, cudaStreamNonBlocking));
      MONO_CUDA(cudaHostAlloc((void**)&mt->h_flag, 256, cudaHostAllocDefault));
      MONO_CUDA(cudaMalloc((void**)&mt->d_tables, sizeof(TableDev) * n_tables));
      MONO_CUDA(cudaMalloc((void**)&mt->zero_row, sizeof(float) * 128));
      MONO_CUDA(cudaMemset(mt->zero_row, 0, sizeof(float) * 128));
      mt->tables.resize(n_tables);
      for (int i = 0; i < n_tables; ++i) table_init(mt, mt->tables[i], cfgs[order[i]], 0);
      MONO_CUDA(cudaDeviceSynchronize());
      mt->tables_dirty = true;
    } catch (...) {
      mono_mtable_destroy(mt);
      throw;
    }
    *out = mt;
  });
}

int mono_mtable_destroy(mono_mtable_t* t) {
  if (!t) return MONO_OK;
  cudaSetDevice(t->device);
  cudaDeviceSynchronize();
  for (auto& tb : t->tables) table_free(tb);
  if (t->d_tables) cudaFree(t->d_tables);
  if (t->zero_row) cudaFree(t->zero_row);
  t->ring.destroy();
  t->ws_miss.release(); t->ws_a.release(); t->ws_b.release(); t->ws_c.release(); t->claim_set.release();
  t->ws_d.release(); t->ws_e.release(); t->ws_host_in.release(); t->ws_host_out.release();
  if (t->pinned_in) cudaFreeHost(t->pinned_in);
  if (t->pinned_out) cudaFreeHost(t->pinned_out);
  if (t->h_flag) cudaFreeHost(t->h_flag);
  if (t->own_stream) cudaStreamDestroy(t->own_stream);
  delete t;
  return MONO_OK;
}

int32_t mono_mtable_num_tables(const mono_mtable_t* t) { return (int32_t)t->tables.size(); }
int32_t mono_mtable_table_index(const mono_mtable_t* t, const char* name) {
  for (size_t i = 0; i < t->tables.size(); ++i)
    if (t->tables[i].name == name) return (int32_t)i;
  return -1;
}
const char* mono_mtable_table_name(const mono_mtable_t* t, int32_t k) {
  if (k < 0 || k >= (int)t->tables.size()) return nullptr;
  return t->tables[k].name.c_str();
}
int32_t mono_mtable_dim(const mono_mtable_t* t, int32_t k) { return t->tables[k].dim; }
int32_t mono_mtable_slice_size(const mono_mtable_t* t, int32_t k) { return t->tables[k].slices; }
int32_t mono_mtable_state_floats(const mono_mtable_t* t, int32_t k) { return t->tables[k].state_dim; }
int64_t mono_mtable_max_update_ts(const mono_mtable_t* t, int32_t k) { return t->tables[k].max_update_ts; }

int mono_mtable_size(mono_mtable_t* t, int32_t k, int64_t* out_size, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    uint32_t c[kNumCtrs];
    read_counters_sync(t, k, (cudaStream_t)stream, c);
    *out_size = c[kCtrSize];
  });
}

int mono_mtable_lookup(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                       float* emb_out_dev, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    int64_t n_total = 0;
    auto segs = table_segs(t, id_split_host, 0, &n_total, nullptr);
    if (segs.empty()) return;
    launch_lookup(t, segs.data(), (int)segs.size(), ids_dev, n_total, emb_out_dev, (cudaStream_t)stream);
  });
}

int mono_mtable_fused_offsets(const mono_mtable_t* t, const int32_t* fused_slot_size_host,
                              int32_t num_shards, int32_t* emb_splits_host,
                              int32_t* id_offsets_host, int32_t* emb_offsets_host) {
  return guarded([&] {
    require(num_shards > 0 && fused_slot_size_host && id_offsets_host && emb_offsets_host,
            "fused_offsets: bad arguments");
    fused_offsets(t, fused_slot_size_host, num_shards, emb_splits_host, id_offsets_host, emb_offsets_host);
  });
}

static std::vector<CallSeg> fused_segs(const mono_mtable_t* t, const int32_t* slot_size, int N,
                                       int shard_begin, int shard_end, int64_t* n_total) {
  const int K = (int)t->tables.size();
  std::vector<int32_t> ko(N * K + 1), eo(N * K + 1);
  fused_offsets(t, slot_size, N, nullptr, ko.data(), eo.data());
  std::vector<CallSeg> segs;
  for (int s = shard_begin; s < shard_end; ++s) {
    int lroff = 0;
    for (int k = 0; k < K; ++k) {
      const int idx = s * K + k;
      if (slot_size[idx] > 0) {
        CallSeg sg;
        sg.id_begin = ko[idx];
        sg.id_end = ko[idx + 1];
        sg.val_off = eo[idx];
        sg.table = k;
        sg.lr_off = lroff;
        segs.push_back(sg);
      }
      lroff += t->tables[k].slices;
    }
  }
  *n_total = ko[N * K];
  return segs;
}

int mono_mtable_fused_lookup(mono_mtable_t* t, const int64_t* ids_dev,
                             const int32_t* fused_slot_size_host, int32_t num_shards,
                             int64_t /*req_time*/, float* emb_out_dev, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    require(num_shards > 0 && fused_slot_size_host, "fused_lookup: bad arguments");
    int64_t n_total = 0;
    auto segs = fused_segs(t, fused_slot_size_host, num_shards, 0, num_shards, &n_total);
    if (segs.empty()) return;
    launch_lookup(t, segs.data(), (int)segs.size(), ids_dev, n_total, emb_out_dev, (cudaStream_t)stream);
  });
}

int mono_mtable_contains(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                         uint8_t* out_dev, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    launch_contains(t, k, ids_dev, n, out_dev, (cudaStream_t)stream);
  });
}

int mono_mtable_lookup_pool(mono_mtable_t* t, int32_t k, const int64_t* fids_dev,
                            const int32_t* row_offsets_dev, int64_t n_rows, int32_t pooling,
                            float* out_dev, int64_t out_stride, int32_t out_col, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    launch_lookup_pool(t, k, fids_dev, row_offsets_dev, n_rows, pooling, out_dev, out_stride, out_col,
                       (cudaStream_t)stream);
  });
}

int mono_mtable_pool_backward(mono_mtable_t* t, int32_t k, const int64_t* fids_dev, int64_t n_fids,
                              const int32_t* row_offsets_dev, int64_t n_rows, int32_t pooling,
                              const float* pooled_grad_dev, int64_t grad_stride, int32_t grad_col,
                              const float* learning_rate_host, int64_t update_time,
                              int64_t /*global_step*/, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    require(fids_dev && pooled_grad_dev && learning_rate_host, "pool_backward: null argument");
    require(row_offsets_dev != nullptr || n_rows == n_fids, "pool_backward: n_rows must equal n_fids without offsets");
    HandleGuard hg_(t);
    run_pool_backward(t, k, fids_dev, n_fids, row_offsets_dev, n_rows, pooling, pooled_grad_dev, grad_stride,
                      grad_col, learning_rate_host, update_time, (cudaStream_t)stream);
  });
}

int mono_mtable_lookup_pool_parts(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                  void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    run_lookup_pool_parts(t, parts_host, n_parts, (cudaStream_t)stream, false);
  });
}

int mono_mtable_pool_backward_parts(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                    const float* learning_rate_host, int64_t update_time,
                                    int64_t /*global_step*/, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    run_pool_backward_parts(t, parts_host, n_parts, learning_rate_host, update_time, (cudaStream_t)stream, false);
  });
}

int mono_mtable_lookup_pool_parts_bf16(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                       void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    run_lookup_pool_parts(t, parts_host, n_parts, (cudaStream_t)stream, true);
  });
}

int mono_mtable_pool_backward_parts_bf16(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                         const float* learning_rate_host, int64_t update_time,
                                         int64_t /*global_step*/, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    run_pool_backward_parts(t, parts_host, n_parts, learning_rate_host, update_time, (cudaStream_t)stream, true);
  });
}

int mono_mtable_optimize(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                         const float* grads_dev, const float* learning_rate_host,
                         int64_t update_time, int64_t /*global_step*/, uint32_t flags, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    require(learning_rate_host != nullptr, "learning_rate is null");
    int64_t n_total = 0;
    int n_lr = 0;
    auto segs = table_segs(t, id_split_host, 0, &n_total, &n_lr);
    if (segs.empty()) return;
    run_upsert(t, kOpOptimize, segs.data(), (int)segs.size(), ids_dev, n_total, grads_dev,
               learning_rate_host, n_lr, update_time, flags & MONO_FLAG_IDS_UNIQUE,
               flags & MONO_FLAG_DEDUP_SUM, nullptr, (cudaStream_t)stream);
  });
}

int mono_mtable_fused_optimize(mono_mtable_t* t, const int64_t* ids_dev,
                               const int32_t* fused_slot_size_host, const float* grads_dev,
                               const int32_t* id_offsets_host, const int32_t* grad_offsets_host,
                               const float* learning_rate_host, int64_t req_time,
                               int64_t /*global_step*/, int32_t num_shards, uint32_t flags,
                               void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    require(num_shards > 0 && fused_slot_size_host && learning_rate_host, "fused_optimize: bad arguments");
    const int K = (int)t->tables.size();
    if (id_offsets_host && grad_offsets_host) {  // must agree with ComputeFusedOffsets
      std::vector<int32_t> ko(num_shards * K + 1), eo(num_shards * K + 1);
      fused_offsets(t, fused_slot_size_host, num_shards, nullptr, ko.data(), eo.data());
      require(std::equal(ko.begin(), ko.end(), id_offsets_host) &&
                  std::equal(eo.begin(), eo.end(), grad_offsets_host),
              "id_offsets / grad_offsets do not match fused_slot_size");
    }
    int n_lr = 0;
    for (auto& tb : t->tables) n_lr += tb.slices;
    if ((flags & MONO_FLAG_IDS_UNIQUE) && !(flags & MONO_FLAG_DEDUP_SUM) && num_shards > 1) {
      // ids unique inside every shard: one resolve pass for the whole call, then the shards' rows are
      // applied in shard order (same result as the loop below, without per-shard launch trains)
      int64_t n_total = 0;
      auto segs = fused_segs(t, fused_slot_size_host, num_shards, 0, num_shards, &n_total);
      if (segs.empty()) return;
      std::vector<int32_t> ko(num_shards * K + 1), eo(num_shards * K + 1);
      fused_offsets(t, fused_slot_size_host, num_shards, nullptr, ko.data(), eo.data());
      std::vector<int64_t> gb(num_shards + 1);
      for (int s = 0; s <= num_shards; ++s) gb[s] = ko[s * K];
      run_upsert_groups(t, segs.data(), (int)segs.size(), gb.data(), num_shards, ids_dev, grads_dev,
                        learning_rate_host, n_lr, req_time, (cudaStream_t)stream);
      return;
    }
    // shard by shard = the reference's single-thread order (multi_hash_table_update_op.cc:286-300)
    for (int s = 0; s < num_shards; ++s) {
      int64_t n_total = 0;
      auto segs = fused_segs(t, fused_slot_size_host, num_shards, s, s + 1, &n_total);
      if (segs.empty()) continue;
      run_upsert(t, kOpOptimize, segs.data(), (int)segs.size(), ids_dev, n_total, grads_dev,
                 learning_rate_host, n_lr, req_time, flags & MONO_FLAG_IDS_UNIQUE,
                 flags & MONO_FLAG_DEDUP_SUM, nullptr, (cudaStream_t)stream);
    }
  });
}

static int assign_like(mono_mtable_t* t, UpsertOp op, const int64_t* ids_dev,
                       const int64_t* id_split_host, const float* values_dev, int64_t update_time,
                       uint32_t flags, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    int64_t n_total = 0;
    auto segs = table_segs(t, id_split_host, 0, &n_total, nullptr);
    if (segs.empty()) return;
    run_upsert(t, op, segs.data(), (int)segs.size(), ids_dev, n_total, values_dev, nullptr, 0,
               update_time, flags & MONO_FLAG_IDS_UNIQUE, false, nullptr, (cudaStream_t)stream);
  });
}

int mono_mtable_assign(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                       const float* values_dev, int64_t update_time, uint32_t flags, void* stream) {
  return assign_like(t, kOpAssign, ids_dev, id_split_host, values_dev, update_time, flags, stream);
}
int mono_mtable_assign_add(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                           const float* values_dev, int64_t update_time, uint32_t flags,
                           void* stream) {
  return assign_like(t, kOpAssignAdd, ids_dev, id_split_host, values_dev, update_time, flags, stream);
}

int mono_mtable_reinitialize(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                             int32_t* status_dev, int64_t update_time, void* stream) {
  return guarded([&] {
    HandleGuard hg_(t);
    require(status_dev != nullptr, "status is null");
    if (n <= 0) return;
    if (k < 0 || k >= (int)t->tables.size()) {  // unknown table: all -1 (update_op.cc:207-214)
      MONO_CUDA(cudaMemsetAsync(status_dev, 0xFF, sizeof(int32_t) * n, (cudaStream_t)stream));
      return;
    }
    CallSeg s;
    s.id_begin = 0;
    s.id_end = n;
    s.val_off = 0;
    s.table = k;
    s.lr_off = 0;
    run_upsert(t, kOpReinit, &s, 1, ids_dev, n, nullptr, nullptr, 0, update_time, false, false,
               status_dev, (cudaStream_t)stream);
  });
}

int mono_mtable_evict(mono_mtable_t* t, int32_t k, int64_t max_update_time, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    evict_table(t, k, max_update_time, (cudaStream_t)stream);
  });
}

int mono_mtable_set_hash_filter(mono_mtable_t* t, int32_t k, int64_t capacity, uint32_t default_threshold,
                                const uint32_t* slot_ids_host, const uint32_t* slot_thresholds_host,
                                int32_t n_slots, void* stream) {
  return guarded([&] {
    require(t != nullptr && k >= 0 && k < (int)t->tables.size(), "bad table index");
    require(capacity > 0, "hash filter capacity must be positive");
    require(n_slots == 0 || (slot_ids_host && slot_thresholds_host), "set_hash_filter: null slot arrays");
    HandleGuard hg_(t);
    table_set_filter(t, k, (uint64_t)capacity, default_threshold, slot_ids_host, slot_thresholds_host, n_slots,
                     (cudaStream_t)stream);
  });
}

int mono_mtable_lookup_entry(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                             float* entry_out_dev, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    launch_lookup_entry(t, k, ids_dev, n, entry_out_dev, (cudaStream_t)stream);
  });
}

int mono_mtable_export(mono_mtable_t* t, int32_t k, int64_t* cursor, int64_t max_n,
                       int64_t* ids_out_dev, float* entry_out_dev, int64_t* n_out, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size() && cursor && n_out && max_n > 0, "export: bad arguments");
    HandleGuard hg_(t);
    *n_out = export_rows(t, k, cursor, max_n, ids_out_dev, entry_out_dev, (cudaStream_t)stream);
  });
}

int mono_mtable_restore_rows(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                             const float* entry_in_dev, void* stream) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    if (n <= 0) return;
    CallSeg s;
    s.id_begin = 0;
    s.id_end = n;
    s.val_off = 0;
    s.table = k;
    s.lr_off = 0;
    run_upsert(t, kOpRestore, &s, 1, ids_dev, n, entry_in_dev, nullptr, 0, 0, false, false, nullptr,
               (cudaStream_t)stream);
  });
}

int mono_mtable_note_update_ts(mono_mtable_t* t, int32_t k, int64_t ts) {
  return guarded([&] {
    require(t && k >= 0 && k < (int)t->tables.size(), "bad table index");
    t->tables[k].max_update_ts = std::max<int64_t>(t->tables[k].max_update_ts, ts);
  });
}

int mono_reorder_by_indices(int32_t device, const int64_t* ids_dev, const int64_t* id_split_host,
                            int32_t num_lists, int32_t num_shards, const int32_t* dims_host,
                            int32_t rank0_empty, int64_t* output_dev, int32_t* sizes_dev,
                            int32_t* fused_emb_offset_dev, int32_t* shard_sizes_host,
                            int32_t* sharded_slot_sizes_host, int64_t* n_unique_host, void* stream) {
  return guarded([&] {
    require(id_split_host && dims_host && output_dev && fused_emb_offset_dev, "reorder: null argument");
    run_reorder(device, ids_dev, id_split_host, num_lists, num_shards, dims_host, rank0_empty,
                output_dev, sizes_dev, fused_emb_offset_dev, shard_sizes_host, sharded_slot_sizes_host,
                n_unique_host, nullptr, (cudaStream_t)stream);
  });
}

int mono_dedup(int32_t device, const int64_t* ids_dev, int64_t n, int64_t* unique_out_dev,
               int32_t* inverse_out_dev, int32_t* n_unique_dev, int64_t* n_unique_host, void* stream) {
  return guarded([&] {
    require(n >= 0 && unique_out_dev && inverse_out_dev, "dedup: bad arguments");
    const int64_t split[2] = {0, n};
    const int32_t dim = 1;
    run_reorder(device, ids_dev, split, 1, 1, &dim, 0, unique_out_dev, nullptr, inverse_out_dev, nullptr,
                nullptr, n_unique_host, n_unique_dev, (cudaStream_t)stream);
  });
}

int mono_grouping_create(int32_t device, mono_grouping_t** out) {
  return guarded([&] {
    require(out != nullptr, "grouping_create: null out");
    MONO_CUDA(cudaSetDevice(device));
    *out = grouping_create(device);
  });
}

int mono_grouping_destroy(mono_grouping_t* g) {
  grouping_destroy(g);
  return MONO_OK;
}

int mono_grouping_build(mono_grouping_t* g, const int64_t* fids_dev, int64_t n_fids, int32_t num_shards,
                        int32_t dim, int64_t* uniq_out_dev, int32_t* occ_offset_out_dev,
                        int32_t* shard_counts_host, int64_t* n_unique_host, void* stream) {
  return guarded([&] {
    // an empty batch may come with a null FID pointer (an empty tensor has no storage)
    require(g && (fids_dev || n_fids == 0) && uniq_out_dev && occ_offset_out_dev && shard_counts_host,
            "grouping_build: null argument");
    grouping_build(g, fids_dev, n_fids, num_shards, dim, uniq_out_dev, occ_offset_out_dev, shard_counts_host,
                   n_unique_host, (cudaStream_t)stream);
  });
}

int mono_grouping_reduce(mono_grouping_t* g, const float* pooled_grad_dev, int64_t grad_stride,
                         int32_t grad_col, const int32_t* row_offsets_dev, int64_t n_rows,
                         int32_t pooling, float* out_rows_dev, void* stream) {
  return guarded([&] {
    require(g && pooled_grad_dev && out_rows_dev, "grouping_reduce: null argument");
    grouping_reduce(g, pooled_grad_dev, grad_stride, grad_col, row_offsets_dev, n_rows, pooling, out_rows_dev,
                    (cudaStream_t)stream);
  });
}

int mono_peer_create(int32_t device, int32_t world, int32_t rank, int64_t bytes, mono_peer_t** out) {
  return guarded([&] {
    require(out != nullptr && bytes >= 0, "mono_peer_create: bad arguments");
    *out = peer_create(device, world, rank, (size_t)bytes);
  });
}

int mono_peer_destroy(mono_peer_t* p) {
  return guarded([&] { peer_destroy(p); });
}

int mono_peer_detach(mono_peer_t* p) {
  return guarded([&] {
    require(p != nullptr, "mono_peer_detach: null argument");
    peer_detach(p);
  });
}

int mono_peer_handle(mono_peer_t* p, void* handle_out_64) {
  return guarded([&] {
    require(p && handle_out_64, "mono_peer_handle: null argument");
    peer_handle(p, handle_out_64);
  });
}

int mono_peer_attach(mono_peer_t* p, const void* handles, int32_t n_handles) {
  return guarded([&] {
    require(p && handles, "mono_peer_attach: null argument");
    require(n_handles == p->world, "mono_peer_attach: one handle per rank");
    peer_attach(p, handles);
  });
}

int mono_peer_local(mono_peer_t* p, void** data_dev_out) {
  return guarded([&] {
    require(p && data_dev_out, "mono_peer_local: null argument");
    *data_dev_out = p->local + kPeerFlagBytes;
  });
}

int mono_peer_barrier(mono_peer_t* p, void* stream) {
  return guarded([&] {
    require(p != nullptr, "mono_peer_barrier: null argument");
    peer_barrier(p, (cudaStream_t)stream);
  });
}

int mono_peer_put(mono_peer_t* p, int64_t region_off, const int64_t* dst_off, const void* src_dev,
                  const int64_t* src_off, const int64_t* nbytes, void* stream) {
  return guarded([&] {
    require(p && dst_off && src_dev && src_off && nbytes, "mono_peer_put: null argument");
    peer_put(p, region_off, dst_off, src_dev, src_off, nbytes, (cudaStream_t)stream);
  });
}

int mono_peer_get(mono_peer_t* p, int64_t region_off, const int64_t* src_off, void* dst_dev,
                  const int64_t* dst_off, const int64_t* nbytes, void* stream) {
  return guarded([&] {
    require(p && src_off && dst_dev && dst_off && nbytes, "mono_peer_get: null argument");
    peer_get(p, region_off, src_off, dst_dev, dst_off, nbytes, (cudaStream_t)stream);
  });
}

int mono_mtable_lookup_push(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, const int64_t* counts,
                            mono_peer_t* p, int64_t region_off, const int64_t* dst_row_off, void* stream) {
  return guarded([&] {
    require(t && counts && p && dst_row_off, "mono_mtable_lookup_push: null argument");
    require(k >= 0 && k < (int)t->tables.size(), "mono_mtable_lookup_push: bad table index");
    require(p->device == t->device, "mono_mtable_lookup_push: window and table on different devices");
    HandleGuard hg_(t);
    const int D = t->tables[k].dim;
    PeerOut po = peer_out(p, region_off, dst_row_off, counts, (int64_t)D * 4);
    const int64_t n = po.start[po.n];
    require(n == 0 || ids_dev != nullptr, "mono_mtable_lookup_push: null ids");
    launch_lookup_push(t, k, ids_dev, n, po, (cudaStream_t)stream);
  });
}

int mono_grouping_reduce_push(mono_grouping_t* g, const float* pooled_grad_dev, int64_t grad_stride,
                              int32_t grad_col, const int32_t* row_offsets_dev, int64_t n_rows,
                              int32_t pooling, const int64_t* shard_counts, mono_peer_t* p,
                              int64_t region_off, const int64_t* dst_row_off, void* stream) {
  return guarded([&] {
    require(g && pooled_grad_dev && shard_counts && p && dst_row_off, "grouping_reduce_push: null argument");
    require(p->device == g->device, "grouping_reduce_push: window and grouping on different devices");
    PeerOut po = peer_out(p, region_off, dst_row_off, shard_counts, (int64_t)g->dim * 4);
    grouping_reduce_push(g, pooled_grad_dev, grad_stride, grad_col, row_offsets_dev, n_rows, pooling, po,
                         (cudaStream_t)stream);
  });
}

int64_t mono_xstep_window_bytes(int32_t world, int64_t cap_pair, int32_t dim) {
  if (world < 1 || world > kMaxPeers || cap_pair <= 0 || dim <= 0) return -1;
  return xstep_window_bytes(world, cap_pair, dim);
}

int mono_xstep_create(mono_mtable_t* t, int32_t k, mono_peer_t* window, int64_t cap_pair, mono_xstep_t** out) {
  return guarded([&] {
    require(t && window && out, "xstep_create: null argument");
    require(k >= 0 && k < (int)t->tables.size(), "xstep_create: bad table index");
    *out = xstep_create(t, k, window, cap_pair);
  });
}

int mono_xstep_destroy(mono_xstep_t* x) {
  return guarded([&] { xstep_destroy(x); });
}

int mono_xstep_prepare(mono_xstep_t* x, const int64_t* fids_next_dev, int64_t n_fids, void* stream2) {
  return guarded([&] {
    require(x && fids_next_dev, "xstep_prepare: null argument");
    HandleGuard hg_(x->mt);
    xstep_prepare(x, fids_next_dev, n_fids, (cudaStream_t)stream2);
  });
}

int mono_xstep_forward(mono_xstep_t* x, const int64_t* fids_dev, int64_t n_fids, const int32_t* row_offsets_dev,
                       int64_t n_rows, int32_t pooling, float* out_dev, int64_t out_stride, int32_t out_col,
                       void* stream) {
  return guarded([&] {
    require(x && fids_dev && out_dev, "xstep_forward: null argument");
    HandleGuard hg_(x->mt);
    xstep_forward(x, fids_dev, n_fids, row_offsets_dev, n_rows, pooling, out_dev, out_stride, out_col,
                  (cudaStream_t)stream);
  });
}

int mono_xstep_backward(mono_xstep_t* x, const float* pooled_grad_dev, int64_t grad_stride, int32_t grad_col,
                        const int32_t* row_offsets_dev, int32_t pooling, const float* lr_host, int64_t update_time,
                        void* stream) {
  return guarded([&] {
    require(x && pooled_grad_dev && lr_host, "xstep_backward: null argument");
    HandleGuard hg_(x->mt);
    xstep_backward(x, pooled_grad_dev, grad_stride, grad_col, row_offsets_dev, pooling, lr_host, update_time,
                   (cudaStream_t)stream);
  });
}

int mono_gather_pool(int32_t device, const float* fused_emb_dev, const int32_t* emb_offset_dev,
                     const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim, int32_t pooling,
                     float* out_dev, int64_t out_stride, int32_t out_col, void* stream) {
  return guarded([&] {
    MONO_CUDA(cudaSetDevice(device));
    require(dim > 0, "dim must be positive");
    launch_gather_pool(fused_emb_dev, emb_offset_dev, row_offsets_dev, n_rows, dim, pooling, out_dev,
                       out_stride, out_col, (cudaStream_t)stream);
  });
}

int mono_gather_pool_grad(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                          int32_t grad_col, const int32_t* emb_offset_dev,
                          const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                          int32_t pooling, float* grad_fused_dev, void* stream) {
  return guarded([&] {
    MONO_CUDA(cudaSetDevice(device));
    require(dim > 0, "dim must be positive");
    launch_gather_pool_grad(pooled_grad_dev, grad_stride, grad_col, emb_offset_dev, row_offsets_dev,
                            n_rows, dim, pooling, grad_fused_dev, (cudaStream_t)stream);
  });
}

int mono_scatter_grad_rows(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                           int32_t grad_col, const int32_t* emb_offset_dev, int64_t n_occurrences,
                           const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                           int32_t pooling, float* grad_fused_dev, int64_t total_floats,
                           void* stream) {
  return guarded([&] {
    require(pooled_grad_dev && emb_offset_dev && grad_fused_dev, "scatter_grad_rows: null argument");
    require(row_offsets_dev != nullptr || n_rows == n_occurrences, "scatter_grad_rows: n_rows != n_occurrences");
    run_scatter_rows(device, emb_offset_dev, n_occurrences, dim, row_offsets_dev, n_rows, pooling,
                     pooled_grad_dev, grad_stride, grad_col, grad_fused_dev, total_floats, (cudaStream_t)stream);
  });
}

int mono_embedding_to_layout(int32_t device, const float* const* emb_ptrs_dev,
                             const int32_t* emb_strides_dev, int32_t n_emb,
                             const uint64_t* fid_offset_dev, int64_t total_fid,
                             const int32_t* feature_offset_dev, int32_t total_feature,
                             const uint32_t* nfl_offset_dev, int32_t total_nfl, int32_t batch_size,
                             const mono_slice_task* tasks_host, int32_t n_tasks,
                             float* const* out_ptrs_dev, void* stream) {
  return guarded([&] {
    check_layout_tasks(tasks_host, n_tasks, total_nfl);
    MONO_CUDA(cudaSetDevice(device));
    launch_layout(false, const_cast<float* const*>(emb_ptrs_dev), emb_strides_dev, n_emb, fid_offset_dev,
                  total_fid, feature_offset_dev, total_feature, nfl_offset_dev, total_nfl, batch_size,
                  tasks_host, n_tasks, out_ptrs_dev, (cudaStream_t)stream);
  });
}

int mono_embedding_to_layout_grad(int32_t device, float* const* emb_grad_ptrs_dev,
                                  const int32_t* emb_strides_dev, int32_t n_emb,
                                  const uint64_t* fid_offset_dev, int64_t total_fid,
                                  const int32_t* feature_offset_dev, int32_t total_feature,
                                  const uint32_t* nfl_offset_dev, int32_t total_nfl,
                                  int32_t batch_size, const mono_slice_task* tasks_host,
                                  int32_t n_tasks, const float* const* out_grad_ptrs_dev,
                                  void* stream) {
  return guarded([&] {
    check_layout_tasks(tasks_host, n_tasks, total_nfl);
    MONO_CUDA(cudaSetDevice(device));
    launch_layout(true, emb_grad_ptrs_dev, emb_strides_dev, n_emb, fid_offset_dev, total_fid,
                  feature_offset_dev, total_feature, nfl_offset_dev, total_nfl, batch_size, tasks_host,
                  n_tasks, const_cast<float* const*>(out_grad_ptrs_dev), (cudaStream_t)stream);
  });
}

int mono_gather_pool_bf16(int32_t device, const float* fused_emb_dev, const int32_t* emb_offset_dev,
                          const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim, int32_t pooling,
                          float* out_dev, int64_t out_stride, int32_t out_col, void* stream) {
  return guarded([&] {
    MONO_CUDA(cudaSetDevice(device));
    require(dim > 0, "dim must be positive");
    launch_gather_pool_bf16(fused_emb_dev, emb_offset_dev, row_offsets_dev, n_rows, dim, pooling,
                            reinterpret_cast<__nv_bfloat16*>(out_dev), out_stride, out_col, (cudaStream_t)stream);
  });
}

int mono_gather_pool_grad_bf16(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                               int32_t grad_col, const int32_t* emb_offset_dev,
                               const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                               int32_t pooling, float* grad_fused_dev, void* stream) {
  return guarded([&] {
    MONO_CUDA(cudaSetDevice(device));
    require(dim > 0, "dim must be positive");
    launch_gather_pool_grad_bf16(reinterpret_cast<const __nv_bfloat16*>(pooled_grad_dev), grad_stride, grad_col,
                                 emb_offset_dev, row_offsets_dev, n_rows, dim, pooling, grad_fused_dev,
                                 (cudaStream_t)stream);
  });
}

int mono_scatter_grad_rows_bf16(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                                int32_t grad_col, const int32_t* emb_offset_dev, int64_t n_occurrences,
                                const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                                int32_t pooling, float* grad_fused_dev, int64_t total_floats,
                                void* stream) {
  return guarded([&] {
    require(pooled_grad_dev && emb_offset_dev && grad_fused_dev, "scatter_grad_rows: null argument");
    require(row_offsets_dev != nullptr || n_rows == n_occurrences, "scatter_grad_rows: n_rows != n_occurrences");
    run_scatter_rows(device, emb_offset_dev, n_occurrences, dim, row_offsets_dev, n_rows, pooling,
                     pooled_grad_dev, grad_stride, grad_col, grad_fused_dev, total_floats, (cudaStream_t)stream,
                     true);
  });
}

int mono_embedding_to_layout_bf16(int32_t device, const float* const* emb_ptrs_dev,
                                  const int32_t* emb_strides_dev, int32_t n_emb,
                                  const uint64_t* fid_offset_dev, int64_t total_fid,
                                  const int32_t* feature_offset_dev, int32_t total_feature,
                                  const uint32_t* nfl_offset_dev, int32_t total_nfl, int32_t batch_size,
                                  const mono_slice_task* tasks_host, int32_t n_tasks,
                                  float* const* out_ptrs_dev, void* stream) {
  return guarded([&] {
    check_layout_tasks(tasks_host, n_tasks, total_nfl);
    MONO_CUDA(cudaSetDevice(device));
    launch_layout(false, const_cast<float* const*>(emb_ptrs_dev), emb_strides_dev, n_emb, fid_offset_dev,
                  total_fid, feature_offset_dev, total_feature, nfl_offset_dev, total_nfl, batch_size,
                  tasks_host, n_tasks, out_ptrs_dev, (cudaStream_t)stream, true);
  });
}

int mono_embedding_to_layout_grad_bf16(int32_t device, float* const* emb_grad_ptrs_dev,
                                       const int32_t* emb_strides_dev, int32_t n_emb,
                                       const uint64_t* fid_offset_dev, int64_t total_fid,
                                       const int32_t* feature_offset_dev, int32_t total_feature,
                                       const uint32_t* nfl_offset_dev, int32_t total_nfl,
                                       int32_t batch_size, const mono_slice_task* tasks_host,
                                       int32_t n_tasks, const float* const* out_grad_ptrs_dev,
                                       void* stream) {
  return guarded([&] {
    check_layout_tasks(tasks_host, n_tasks, total_nfl);
    MONO_CUDA(cudaSetDevice(device));
    launch_layout(true, emb_grad_ptrs_dev, emb_strides_dev, n_emb, fid_offset_dev, total_fid,
                  feature_offset_dev, total_feature, nfl_offset_dev, total_nfl, batch_size, tasks_host,
                  n_tasks, const_cast<float* const*>(out_grad_ptrs_dev), (cudaStream_t)stream, true);
  });
}

// ---- host-buffer entry points --------------------------------------------------------------
int mono_mtable_lookup_host(mono_mtable_t* t, const int64_t* ids_host, const int64_t* id_split_host,
                            float* emb_out_host) {
  return guarded([&] {
    HandleGuard hg_(t);
    cudaStream_t s = t->own_stream;
    int64_t n_total = 0;
    auto segs = table_segs(t, id_split_host, 0, &n_total, nullptr);
    if (segs.empty()) return;
    size_t out_floats = 0;
    for (auto& sg : segs)
      out_floats = std::max<size_t>(out_floats, sg.val_off + (sg.id_end - sg.id_begin) * t->tables[sg.table].dim);
    ensure_pinned(&t->pinned_in, &t->pinned_in_cap, sizeof(int64_t) * n_total);
    ensure_pinned(&t->pinned_out, &t->pinned_out_cap, sizeof(float) * out_floats);
    int64_t* d_ids = (int64_t*)t->ws_host_in.get(sizeof(int64_t) * n_total, s);
    float* d_out = (float*)t->ws_host_out.get(sizeof(float) * out_floats, s);
    std::memcpy(t->pinned_in, ids_host, sizeof(int64_t) * n_total);
    MONO_CUDA(cudaMemcpyAsync(d_ids, t->pinned_in, sizeof(int64_t) * n_total, cudaMemcpyHostToDevice, s));
    launch_lookup(t, segs.data(), (int)segs.size(), d_ids, n_total, d_out, s);
    MONO_CUDA(cudaMemcpyAsync(t->pinned_out, d_out, sizeof(float) * out_floats, cudaMemcpyDeviceToHost, s));
    MONO_CUDA(cudaStreamSynchronize(s));
    std::memcpy(emb_out_host, t->pinned_out, sizeof(float) * out_floats);
  });
}

int mono_mtable_lookup_pool_host(mono_mtable_t* t, int32_t k, const int64_t* fids_host,
                                 const int32_t* row_offsets_host, int64_t n_rows, int64_t n_fids,
                                 int32_t pooling, float* out_host) {
  return guarded([&] {
    require(k >= 0 && k < (int)t->tables.size(), "bad table index");
    HandleGuard hg_(t);
    cudaStream_t s = t->own_stream;
    if (n_rows <= 0) return;
    const int D = t->tables[k].dim;
    const size_t in_bytes = sizeof(int64_t) * n_fids + (row_offsets_host ? sizeof(int32_t) * (n_rows + 1) : 0);
    const size_t out_bytes = sizeof(float) * (size_t)n_rows * D;
    ensure_pinned(&t->pinned_in, &t->pinned_in_cap, in_bytes);
    ensure_pinned(&t->pinned_out, &t->pinned_out_cap, out_bytes);
    char* d_in = (char*)t->ws_host_in.get(in_bytes, s);
    float* d_out = (float*)t->ws_host_out.get(out_bytes, s);
    std::memcpy(t->pinned_in, fids_host, sizeof(int64_t) * n_fids);
    if (row_offsets_host)
      std::memcpy((char*)t->pinned_in + sizeof(int64_t) * n_fids, row_offsets_host, sizeof(int32_t) * (n_rows + 1));
    MONO_CUDA(cudaMemcpyAsync(d_in, t->pinned_in, in_bytes, cudaMemcpyHostToDevice, s));
    const int32_t* d_off = row_offsets_host ? (const int32_t*)(d_in + sizeof(int64_t) * n_fids) : nullptr;
    launch_lookup_pool(t, k, (const int64_t*)d_in, d_off, n_rows, pooling, d_out, D, 0, s);
    MONO_CUDA(cudaMemcpyAsync(t->pinned_out, d_out, out_bytes, cudaMemcpyDeviceToHost, s));
    MONO_CUDA(cudaStreamSynchronize(s));
    std::memcpy(out_host, t->pinned_out, out_bytes);
  });
}

int mono_mtable_optimize_host(mono_mtable_t* t, const int64_t* ids_host,
                              const int64_t* id_split_host, const float* grads_host,
                              const float* learning_rate_host, int64_t update_time,
                              int64_t /*global_step*/, uint32_t flags) {
  return guarded([&] {
    HandleGuard hg_(t);
    cudaStream_t s = t->own_stream;
    int64_t n_total = 0;
    int n_lr = 0;
    auto segs = table_segs(t, id_split_host, 0, &n_total, &n_lr);
    if (segs.empty()) return;
    size_t g_floats = 0;
    for (auto& sg : segs)
      g_floats = std::max<size_t>(g_floats, sg.val_off + (sg.id_end - sg.id_begin) * t->tables[sg.table].dim);
    const size_t id_bytes = (sizeof(int64_t) * n_total + 15) & ~(size_t)15;
    const size_t in_bytes = id_bytes + sizeof(float) * g_floats;
    ensure_pinned(&t->pinned_in, &t->pinned_in_cap, in_bytes);
    char* d_in = (char*)t->ws_host_in.get(in_bytes, s);
    std::memcpy(t->pinned_in, ids_host, sizeof(int64_t) * n_total);
    std::memcpy((char*)t->pinned_in + id_bytes, grads_host, sizeof(float) * g_floats);
    MONO_CUDA(cudaMemcpyAsync(d_in, t->pinned_in, in_bytes, cudaMemcpyHostToDevice, s));
    run_upsert(t, kOpOptimize, segs.data(), (int)segs.size(), (const int64_t*)d_in, n_total,
               (const float*)(d_in + id_bytes), learning_rate_host, n_lr, update_time,
               flags & MONO_FLAG_IDS_UNIQUE, flags & MONO_FLAG_DEDUP_SUM, nullptr, s);
    MONO_CUDA(cudaStreamSynchronize(s));
  });
}

}  // extern "C"
