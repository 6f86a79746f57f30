// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement of the reference (bytedance/monolith) algorithms on the embedding hot path.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load this library.  The product (monolith_b200/) never links, imports or calls it.
//
// Every function cites the reference file:line it restates (paths relative to
// monolith/native_training/, RT = runtime/).  The restatement is pinned against the reference's
// own known-answer tests transcribed in tests/golden/ (see tests/test_oracle_golden.py) and, for
// Adagrad, against the reference header RT/hash_table/optimizer/avx_utils.h compiled verbatim into
// oracle/_ref (see oracle/Makefile, tests/test_oracle_ref.py).
//
// Parity status: observable results (key membership, row values, integer index encodings) are
// pinned.  Bucket positions inside the reference's libcuckoo map are NOT reproducible (absl::Hash
// is per-process salted): "parity unpinned" for bucket placement, by construction.
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fPIC -shared (see oracle/Makefile).
// -ffp-contract=off keeps a*b+c unfused unless std::fma is written explicitly, so that the float
// sequence below is exactly what is written.

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../include/mono_emb.h"

namespace {

thread_local std::string g_err;

// ---------------------------------------------------------------------------------------------
// Optimizers
// ---------------------------------------------------------------------------------------------

// ref: RT/hash_table/optimizer/avx_utils.h:96-119 (Avx256AdagradOptimize, blocks of 8 lanes) and
// :29-38 (BaselineAdagradOptimize, tail).  The reference is built with -mavx -mfma and
// _ENABLE_AVX, so AdagradOptimize (:238-245) takes the AVX path: the first floor(len/8)*8 lanes
// use FMA forms and apply the RAW grad in the last step (:112); the tail uses the baseline form.
void AdagradOptimize(float* num, float* norm, const float* grad, size_t len, float lr,
                     float w_decay) {
  size_t i = 0;
  for (; i + 8 <= len; i += 8) {
    for (size_t j = i; j < i + 8; ++j) {
      float updated_grad = std::fma(w_decay, num[j], grad[j]);        // _mm256_fmadd_ps(lamda,_num,_grad)
      float norm_new = std::fma(updated_grad, updated_grad, norm[j]);  // _mm256_fmadd_ps(ug,ug,_norm)
      norm[j] = norm_new;
      float effective_lr = lr / std::sqrt(norm_new);                   // _mm256_div_ps(_lr, sqrt)
      num[j] = std::fma(-effective_lr, grad[j], num[j]);               // _mm256_fnmadd_ps(eff,_grad,_num)
    }
  }
  for (; i < len; ++i) {  // BaselineAdagradOptimize
    float g = grad[i] + w_decay * num[i];
    norm[i] += g * g;
    float effective_lr = lr / std::sqrt(norm[i]);
    num[i] -= effective_lr * g;
  }
}

// ref: RT/hash_table/optimizer/ftrl_optimizer.cc:56-76.  signbit() is 0/1 (not +-1), mirrored.
void FtrlOptimize(float* num, float* norm, float* zero, const float* grad, int dim, float lr,
                  float beta, float l1, float l2) {
  for (int i = 0; i < dim; ++i) {
    float norm_new = norm[i] + grad[i] * grad[i];
    float sigma = (std::sqrt(norm_new) - std::sqrt(norm[i])) / lr;
    zero[i] += (grad[i] - sigma * num[i]);
    norm[i] = norm_new;
    num[i] = (std::fabs(zero[i]) > l1)
                 ? lr * ((std::signbit(zero[i]) ? 1.0f : 0.0f) * l1 - zero[i]) /
                       (std::sqrt(norm[i]) + beta + l2 * lr)
                 : 0.0f;
  }
}

// ref: RT/hash_table/optimizer/adam_optimizer.cc:57-84.  Per-row beta powers live in the entry
// (state = m[dim], v[dim], beta1_power, beta2_power; :30-55).  All arithmetic in float.
void AdamOptimize(float* num, float* m, float* v, float* b1p, float* b2p, const float* grad,
                  int dim, float lr0, float beta1, float beta2, float eps, float wd,
                  bool nesterov) {
  float lr = lr0 * std::sqrt(1.0f - *b2p) / (1.0f - *b1p);
  for (int i = 0; i < dim; ++i) {
    float cur_grad = grad[i] + wd * num[i];
    float new_m = m[i] + (cur_grad - m[i]) * (1.0f - beta1);
    float new_v = v[i] + (cur_grad * cur_grad - v[i]) * (1.0f - beta2);
    float new_w = num[i];
    if (nesterov) {
      new_w -= ((cur_grad * (1.0f - beta1) + beta1 * new_m) * lr) / (std::sqrt(new_v) + eps);
    } else {
      new_w -= (new_m * lr) / (std::sqrt(new_v) + eps);
    }
    num[i] = new_w;
    m[i] = new_m;
    v[i] = new_v;
  }
  *b1p *= beta1;
  *b2p *= beta2;
}

// ref: RT/hash_table/optimizer/sgd_optimizer.cc:42-49
void SgdOptimize(float* num, const float* grad, int dim, float lr) {
  for (int i = 0; i < dim; ++i) num[i] -= lr * grad[i];
}

// ref: RT/hash_table/optimizer/moving_average_optimizer.cc:44-52
void MovingAverageOptimize(float* num, const float* grad, int dim, float momentum) {
  for (int i = 0; i < dim; ++i) {
    float new_w = momentum * num[i] + (1 - momentum) * grad[i];
    num[i] = new_w;
  }
}

// ref: RT/hash_table/optimizer/group_adagrad_optimizer.cc:50-89
void GroupAdagradOptimize(float* num, float* grad_square_sum, const float* grad, int dim, float effective_lr, float wd,
                          float beta, float l2) {
  float max_grad_square = 0.0f;
  std::vector<float> g_decayed(dim);
  for (int i = 0; i < dim; ++i) {
    float g = grad[i] + wd * num[i];
    if (g * g > max_grad_square) max_grad_square = g * g;
    g_decayed[i] = g;
  }
  *grad_square_sum = *grad_square_sum + max_grad_square;
  float lr = effective_lr / (beta + std::sqrt(*grad_square_sum));
  float z_norm = 0.0f;
  for (int i = 0; i < dim; ++i) {
    num[i] = g_decayed[i] - num[i] / lr;
    z_norm += num[i] * num[i];
  }
  z_norm = std::sqrt(z_norm);
  if (z_norm < l2) {
    for (int i = 0; i < dim; ++i) num[i] = 0;
  } else {
    float coeffi = -lr * (z_norm - l2) / z_norm;
    for (int i = 0; i < dim; ++i) num[i] = coeffi * num[i];
  }
}

int StateFloats(const mono_segment_cfg& s) {
  switch (s.opt_type) {
    case MONO_OPT_SGD: return 0;                 // sgd_optimizer.cc:28
    case MONO_OPT_ADAGRAD: return s.dim;         // adagrad_optimizer.cc:31-33
    case MONO_OPT_FTRL: return 2 * s.dim;        // ftrl_optimizer.cc:31-33
    case MONO_OPT_ADAM: return 2 * s.dim + 2;    // adam_optimizer.cc:30-32
    case MONO_OPT_MOMENTUM: case MONO_OPT_RMSPROP: case MONO_OPT_RMSPROPV2: return s.dim;  // momentum_optimizer.cc:29, rmsprop_optimizer.cc:29,99
    case MONO_OPT_ADADELTA: return 2 * s.dim;    // adadelta_optimizer.cc:29-31
    case MONO_OPT_AMSGRAD: return 3 * s.dim + 2; // amsgrad_optimizer.cc:30-32
    case MONO_OPT_MOVING_AVERAGE: return 0;      // moving_average_optimizer.cc:30
    case MONO_OPT_GROUP_ADAGRAD: return 1;       // group_adagrad_optimizer.cc:31 (one float: grad_square_sum)
  }
  return 0;
}

// ref: RT/hash_table/optimizer/momentum_optimizer.cc:52-72
void MomentumOptimize(float* num, float* n, const float* grad, int dim, float lr, float momentum, float wd, bool nesterov) {
  for (int i = 0; i < dim; ++i) {
    float dx = lr * (grad[i] + wd * num[i]);
    float new_n = n[i];
    float new_w = num[i];
    if (nesterov) {
      float prev_n = new_n;
      new_n = momentum * new_n - dx;
      new_w += -momentum * prev_n + (1 + momentum) * new_n;
    } else {
      new_n = momentum * new_n - dx;
      new_w += new_n;
    }
    n[i] = new_n;
    num[i] = new_w;
  }
}

// ref: RT/hash_table/optimizer/rmsprop_optimizer.cc:49-68 (v1: the CONFIG's learning rate, (1 - momentum) dx^2) and
// :121-141 (v2: learning_rates[0], dx^2); both compute in double and store floats.
void RmspropOptimize(float* num, float* n, const float* grad, int dim, float lr, float momentum, float wd, bool v2) {
  for (int i = 0; i < dim; ++i) {
    float new_n = n[i];
    float new_w = num[i];
    double dx = grad[i] + static_cast<double>(wd) * new_w;
    if (v2) new_n = static_cast<double>(momentum) * new_n + dx * dx;
    else new_n = static_cast<double>(momentum) * new_n + (1 - static_cast<double>(momentum)) * dx * dx;
    double eta = static_cast<double>(lr) / (std::sqrt(new_n) + 1);
    new_w -= eta * dx;
    n[i] = new_n;
    num[i] = new_w;
  }
}

// ref: RT/hash_table/optimizer/adadelta_optimizer.cc:51-72
void AdadeltaOptimize(float* num, float* accum, float* accum_update, const float* grad, int dim, float lr, float rho,
                      float eps, float wd) {
  for (int i = 0; i < dim; ++i) {
    float cur_grad = grad[i] + wd * num[i];
    float new_accum = accum[i] * rho + cur_grad * cur_grad * (1 - rho);
    float update = std::sqrt(accum_update[i] + eps) / std::sqrt(new_accum + eps) * cur_grad;
    float new_w = num[i] - update * lr;
    float new_accum_update = accum_update[i] * rho + update * update * (1 - rho);
    num[i] = new_w;
    accum[i] = new_accum;
    accum_update[i] = new_accum_update;
  }
}

// ref: RT/hash_table/optimizer/amsgrad_optimizer.cc:58-88
void AmsgradOptimize(float* num, float* m, float* v, float* vhat, float* b1p, float* b2p, const float* grad, int dim,
                     float lr0, float beta1, float beta2, float eps, float wd, bool nesterov) {
  float lr = lr0 * std::sqrt(1.0f - *b2p) / (1.0f - *b1p);
  for (int i = 0; i < dim; ++i) {
    float cur_grad = grad[i] + wd * num[i];
    float new_m = m[i] + (cur_grad - m[i]) * (1.0f - beta1);
    float new_v = v[i] + (cur_grad * cur_grad - v[i]) * (1.0f - beta2);
    float new_vhat = std::max(vhat[i], new_v);
    float new_w = num[i];
    if (nesterov) new_w -= ((cur_grad * (1.0f - beta1) + beta1 * new_m) * lr) / (std::sqrt(new_vhat) + eps);
    else new_w -= (new_m * lr) / (std::sqrt(new_vhat) + eps);
    num[i] = new_w;
    m[i] = new_m;
    v[i] = new_v;
    vhat[i] = new_vhat;
  }
  *b1p *= beta1;
  *b2p *= beta2;
}

// splitmix64: used only for the counter-based uniform initializer, which is an engine-defined
// replacement of the reference's unseeded thread_local mt19937
// (ref: RT/hash_table/initializer/random_uniform_initializer.cc:31-37 — not reproducible, so the
// oracle mirrors the ENGINE's definition here; parity for random init is statistical vs the ref).
inline uint64_t Mix64(uint64_t x) {
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  x ^= x >> 31;
  return x;
}
inline float UniformInit(uint64_t seed, int64_t fid, int col, float lo, float hi) {
  uint64_t h = Mix64(Mix64(seed ^ 0x9E3779B97F4A7C15ULL) + (uint64_t)fid) ;
  h = Mix64(h + (uint64_t)col * 0xD1B54A32D192ED03ULL);
  float u = (float)(h >> 40) * (1.0f / 16777216.0f);  // 24 bits -> [0,1)
  return lo + (hi - lo) * u;
}

struct Row {
  std::vector<float> data;  // [emb dim | opt state]  (ref: entry_accessor.cc:113-115)
  uint32_t ts = 0;          // ref: RT/hash_table/entry_defs.h:31-39
};

// Counting admission filter — restatement of monolith::hash_filter::HashFilter<uint16_t>
// (RT/hash_filter/hash_filter.h:34-165, filter.h:60-61): open addressing over capacity * 1.5 (+64) 16-bit cells,
// cell = 12-bit signature << 4 | 4-bit saturating count, at most 64 probes; add() returns the count BEFORE the
// increment (0 for a new FID, 15 when the probe window is exhausted).  The cell a FID lands in depends on
// absl::Hash (salted per process) and is therefore unpinned; counts are pinned as long as signatures do not collide.
struct HashFilter {
  static constexpr int kCountBit = 4, kMaxStep = 64;
  static constexpr uint32_t kMaxCount = (1u << kCountBit) - 1;
  std::vector<uint16_t> map;
  uint64_t total_size = 0, capacity = 0, num_elements = 0, failure_count = 0;
  explicit HashFilter(uint64_t cap) : capacity(cap) {
    total_size = (uint64_t)(cap * 1.5);
    if (total_size == 0) total_size = 1;
    map.assign(total_size + kMaxStep, 0);
  }
  static uint16_t Signature(uint64_t fid) { return (uint16_t)(((fid >> 17) | (fid << 15)) & 0x0FFF); }  // :128
  uint32_t Add(int64_t fid_, uint32_t count) {  // :69-76 + iterator add :40-62
    const uint64_t fid = (uint64_t)fid_;
    const uint16_t sign = Signature(fid);
    size_t pos = (size_t)(Mix64(fid) % total_size);
    for (int step = 0; step < kMaxStep; ++step) {
      uint16_t& v = map[pos];
      if (v == 0 || (v >> kCountBit) == sign) {
        if (count > kMaxCount) count = kMaxCount;
        if (v == 0) {
          num_elements = std::min(num_elements + 1, capacity);
          v = (uint16_t)((sign << kCountBit) + count);
          return 0;
        }
        const uint32_t c = v & kMaxCount;
        if (c + count >= kMaxCount) v |= (uint16_t)kMaxCount; else v = (uint16_t)(v + count);
        return c;
      }
      if (++pos == map.size()) pos = 0;
    }
    ++failure_count;
    return kMaxCount;
  }
};

struct Table {
  std::string name;
  std::vector<mono_segment_cfg> segs;
  int dim = 0, state = 0, slices = 0;
  uint32_t default_expire_days = 36500;
  std::unordered_map<uint32_t, uint32_t> slot_expire;
  uint64_t seed = 0;
  int64_t max_update_ts = 0;
  std::unordered_map<int64_t, Row> m;
  // admission filter (absent = the dummy filter, which never filters: dummy_hash_filter.h:31-52)
  std::shared_ptr<HashFilter> filter;
  uint32_t default_threshold = 0;
  std::unordered_map<uint32_t, uint32_t> slot_threshold;
  // ref: HashFilterTfBridge::ShouldBeFiltered (hash_filter_tf_bridge.h:36-47) -> HashFilter::ShouldBeFiltered
  // (hash_filter.h:137-144): threshold <= 0 never filters; otherwise add(fid, count) < threshold
  bool ShouldBeFiltered(int64_t fid, uint32_t count) {
    if (!filter) return false;
    const uint32_t slot = (uint32_t)(((uint64_t)fid >> 48) & 0x7FFF);
    auto it = slot_threshold.find(slot);
    const uint32_t thr = it == slot_threshold.end() ? default_threshold : it->second;
    return FilterAtThreshold(filter.get(), fid, count, thr);
  }
  static bool FilterAtThreshold(HashFilter* f, int64_t fid, uint32_t count, uint32_t thr) {
    if (thr == 0) return false;
    return f->Add(fid, count) < thr;
  }

  // ref: EntryAccessor::Init (entry_accessor.cc:165-169): initializer then optimizer Init.
  void Init(int64_t fid, Row* r) const {
    r->data.assign(dim + state, 0.f);
    int col = 0;
    float* st = r->data.data() + dim;
    for (const auto& s : segs) {
      for (int i = 0; i < s.dim; ++i) {
        float v = 0.f;
        switch (s.init_type) {
          case MONO_INIT_ZEROS: v = 0.f; break;
          case MONO_INIT_ONES: v = 1.f; break;
          case MONO_INIT_CONSTANT: v = s.init_a; break;
          case MONO_INIT_UNIFORM: v = UniformInit(seed, fid, col + i, s.init_a, s.init_b); break;
        }
        r->data[col + i] = v;
      }
      switch (s.opt_type) {
        case MONO_OPT_ADAGRAD:  // adagrad_optimizer.cc:47-52
          for (int i = 0; i < s.dim; ++i) st[i] = s.opt_p[0];
          break;
        case MONO_OPT_FTRL:  // ftrl_optimizer.cc:45-52: norm = init_acc, zero = 0
          for (int i = 0; i < s.dim; ++i) { st[i] = s.opt_p[0]; st[s.dim + i] = 0.f; }
          break;
        case MONO_OPT_ADAM:  // adam_optimizer.cc:44-55
          for (int i = 0; i < 2 * s.dim; ++i) st[i] = 0.f;
          st[2 * s.dim] = s.opt_p[0];
          st[2 * s.dim + 1] = s.opt_p[1];
          break;
        case MONO_OPT_AMSGRAD:  // amsgrad_optimizer.cc:44-56
          for (int i = 0; i < 3 * s.dim; ++i) st[i] = 0.f;
          st[3 * s.dim] = s.opt_p[0];
          st[3 * s.dim + 1] = s.opt_p[1];
          break;
        case MONO_OPT_MOMENTUM: case MONO_OPT_RMSPROP: case MONO_OPT_RMSPROPV2:
          for (int i = 0; i < s.dim; ++i) st[i] = 0.f;
          break;
        case MONO_OPT_ADADELTA:
          for (int i = 0; i < 2 * s.dim; ++i) st[i] = 0.f;
          break;
        case MONO_OPT_GROUP_ADAGRAD:  // group_adagrad_optimizer.cc:45-48
          st[0] = s.opt_p[0];
          break;
        default: break;
      }
      st += StateFloats(s);
      col += s.dim;
    }
  }

  // ref: CombinedOptimizer::Optimize (optimizer_combination.cc:62-72): segment s uses
  // learning_rates[s], its own num/grad sub-span and its own state block.
  void Optimize(Row* r, const float* grad, const float* lr) const {
    float* num = r->data.data();
    float* st = r->data.data() + dim;
    int col = 0, sl = 0;
    for (const auto& s : segs) {
      switch (s.opt_type) {
        case MONO_OPT_SGD: SgdOptimize(num + col, grad + col, s.dim, lr[sl]); break;
        case MONO_OPT_ADAGRAD:
          AdagradOptimize(num + col, st, grad + col, s.dim, lr[sl], s.opt_p[1]);
          break;
        case MONO_OPT_FTRL:
          FtrlOptimize(num + col, st, st + s.dim, grad + col, s.dim, lr[sl], s.opt_p[1],
                       s.opt_p[2], s.opt_p[3]);
          break;
        case MONO_OPT_ADAM:
          AdamOptimize(num + col, st, st + s.dim, st + 2 * s.dim, st + 2 * s.dim + 1, grad + col,
                       s.dim, lr[sl], s.opt_p[0], s.opt_p[1], s.opt_p[2], s.opt_p[3],
                       s.opt_p[4] != 0.f);
          break;
        case MONO_OPT_MOMENTUM:
          MomentumOptimize(num + col, st, grad + col, s.dim, lr[sl], s.opt_p[0], s.opt_p[1], s.opt_p[2] != 0.f);
          break;
        case MONO_OPT_RMSPROP:  // the config's learning rate, not the call's (rmsprop_optimizer.cc:62)
          RmspropOptimize(num + col, st, grad + col, s.dim, s.opt_p[2], s.opt_p[0], s.opt_p[1], false);
          break;
        case MONO_OPT_RMSPROPV2:
          RmspropOptimize(num + col, st, grad + col, s.dim, lr[sl], s.opt_p[0], s.opt_p[1], true);
          break;
        case MONO_OPT_ADADELTA:
          AdadeltaOptimize(num + col, st, st + s.dim, grad + col, s.dim, lr[sl], s.opt_p[0], s.opt_p[1], s.opt_p[2]);
          break;
        case MONO_OPT_AMSGRAD:
          AmsgradOptimize(num + col, st, st + s.dim, st + 2 * s.dim, st + 3 * s.dim, st + 3 * s.dim + 1, grad + col, s.dim,
                          lr[sl], s.opt_p[0], s.opt_p[1], s.opt_p[2], s.opt_p[3], s.opt_p[4] != 0.f);
          break;
        case MONO_OPT_MOVING_AVERAGE:
          MovingAverageOptimize(num + col, grad + col, s.dim, s.opt_p[0]);
          break;
        case MONO_OPT_GROUP_ADAGRAD:
          GroupAdagradOptimize(num + col, st, grad + col, s.dim, lr[sl], s.opt_p[1], s.opt_p[2], s.opt_p[3]);
          break;
      }
      st += StateFloats(s);
      col += s.dim;
      ++sl;
    }
  }

  // ref: CuckooEmbeddingHashTable::UpsertEntry (cuckoo_embedding_hash_table.cc:346-353):
  // absent -> allocate + Init, then apply fn.  Returns true when the key was inserted.
  template <class F>
  bool Upsert(int64_t id, F fn) {
    auto it = m.find(id);
    bool inserted = false;
    if (it == m.end()) {
      Row r;
      Init(id, &r);
      it = m.emplace(id, std::move(r)).first;
      inserted = true;
    }
    fn(&it->second);
    return inserted;
  }

  void BumpMaxTs(int64_t update_time) {  // ref: tf_bridge.cc:202-206,262-263
    max_update_ts = std::max(max_update_ts, update_time);
  }
};

}  // namespace

struct orc_mtable {
  std::vector<Table> tables;  // sorted by name (ref: multi_hash_table_ops.py:72,83)
};

namespace {

// ref: NT/data/training_instance/cc/reader_util.h:36-38
inline int SlotIdV2(uint64_t fid) { return (fid >> 48) & ((1 << 15) - 1); }

void TableLookup(const Table& t, const int64_t* ids, int64_t n, float* out) {
  // ref: CuckooEmbeddingHashTable::Lookup (cuckoo_embedding_hash_table.cc:161-171): hit -> copy
  // dim floats (RawRetriever), miss -> zeros; never inserts.
  for (int64_t i = 0; i < n; ++i) {
    auto it = t.m.find(ids[i]);
    if (it != t.m.end()) {
      std::memcpy(out + i * t.dim, it->second.data.data(), sizeof(float) * t.dim);
    } else {
      std::memset(out + i * t.dim, 0, sizeof(float) * t.dim);
    }
  }
}

// ref: EmbeddingHashTableTfBridge::BatchOptimize (tf_bridge.cc:258-341) with the dummy hash filter
// (never filters, RT/hash_filter/dummy_hash_filter.h:31-52) ->
// CuckooEmbeddingHashTable::BatchOptimize/Optimize (cuckoo_embedding_hash_table.cc:228-247).
void TableBatchOptimize(Table* t, const int64_t* ids, int64_t n, const float* grads,
                        const float* lr, int64_t update_time, bool enable_dedup) {
  t->BumpMaxTs(update_time);
  const int D = t->dim;
  if (enable_dedup) {
    // tf_bridge.cc:270-310: first occurrence copies, later occurrences ReduceSum into it.
    std::vector<float> cache((size_t)n * D);
    std::unordered_map<int64_t, float*> ids_to_grads;
    std::unordered_map<int64_t, uint32_t> ids_to_counts;
    std::vector<int64_t> order;
    for (int64_t i = 0; i < n; ++i) {
      auto it = ids_to_grads.find(ids[i]);
      if (it == ids_to_grads.end()) {
        float* dst = cache.data() + ids_to_grads.size() * D;
        std::memcpy(dst, grads + i * D, sizeof(float) * D);
        ids_to_grads[ids[i]] = dst;
        ids_to_counts[ids[i]] = 1;
        order.push_back(ids[i]);
      } else {
        float* dst = it->second;
        const float* src = grads + i * D;
        for (int j = 0; j < D; ++j) dst[j] = dst[j] + src[j];  // avx_utils.h:247-254 ReduceSum(a,b)
        ++ids_to_counts[ids[i]];
      }
    }
    // second step (tf_bridge.cc:296-310): ids absent from the table pass the filter with their occurrence count
    std::vector<int64_t> kept;
    for (int64_t id : order)
      if (t->m.count(id) || !t->ShouldBeFiltered(id, ids_to_counts[id])) kept.push_back(id);
    for (int64_t id : kept) {
      const float* g = ids_to_grads[id];
      t->Upsert(id, [&](Row* r) { r->ts = (uint32_t)update_time; t->Optimize(r, g, lr); });
    }
  } else {
    // tf_bridge.cc:312-326: the whole id list is filtered FIRST (Contains sees the table as it was before this
    // call, each absent occurrence adds 1 to its counter), then the survivors are optimized in order
    std::vector<int64_t> kept;
    for (int64_t i = 0; i < n; ++i)
      if (t->m.count(ids[i]) || !t->ShouldBeFiltered(ids[i], 1)) kept.push_back(i);
    for (int64_t i : kept) {
      const float* g = grads + i * D;
      t->Upsert(ids[i], [&](Row* r) { r->ts = (uint32_t)update_time; t->Optimize(r, g, lr); });
    }
  }
}

}  // namespace

extern "C" {

const char* orc_last_error() { return g_err.c_str(); }

// ref: CreateMultiHashTableOp::CreateResource (RT/ops/multi_hash_table_op.cc:86-103) +
// EmbeddingHashTableTfBridge::New (tf_bridge.cc:49-108: dim = sum of segment dims).
int orc_mtable_create(const mono_table_cfg* cfgs, int32_t n, orc_mtable** out) {
  auto mt = std::make_unique<orc_mtable>();
  std::vector<int> order(n);
  for (int i = 0; i < n; ++i) order[i] = i;
  std::sort(order.begin(), order.end(),
            [&](int a, int b) { return std::string(cfgs[a].name) < std::string(cfgs[b].name); });
  for (int idx : order) {
    const auto& c = cfgs[idx];
    Table t;
    t.name = c.name;
    for (int s = 0; s < c.n_segments; ++s) {
      t.segs.push_back(c.segments[s]);
      t.dim += c.segments[s].dim;
      t.state += StateFloats(c.segments[s]);
      t.slices += 1;  // every optimizer has SliceSize()==1; combination sums them
    }
    t.default_expire_days = c.default_expire_days;
    for (int s = 0; s < c.n_slot_expire; ++s) t.slot_expire[c.slot_ids[s]] = c.slot_expire_days[s];
    t.seed = c.init_seed;
    mt->tables.push_back(std::move(t));
  }
  *out = mt.release();
  return 0;
}
int orc_mtable_destroy(orc_mtable* t) { delete t; return 0; }
int32_t orc_mtable_num_tables(const orc_mtable* t) { return (int32_t)t->tables.size(); }
int32_t orc_mtable_dim(const orc_mtable* t, int k) { return t->tables[k].dim; }
int32_t orc_mtable_slice_size(const orc_mtable* t, int k) { return t->tables[k].slices; }
int32_t orc_mtable_state_floats(const orc_mtable* t, int k) { return t->tables[k].state; }
int64_t orc_mtable_size(const orc_mtable* t, int k) { return (int64_t)t->tables[k].m.size(); }
int64_t orc_mtable_max_update_ts(const orc_mtable* t, int k) { return t->tables[k].max_update_ts; }
int32_t orc_mtable_table_index(const orc_mtable* t, const char* name) {
  for (size_t i = 0; i < t->tables.size(); ++i)
    if (t->tables[i].name == name) return (int32_t)i;
  return -1;
}

// ref: MultiHashTableLookupOp::Compute (RT/ops/multi_hash_table_lookup_op.cc:37-88), req_size==1.
int orc_mtable_lookup(orc_mtable* t, const int64_t* ids, const int64_t* id_split, float* out) {
  int64_t off = 0;
  for (size_t k = 0; k < t->tables.size(); ++k) {
    int64_t n = id_split[k + 1] - id_split[k];
    TableLookup(t->tables[k], ids + id_split[k], n, out + off);
    off += n * t->tables[k].dim;
  }
  return 0;
}

// ref: ComputeFusedOffsets<false> (RT/hash_table/utils.h:28-61)
int orc_fused_offsets(const int32_t* slot_size, const int32_t* dims, int K, int N,
                      int32_t* emb_splits, int32_t* key_offsets, int32_t* emb_offsets) {
  int total_embs = 0, prev = 0;
  key_offsets[0] = emb_offsets[0] = 0;
  for (int s = 0; s < N; ++s) {
    for (int k = 0; k < K; ++k) {
      int idx = K * s + k;
      int seg = dims[k] * slot_size[idx];
      total_embs += seg;
      key_offsets[idx + 1] = key_offsets[idx] + slot_size[idx];
      emb_offsets[idx + 1] = emb_offsets[idx] + seg;
    }
    emb_splits[s] = total_embs - prev;
    prev = total_embs;
  }
  return 0;
}

int orc_mtable_fused_offsets(const orc_mtable* t, const int32_t* slot_size, int N,
                             int32_t* emb_splits, int32_t* key_offsets, int32_t* emb_offsets) {
  std::vector<int32_t> dims;
  for (auto& tb : t->tables) dims.push_back(tb.dim);
  return orc_fused_offsets(slot_size, dims.data(), (int)dims.size(), N, emb_splits, key_offsets,
                           emb_offsets);
}

// ref: MultiHashTableFusedLookupOp<CPU>::ComputeH (multi_hash_table_lookup_op.cc:143-197)
int orc_mtable_fused_lookup(orc_mtable* t, const int64_t* ids, const int32_t* slot_size, int N,
                            float* out) {
  int K = (int)t->tables.size();
  std::vector<int32_t> es(N), ko(N * K + 1), eo(N * K + 1);
  orc_mtable_fused_offsets(t, slot_size, N, es.data(), ko.data(), eo.data());
  for (int s = 0; s < N; ++s)
    for (int k = 0; k < K; ++k) {
      int idx = s * K + k;
      TableLookup(t->tables[k], ids + ko[idx], slot_size[idx], out + eo[idx]);
    }
  return 0;
}

// ref: MultiHashTableOptimizeOp::Compute (RT/ops/multi_hash_table_update_op.cc:47-89)
int orc_mtable_optimize(orc_mtable* t, const int64_t* ids, const int64_t* id_split,
                        const float* grads, const float* lr, int64_t update_time,
                        int64_t /*global_step*/, int enable_dedup) {
  int64_t voff = 0;
  int lroff = 0;
  for (size_t k = 0; k < t->tables.size(); ++k) {
    Table& tb = t->tables[k];
    int64_t n = id_split[k + 1] - id_split[k];
    TableBatchOptimize(&tb, ids + id_split[k], n, grads + voff, lr + lroff, update_time,
                       enable_dedup != 0);
    voff += n * tb.dim;
    lroff += tb.slices;
  }
  return 0;
}

// ref: MultiHashTableFusedOptimizeOp<CPU>::ComputeH (multi_hash_table_update_op.cc:268-308),
// executed in shard order (the single-thread schedule of Shard()).
int orc_mtable_fused_optimize(orc_mtable* t, const int64_t* ids, const int32_t* slot_size,
                              const float* grads, const int32_t* key_offsets,
                              const int32_t* emb_offsets, const float* lr, int64_t req_time,
                              int64_t /*global_step*/, int N, int enable_grad_accumulation) {
  int K = (int)t->tables.size();
  for (int s = 0; s < N; ++s) {
    int lroff = 0;
    for (int k = 0; k < K; ++k) {
      int idx = s * K + k;
      Table& tb = t->tables[k];
      TableBatchOptimize(&tb, ids + key_offsets[idx], slot_size[idx], grads + emb_offsets[idx],
                         lr + lroff, req_time, enable_grad_accumulation != 0);
      lroff += tb.slices;
    }
  }
  return 0;
}

// Attach a counting hash filter to table k (ref: hash_filter_ops.create_hash_filters + SlotOccurrenceThresholdConfig,
// embedding_hash_table.proto:100-110).  n_slots per-slot thresholds override the default; threshold 0 = never filter.
int orc_mtable_set_hash_filter(orc_mtable* t, int32_t k, int64_t capacity, uint32_t default_threshold,
                               const uint32_t* slots, const uint32_t* thresholds, int32_t n_slots) {
  if (k < 0 || k >= (int)t->tables.size()) return 1;
  Table& tb = t->tables[k];
  tb.filter = std::make_shared<HashFilter>((uint64_t)capacity);
  tb.default_threshold = default_threshold;
  tb.slot_threshold.clear();
  for (int i = 0; i < n_slots; ++i) tb.slot_threshold[slots[i]] = thresholds[i];
  return 0;
}

// ref: MultiHashTableAssignOp (multi_hash_table_update_op.cc:106-145) -> TfBridge::Assign
// (tf_bridge.cc:179-206) -> CuckooEmbeddingHashTable::Assign (cuckoo_..cc:185-203).
int orc_mtable_assign(orc_mtable* t, const int64_t* ids, const int64_t* id_split,
                      const float* values, int64_t update_time) {
  int64_t voff = 0;
  for (size_t k = 0; k < t->tables.size(); ++k) {
    Table& tb = t->tables[k];
    tb.BumpMaxTs(update_time);
    // tf_bridge.cc:179-190: the whole id list is filtered FIRST (Contains sees the table as it was before this call,
    // each absent occurrence adds 1 to its counter), then the survivors are assigned in order
    std::vector<int64_t> kept;
    for (int64_t i = id_split[k]; i < id_split[k + 1]; ++i)
      if (tb.m.count(ids[i]) || !tb.ShouldBeFiltered(ids[i], 1)) kept.push_back(i);
    for (int64_t i : kept) {
      const float* v = values + voff + (i - id_split[k]) * tb.dim;
      tb.Upsert(ids[i], [&](Row* r) {
        r->ts = (uint32_t)update_time;
        std::memcpy(r->data.data(), v, sizeof(float) * tb.dim);  // entry_accessor.cc:175-179
      });
    }
    voff += (id_split[k + 1] - id_split[k]) * tb.dim;
  }
  return 0;
}

// The [total + 64] cells of table k's filter (1 when the table has none or n is not its cell count).
int orc_mtable_hash_filter_cells(const orc_mtable* t, int32_t k, uint16_t* out, int64_t n) {
  if (k < 0 || k >= (int)t->tables.size()) return 1;
  const auto& f = t->tables[k].filter;
  if (!f || n != (int64_t)f->map.size()) return 1;
  std::memcpy(out, f->map.data(), sizeof(uint16_t) * (size_t)n);
  return 0;
}

// One HashFilter of `capacity` on its own, fed fids[i] in order: thresholds null -> out[i] = add(fids[i], counts[i])
// (the count before the add); else out[i] = ShouldBeFiltered(fids[i], counts[i], thresholds[i]) (0 never adds).
// cells [n_cells = total + 64] receive the final state.
int orc_hash_filter_run(int64_t capacity, const int64_t* fids, const uint32_t* counts, const uint32_t* thresholds,
                        int64_t n, uint32_t* out, uint16_t* cells, int64_t n_cells) {
  HashFilter f((uint64_t)capacity);
  if (n_cells != (int64_t)f.map.size()) return 1;
  for (int64_t i = 0; i < n; ++i)
    out[i] = thresholds ? (uint32_t)Table::FilterAtThreshold(&f, fids[i], counts[i], thresholds[i])
                        : f.Add(fids[i], counts[i]);
  std::memcpy(cells, f.map.data(), sizeof(uint16_t) * (size_t)n_cells);
  return 0;
}

// ref: MultiHashTableAssignAddOp (multi_hash_table_update_op.cc:151-190): per-id serial AssignAdd2
// (tf_bridge.cc:224-240) -> CuckooEmbeddingHashTable::AssignAdd (cuckoo_..cc:205-212).
int orc_mtable_assign_add(orc_mtable* t, const int64_t* ids, const int64_t* id_split,
                          const float* values, int64_t update_time) {
  int64_t voff = 0;
  for (size_t k = 0; k < t->tables.size(); ++k) {
    Table& tb = t->tables[k];
    for (int64_t i = id_split[k]; i < id_split[k + 1]; ++i) {
      tb.BumpMaxTs(update_time);
      const float* v = values + voff;
      voff += tb.dim;
      if (tb.ShouldBeFiltered(ids[i], 1)) continue;  // AssignAdd2 has no Contains check (tf_bridge.cc:224-232)
      tb.Upsert(ids[i], [&](Row* r) {
        r->ts = (uint32_t)update_time;
        for (int j = 0; j < tb.dim; ++j) r->data[j] += v[j];  // entry_accessor.cc:181-187
      });
    }
  }
  return 0;
}

// ref: MultiHashTableReinitializeOp (multi_hash_table_update_op.cc:192-241) ->
// CuckooEmbeddingHashTable::Reinitialize (cuckoo_..cc:214-226): status 1 existed, 0 inserted,
// -1 unknown table.  (update_time is wall clock in the reference; passed explicitly here.)
int orc_mtable_reinitialize(orc_mtable* t, int k, const int64_t* ids, int64_t n, int32_t* status,
                            int64_t update_time) {
  if (k < 0 || k >= (int)t->tables.size()) {
    for (int64_t i = 0; i < n; ++i) status[i] = -1;
    return 0;
  }
  Table& tb = t->tables[k];
  for (int64_t i = 0; i < n; ++i) {
    int64_t id = ids[i];
    bool inserted = tb.Upsert(id, [&](Row* r) {
      r->ts = (uint32_t)update_time;
      tb.Init(id, r);
    });
    status[i] = inserted ? 0 : 1;
  }
  return 0;
}

// ref: CuckooEmbeddingHashTable::Evict (cuckoo_embedding_hash_table.cc:251-264)
int orc_mtable_evict(orc_mtable* t, int k, int64_t max_update_time) {
  Table& tb = t->tables[k];
  const int64_t kSecPerDay = 86400;
  for (auto it = tb.m.begin(); it != tb.m.end();) {
    const int64_t timestamp = it->second.ts;
    int64_t expire = tb.default_expire_days;
    auto e = tb.slot_expire.find((uint32_t)SlotIdV2((uint64_t)it->first));
    if (e != tb.slot_expire.end()) expire = e->second;
    if (max_update_time - timestamp >= expire * kSecPerDay) it = tb.m.erase(it);
    else ++it;
  }
  return 0;
}

int orc_mtable_contains(const orc_mtable* t, int k, const int64_t* ids, int64_t n, uint8_t* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = t->tables[k].m.count(ids[i]) ? 1 : 0;
  return 0;
}

// Entry dump in the engine's flat format: [emb | state | found | ts(bits)] per id.
// ref: LookupEntry (cuckoo_..cc:173-183), EntryAccessor::Save (entry_accessor.cc:225-232).
int orc_mtable_lookup_entry(const orc_mtable* t, int k, const int64_t* ids, int64_t n, float* out) {
  const Table& tb = t->tables[k];
  int W = tb.dim + tb.state + 2;
  for (int64_t i = 0; i < n; ++i) {
    float* o = out + i * W;
    auto it = tb.m.find(ids[i]);
    if (it == tb.m.end()) {
      std::memset(o, 0, sizeof(float) * W);
    } else {
      std::memcpy(o, it->second.data.data(), sizeof(float) * (tb.dim + tb.state));
      uint32_t one = 1, ts = it->second.ts;
      std::memcpy(o + tb.dim + tb.state, &one, 4);
      std::memcpy(o + tb.dim + tb.state + 1, &ts, 4);
    }
  }
  return 0;
}

// Export all keys (unordered) — test helper for key-set comparison.
int64_t orc_mtable_keys(const orc_mtable* t, int k, int64_t* out, int64_t cap) {
  int64_t i = 0;
  for (auto& kv : t->tables[k].m) {
    if (i < cap) out[i] = kv.first;
    ++i;
  }
  return i;
}

// ---------------------------------------------------------------------------------------------
// Dedup + shard
// ---------------------------------------------------------------------------------------------

// ref: FusedReorderByIndicesOp::Compute (RT/ops/fused_reorder_by_indices.cc:38-123).
// Returns number of unique ids.  `output` must hold sum(n_m) ids.
int64_t orc_reorder_by_indices(const int64_t* ids, const int64_t* id_split, int K, int N,
                               const int32_t* dims, int rank0_empty, int64_t* output,
                               int32_t* shard_sizes, int32_t* sharded_slot_sizes,
                               int32_t* emb_offset_sz, int32_t* fused_emb_offset) {
  auto shard_func = [&](int64_t v) -> int {
    // :121-123; defined on the unsigned value so that negative FIDs do not index out of range
    // (the reference's int64 % would be negative; identical for v >= 0).
    return (int)((uint64_t)v % (uint64_t)(N - rank0_empty)) + rank0_empty;
  };
  std::vector<std::unordered_map<int64_t, int>> ids_sets(K);
  std::vector<std::vector<int64_t>> ids_for_splits((size_t)K * N);
  for (int m = 0; m < K; ++m) {
    int dim = dims[m];
    for (int64_t i = id_split[m]; i < id_split[m + 1]; ++i) {
      int64_t val = ids[i];
      auto& vec = ids_for_splits[(size_t)shard_func(val) * K + m];
      if (ids_sets[m].insert({val, (int)vec.size() * dim}).second) vec.push_back(val);
    }
  }
  for (int n = 0; n < N; ++n) shard_sizes[n] = 0;
  int64_t uniq = 0;
  int emb_offset = 0;
  std::vector<int> emb_offsets_cm((size_t)K * N);
  for (int n = 0; n < N; ++n)
    for (int m = 0; m < K; ++m) {
      int idx = n * K + m;
      int sz = (int)ids_for_splits[idx].size();
      sharded_slot_sizes[idx] = sz;
      shard_sizes[n] += sz;
      uniq += sz;
      emb_offsets_cm[(size_t)m * N + n] = emb_offset;
      emb_offset += sz * dims[m];
    }
  int64_t* op = output;
  for (auto& vec : ids_for_splits) {
    std::memcpy(op, vec.data(), sizeof(int64_t) * vec.size());
    op += vec.size();
  }
  for (int m = 0; m < K; ++m) {
    if (emb_offset_sz) emb_offset_sz[m] = (int32_t)(id_split[m + 1] - id_split[m]);
    for (int64_t i = id_split[m]; i < id_split[m + 1]; ++i) {
      int64_t val = ids[i];
      fused_emb_offset[i] = ids_sets[m][val] + emb_offsets_cm[(size_t)shard_func(val) + (size_t)m * N];
    }
  }
  return uniq;
}

// First-occurrence dedup of one list (tf.unique semantics; ref: NT/data/kernels/internal/
// uniq_hashtable.h:240-247 uniq_fid returns the first-occurrence ordinal).
int64_t orc_dedup(const int64_t* ids, int64_t n, int64_t* uniq_out, int32_t* inverse) {
  std::unordered_map<int64_t, int32_t> seen;
  seen.reserve((size_t)n * 2);
  int64_t u = 0;
  for (int64_t i = 0; i < n; ++i) {
    auto it = seen.find(ids[i]);
    if (it == seen.end()) {
      seen.emplace(ids[i], (int32_t)u);
      uniq_out[u] = ids[i];
      inverse[i] = (int32_t)u;
      ++u;
    } else {
      inverse[i] = it->second;
    }
  }
  return u;
}

// ---------------------------------------------------------------------------------------------
// Pooling
// ---------------------------------------------------------------------------------------------

// ref: OptimizedSumpooling (RT/ops/fused_embedding_to_layout.cc:26-59): first term assigns, later
// terms add; MEAN divides each term by the fid count.
static inline void SumPool(const float* src, int dim, bool* init, float* dst, int mean_n) {
  if (*init) {
    if (mean_n) for (int i = 0; i < dim; ++i) dst[i] = src[i] / mean_n;
    else std::memcpy(dst, src, sizeof(float) * dim);
    *init = false;
  } else {
    if (mean_n) for (int i = 0; i < dim; ++i) dst[i] += src[i] / mean_n;
    else for (int i = 0; i < dim; ++i) dst[i] += src[i];
  }
}

// Fused lookup + pool oracle: MultiHashTable.lookup followed by the per-row pool.
// SUM == ReduceSumOp (RT/ops/reduce_op.cc:29-51) == GatherEmb SUM
// (fused_embedding_to_layout.h:237-240); MEAN uses GatherEmb semantics (:241-243).
int orc_mtable_lookup_pool(orc_mtable* t, int k, const int64_t* fids, const int32_t* row_offsets,
                           int64_t n_rows, int pooling, float* out, int64_t out_stride,
                           int out_col) {
  const Table& tb = t->tables[k];
  const int D = tb.dim;
  std::vector<float> row(D);
  for (int64_t r = 0; r < n_rows; ++r) {
    int64_t b = row_offsets ? row_offsets[r] : r;
    int64_t e = row_offsets ? row_offsets[r + 1] : r + 1;
    float* dst = out + r * out_stride + out_col;
    std::memset(dst, 0, sizeof(float) * D);
    bool init = true;
    int n = (int)(e - b);
    for (int64_t i = b; i < e; ++i) {
      TableLookup(tb, fids + i, 1, row.data());
      SumPool(row.data(), D, &init, dst, pooling == MONO_POOL_MEAN ? n : 0);
    }
  }
  return 0;
}

// ref: FusedGatherKernel (RT/ops/map_id_to_embedding.cu.cc:30-74) + per-row pool.
int orc_gather_pool(const float* fused_emb, const int32_t* emb_offset, const int32_t* row_offsets,
                    int64_t n_rows, int dim, int pooling, float* out, int64_t out_stride,
                    int out_col) {
  for (int64_t r = 0; r < n_rows; ++r) {
    int64_t b = row_offsets ? row_offsets[r] : r;
    int64_t e = row_offsets ? row_offsets[r + 1] : r + 1;
    float* dst = out + r * out_stride + out_col;
    std::memset(dst, 0, sizeof(float) * dim);
    bool init = true;
    int n = (int)(e - b);
    for (int64_t i = b; i < e; ++i)
      SumPool(fused_emb + emb_offset[i], dim, &init, dst, pooling == MONO_POOL_MEAN ? n : 0);
  }
  return 0;
}

// ref: FusedGatherGradKernel (map_id_to_embedding.cu.cc:75-118) / ScatterGrad
// (fused_embedding_to_layout.h:286-347): grad_fused[offset[m]] += g (SUM) or g/n (MEAN), in
// occurrence order (the CPU reference order; the GPU reference uses atomics).
int orc_gather_pool_grad(const float* pooled_grad, int64_t grad_stride, int grad_col,
                         const int32_t* emb_offset, const int32_t* row_offsets, int64_t n_rows,
                         int dim, int pooling, float* grad_fused) {
  for (int64_t r = 0; r < n_rows; ++r) {
    int64_t b = row_offsets ? row_offsets[r] : r;
    int64_t e = row_offsets ? row_offsets[r + 1] : r + 1;
    const float* g = pooled_grad + r * grad_stride + grad_col;
    int n = (int)(e - b);
    for (int64_t i = b; i < e; ++i) {
      float* dst = grad_fused + emb_offset[i];
      if (pooling == MONO_POOL_MEAN) for (int j = 0; j < dim; ++j) dst[j] += g[j] / n;
      else for (int j = 0; j < dim; ++j) dst[j] += g[j];
    }
  }
  return 0;
}

// ref: ParseFidOffset / ParseNflOffset / GetFeatureInfo (fused_embedding_to_layout.h:50-76)
static inline void GetFeatureInfo(int nfl_idx, const uint32_t* nfl_offset, int total_nfl,
                                  int total_feature, bool* is_shared, int* off, int* feature_num) {
  *is_shared = nfl_offset[nfl_idx] >> 31;
  *off = nfl_offset[nfl_idx] & 0x7fffffff;
  if (nfl_idx < total_nfl - 1) *feature_num = (int)(nfl_offset[nfl_idx + 1] & 0x7fffffff) - *off;
  else *feature_num = total_feature - *off;
}

// ref: MonolithEmbeddingToLayoutOp::TaskRun + ForwardTaskRunImpl + GatherEmb
// (fused_embedding_to_layout.cc:542-606,608-676; .h:204-261), versions 3/4/5 (PtrWrapper.offset
// given per list in emb_strides).  Tasks are the flattened (layout, slice_config) pairs in the
// reference's iteration order (layouts sorted by name, slices in config order).
int orc_embedding_to_layout(const float* const* emb_ptrs, const int32_t* emb_strides, int n_emb,
                            const uint64_t* fid_offset, int64_t total_fid,
                            const int32_t* feature_offset, int total_feature,
                            const uint32_t* nfl_offset, int total_nfl, int batch_size,
                            const mono_slice_task* tasks, int n_tasks, float* const* out_ptrs,
                            const int64_t* out_sizes, int n_out) {
  (void)n_emb;
  for (int o = 0; o < n_out; ++o) std::memset(out_ptrs[o], 0, sizeof(float) * out_sizes[o]);
  for (int ti = 0; ti < n_tasks; ++ti) {
    const mono_slice_task& tk = tasks[ti];
    bool is_shared; int nfl_off, feature_num;
    GetFeatureInfo(tk.nfl_idx, nfl_offset, total_nfl, total_feature, &is_shared, &nfl_off,
                   &feature_num);
    if (!feature_num) continue;
    float* base = out_ptrs[tk.out_tensor] + tk.out_col;
    std::vector<float> tmp;
    if (is_shared && tk.accumulate) tmp.assign(tk.dim, 0.f);
    int feature_idx = nfl_off;
    for (int b = 0; b < batch_size; ++b) {
      float* dst_row = base + (int64_t)b * tk.out_row_stride;
      if (!is_shared || b == 0) {
        bool init = (!tk.accumulate) || !tmp.empty();
        float* dst = tmp.empty() ? dst_row : tmp.data();
        // GatherEmb
        int fid_num = (feature_idx < total_feature - 1)
                          ? feature_offset[feature_idx + 1] - feature_offset[feature_idx]
                          : (int)total_fid - feature_offset[feature_idx];
        int start = feature_offset[feature_idx];
        int seq_idx = 0;
        for (int f = 0; f < fid_num; ++f) {
          uint64_t fo = fid_offset[start + f];
          int index1 = (int)(fo >> 32), index2 = (int)(fo & 0xffffffffu);
          const float* src = emb_ptrs[index1] + (int64_t)index2 * emb_strides[index1] + tk.slice_start;
          switch (tk.pooling) {
            case MONO_POOL_SUM: SumPool(src, tk.dim, &init, dst, 0); break;
            case MONO_POOL_MEAN: SumPool(src, tk.dim, &init, dst, fid_num); break;
            case MONO_POOL_FIRSTN:
              if (seq_idx < tk.max_seq_len)
                std::memcpy(dst + seq_idx * tk.dim, src, sizeof(float) * tk.dim);
              seq_idx++;
              break;
          }
        }
        if (!tmp.empty()) {
          bool init_tmp = false;  // ADDN output rows were zero-filled; always accumulate
          SumPool(tmp.data(), tk.dim, &init_tmp, dst_row, 0);
        }
        feature_idx++;
      } else {
        if (!tmp.empty()) {
          bool init_tmp = false;
          SumPool(tmp.data(), tk.dim, &init_tmp, dst_row, 0);
        } else {
          int n = tk.pooling == MONO_POOL_FIRSTN ? tk.dim * tk.max_seq_len : tk.dim;
          std::memcpy(dst_row, base, sizeof(float) * n);
        }
      }
    }
  }
  return 0;
}

// ref: MonolithEmbeddingToLayoutGradOp::TaskRun + ScatterGrad
// (fused_embedding_to_layout.cc:895-948; .h:286-347), versions 3/4/5 (no init map: outputs are
// zero-filled and every term accumulates).
int orc_embedding_to_layout_grad(float* const* emb_grad_ptrs, const int32_t* emb_strides,
                                 const int64_t* emb_sizes, int n_emb, const uint64_t* fid_offset,
                                 int64_t total_fid, const int32_t* feature_offset,
                                 int total_feature, const uint32_t* nfl_offset, int total_nfl,
                                 int batch_size, const mono_slice_task* tasks, int n_tasks,
                                 const float* const* out_grad_ptrs) {
  for (int e = 0; e < n_emb; ++e) std::memset(emb_grad_ptrs[e], 0, sizeof(float) * emb_sizes[e]);
  for (int ti = 0; ti < n_tasks; ++ti) {
    const mono_slice_task& tk = tasks[ti];
    bool is_shared; int nfl_off, feature_num;
    GetFeatureInfo(tk.nfl_idx, nfl_offset, total_nfl, total_feature, &is_shared, &nfl_off,
                   &feature_num);
    if (!feature_num) continue;
    const float* base = out_grad_ptrs[tk.out_tensor] + tk.out_col;
    int feature_idx = nfl_off;
    for (int b = 0; b < batch_size; ++b) {
      const float* g = base + (int64_t)b * tk.out_row_stride;
      int fid_num = (feature_idx < total_feature - 1)
                        ? feature_offset[feature_idx + 1] - feature_offset[feature_idx]
                        : (int)total_fid - feature_offset[feature_idx];
      int start = feature_offset[feature_idx];
      int seq_idx = 0;
      for (int f = 0; f < fid_num; ++f) {
        uint64_t fo = fid_offset[start + f];
        int index1 = (int)(fo >> 32), index2 = (int)(fo & 0xffffffffu);
        float* dst = emb_grad_ptrs[index1] + (int64_t)index2 * emb_strides[index1] + tk.slice_start;
        switch (tk.pooling) {
          case MONO_POOL_SUM: for (int j = 0; j < tk.dim; ++j) dst[j] += g[j]; break;
          case MONO_POOL_MEAN: for (int j = 0; j < tk.dim; ++j) dst[j] += g[j] / fid_num; break;
          case MONO_POOL_FIRSTN:
            if (seq_idx < tk.max_seq_len)
              for (int j = 0; j < tk.dim; ++j) dst[j] += g[seq_idx * tk.dim + j];
            seq_idx++;
            break;
        }
      }
      if (!is_shared) feature_idx++;
    }
  }
  return 0;
}

// Single-row optimizer steps exposed for known-answer tests (ref: optimizer/*_optimizer_test.cc).
void orc_adagrad(float* num, float* norm, const float* grad, int64_t len, float lr, float wd) {
  AdagradOptimize(num, norm, grad, (size_t)len, lr, wd);
}
void orc_ftrl(float* num, float* norm, float* zero, const float* grad, int dim, float lr,
              float beta, float l1, float l2) {
  FtrlOptimize(num, norm, zero, grad, dim, lr, beta, l1, l2);
}
void orc_adam(float* num, float* m, float* v, float* b1p, float* b2p, const float* grad, int dim,
              float lr, float beta1, float beta2, float eps, float wd, int nesterov) {
  AdamOptimize(num, m, v, b1p, b2p, grad, dim, lr, beta1, beta2, eps, wd, nesterov != 0);
}
void orc_sgd(float* num, const float* grad, int dim, float lr) { SgdOptimize(num, grad, dim, lr); }
float orc_uniform_init(uint64_t seed, int64_t fid, int col, float lo, float hi) {
  return UniformInit(seed, fid, col, lo, hi);
}

// ---------------------------------------------------------------------------------------------
// CPU parameter-server baseline (timed by bench.py).  Same per-id find/upsert structure as the
// reference PS: `num_ps` in-process shards (fid % num_ps, ref: NT/distributed_ps.py:289), one
// worker thread per shard, per-id Span-style row access, reference Adagrad math.  This is the
// "CPU restatement of the reference PS path (reference build unavailable: no bazel/TF)".
// ---------------------------------------------------------------------------------------------
struct orc_ps {
  int num_ps;
  std::vector<std::unique_ptr<orc_mtable>> shards;
};

int orc_ps_create(const mono_table_cfg* cfg, int num_ps, orc_ps** out) {
  auto ps = std::make_unique<orc_ps>();
  ps->num_ps = num_ps;
  for (int i = 0; i < num_ps; ++i) {
    orc_mtable* m = nullptr;
    orc_mtable_create(cfg, 1, &m);
    ps->shards.emplace_back(m);
  }
  *out = ps.release();
  return 0;
}
int orc_ps_destroy(orc_ps* ps) { delete ps; return 0; }

}  // extern "C"
template <class F>
static void ParallelShards(int n, F f) {
  std::vector<std::thread> th;
  for (int i = 0; i < n; ++i) th.emplace_back([&, i] { f(i); });
  for (auto& t : th) t.join();
}
extern "C" {

// Bulk insert keys with default-initialised rows (table pre-fill).
int orc_ps_fill(orc_ps* ps, const int64_t* ids, int64_t n) {
  ParallelShards(ps->num_ps, [&](int s) {
    Table& tb = ps->shards[s]->tables[0];
    for (int64_t i = 0; i < n; ++i)
      if ((int)((uint64_t)ids[i] % (uint64_t)ps->num_ps) == s) tb.Upsert(ids[i], [](Row*) {});
  });
  return 0;
}

// One forward step: every shard looks up its FIDs; rows are pooled (SUM / MEAN) per output row.
// Mirrors: worker splits ids by shard -> PS lookup -> gather back -> ReduceSum.
int orc_ps_lookup_pool(orc_ps* ps, const int64_t* fids, const int32_t* row_offsets, int64_t n_rows,
                       int64_t n_fids, int pooling, float* out) {
  const int D = ps->shards[0]->tables[0].dim;
  std::vector<float> rows((size_t)n_fids * D);
  ParallelShards(ps->num_ps, [&](int s) {
    const Table& tb = ps->shards[s]->tables[0];
    for (int64_t i = 0; i < n_fids; ++i)
      if ((int)((uint64_t)fids[i] % (uint64_t)ps->num_ps) == s)
        TableLookup(tb, fids + i, 1, rows.data() + i * D);
  });
  int nt = ps->num_ps;
  ParallelShards(nt, [&](int s) {
    int64_t r0 = n_rows * s / nt, r1 = n_rows * (s + 1) / nt;
    for (int64_t r = r0; r < r1; ++r) {
      int64_t b = row_offsets ? row_offsets[r] : r, e = row_offsets ? row_offsets[r + 1] : r + 1;
      float* dst = out + r * D;
      std::memset(dst, 0, sizeof(float) * D);
      bool init = true;
      for (int64_t i = b; i < e; ++i)
        SumPool(rows.data() + i * D, D, &init, dst, pooling == MONO_POOL_MEAN ? (int)(e - b) : 0);
    }
  });
  return 0;
}

// One backward step: unique ids + their grads are routed to the owning shard and applied.
int orc_ps_optimize(orc_ps* ps, const int64_t* ids, int64_t n, const float* grads, const float* lr,
                    int64_t update_time) {
  ParallelShards(ps->num_ps, [&](int s) {
    Table& tb = ps->shards[s]->tables[0];
    tb.BumpMaxTs(update_time);
    const int D = tb.dim;
    for (int64_t i = 0; i < n; ++i)
      if ((int)((uint64_t)ids[i] % (uint64_t)ps->num_ps) == s) {
        const float* g = grads + i * D;
        tb.Upsert(ids[i], [&](Row* r) { r->ts = (uint32_t)update_time; tb.Optimize(r, g, lr); });
      }
  });
  return 0;
}

int64_t orc_ps_size(const orc_ps* ps) {
  int64_t n = 0;
  for (auto& s : ps->shards) n += (int64_t)s->tables[0].m.size();
  return n;
}

// Pre-fill: keys (slot << 48) | rank for slot in [1, n_slots], rank in [0, keys_per_slot)
// (ref FID layout: reader_util.h:67-69 GetFidV2), default-initialised rows, generated in C.
int orc_ps_fill_slots(orc_ps* ps, int n_slots, int64_t keys_per_slot) {
  ParallelShards(ps->num_ps, [&](int s) {
    Table& tb = ps->shards[s]->tables[0];
    tb.m.reserve((size_t)(n_slots * keys_per_slot / ps->num_ps * 1.1));
    for (int sl = 1; sl <= n_slots; ++sl)
      for (int64_t r = 0; r < keys_per_slot; ++r) {
        int64_t fid = (int64_t)(((uint64_t)sl << 48) | (uint64_t)r);
        if ((int)((uint64_t)fid % (uint64_t)ps->num_ps) == s) tb.Upsert(fid, [](Row*) {});
      }
  });
  return 0;
}

// One full sparse train step of the reference's CPU parameter-server path, one worker:
//   1. FusedReorderByIndices (serial per-op loop, fused_reorder_by_indices.cc:38-117): dedup + shard
//   2. per-PS lookup of its unique FIDs (one thread per PS shard, distributed_ps.py:289-319)
//   3. gather + per-row pool on the worker (map_id_to_embedding / reduce ops), threads over rows
//   4. backward: scatter pooled grads to unique rows (ScatterGrad; threads over destination ranges,
//      deterministic), then per-PS Optimize of its FIDs (multi_hash_table_update_op.cc:47-89)
// fids: M occurrences, row r pools fids[row_offsets[r]:row_offsets[r+1]] (NULL: one per row).
// Returns the number of unique FIDs.
int64_t orc_ps_train_step(orc_ps* ps, const int64_t* fids, int64_t M, const int32_t* row_offsets,
                          int64_t n_rows, int pooling, const float* pooled_grad, float* pooled_out,
                          const float* lr, int64_t update_time) {
  const int N = ps->num_ps;
  const int D = ps->shards[0]->tables[0].dim;
  const int32_t dims[1] = {D};
  const int64_t split[2] = {0, M};
  std::vector<int64_t> uniq((size_t)M);
  std::vector<int32_t> shard_sizes(N), slot_sizes(N), offs((size_t)M);
  int32_t sz1;
  int64_t U = orc_reorder_by_indices(fids, split, 1, N, dims, 0, uniq.data(), shard_sizes.data(),
                                     slot_sizes.data(), &sz1, offs.data());
  std::vector<int64_t> base(N + 1, 0);
  for (int s = 0; s < N; ++s) base[s + 1] = base[s] + shard_sizes[s];
  std::vector<float> rows((size_t)U * D), ugrad((size_t)U * D, 0.f);
  ParallelShards(N, [&](int s) {
    TableLookup(ps->shards[s]->tables[0], uniq.data() + base[s], shard_sizes[s], rows.data() + base[s] * D);
  });
  ParallelShards(N, [&](int s) {
    int64_t r0 = n_rows * s / N, r1 = n_rows * (s + 1) / N;
    for (int64_t r = r0; r < r1; ++r) {  // orc_gather_pool, rows [r0, r1)
      int64_t b = row_offsets ? row_offsets[r] : r, e = row_offsets ? row_offsets[r + 1] : r + 1;
      float* dst = pooled_out + r * D;
      std::memset(dst, 0, sizeof(float) * D);
      bool init = true;
      for (int64_t i = b; i < e; ++i)
        SumPool(rows.data() + offs[i], D, &init, dst, pooling == MONO_POOL_MEAN ? (int)(e - b) : 0);
    }
  });
  ParallelShards(N, [&](int s) {  // destination-range partition: thread s owns rows of shard s
    const int64_t lo = base[s] * D, hi = base[s + 1] * D;
    for (int64_t r = 0; r < n_rows; ++r) {
      int64_t b = row_offsets ? row_offsets[r] : r, e = row_offsets ? row_offsets[r + 1] : r + 1;
      const float* g = pooled_grad + r * D;
      int n = (int)(e - b);
      for (int64_t i = b; i < e; ++i) {
        if (offs[i] < lo || offs[i] >= hi) continue;
        float* dst = ugrad.data() + offs[i];
        if (pooling == MONO_POOL_MEAN) for (int j = 0; j < D; ++j) dst[j] += g[j] / n;
        else for (int j = 0; j < D; ++j) dst[j] += g[j];
      }
    }
  });
  ParallelShards(N, [&](int s) {
    Table& tb = ps->shards[s]->tables[0];
    TableBatchOptimize(&tb, uniq.data() + base[s], shard_sizes[s], ugrad.data() + base[s] * D, lr,
                       update_time, false);
  });
  return U;
}

}  // extern "C"

// =============================================================================================
// Tuned CPU parameter-server baseline ("fastps") — what bench.py's reference arm / cpu_baseline time.
// TEST / BENCH INFRASTRUCTURE (never linked into the product).  Same algorithm and results as
// orc_ps_train_step above (checked bit for bit by tests/test_oracle_golden.py), engineered the way the
// reference engineers its PS so that the baseline is not sand-bagged:
//   * persistent worker pool (the reference PS serves from a long-lived TF thread pool; no thread is
//     created per step),
//   * every shard a flat open-addressing map fid -> row index over one contiguous row slab
//     [dim embedding | state] (the reference: libcuckoo map + block allocator,
//     RT/hash_table/cuckoohash/cuckoo_embedding_hash_table.cc:120-171, RT/allocator/block_allocator.h),
//   * the worker-side dedup + shard split (FusedReorderByIndices, fused_reorder_by_indices.cc:38-123) is
//     partitioned over the threads (positions -> per-shard lists -> per-shard first-occurrence dedup),
//   * the gradient scatter (ScatterGrad, fused_embedding_to_layout.h:286-347) is partitioned by
//     destination shard over that shard's own occurrence list — no thread ever scans foreign rows,
//   * Adagrad is the reference's AVX form (avx_utils.h:96-119) via AdagradOptimize, compiled -O3 -mavx2 -mfma.
// The hot FID order of the sums is occurrence order, as in the reference's CPU path.
// =============================================================================================
#include <condition_variable>

namespace fastps {

class Pool {  // persistent workers; run(f) executes f(tid) on every worker and returns when all are done
 public:
  explicit Pool(int n) : n_(n) {
    for (int i = 0; i < n; ++i) th_.emplace_back([this, i] { Loop(i); });
  }
  ~Pool() {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
      ++gen_;
    }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  int size() const { return n_; }
  template <class F>
  void run(F f) {
    fn_ = [&f](int i) { f(i); };
    done_.store(0, std::memory_order_relaxed);
    {
      std::lock_guard<std::mutex> lk(mu_);
      ++gen_;
    }
    cv_.notify_all();
    // the caller spins briefly, then sleeps: steps are milliseconds long
    int spins = 0;
    while (done_.load(std::memory_order_acquire) != n_) {
      if (++spins > 2000) std::this_thread::yield();
    }
  }

 private:
  void Loop(int i) {
    uint64_t seen = 0;
    while (true) {
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
      }
      fn_(i);
      done_.fetch_add(1, std::memory_order_release);
    }
  }
  int n_;
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_;
  uint64_t gen_ = 0;
  bool stop_ = false;
  std::function<void(int)> fn_;
  std::atomic<int> done_{0};
};

struct Shard {
  int dim = 0, state = 0, W = 0;
  const Table* proto = nullptr;  // config (segments, seed): Init / Optimize come from the oracle Table
  std::vector<int64_t> keys;
  std::vector<uint32_t> rowidx;  // 0xFFFFFFFF = empty
  std::vector<float> rows;       // [n][W]
  std::vector<uint32_t> ts;
  uint64_t mask = 0, n = 0;

  void Reserve(uint64_t want) {
    uint64_t cap = 1024;
    while (cap < 2 * want) cap <<= 1;
    if (cap <= keys.size()) return;
    std::vector<int64_t> ok;
    std::vector<uint32_t> orow;
    ok.swap(keys);
    orow.swap(rowidx);
    keys.assign(cap, 0);
    rowidx.assign(cap, 0xFFFFFFFFu);
    mask = cap - 1;
    for (size_t i = 0; i < ok.size(); ++i)
      if (orow[i] != 0xFFFFFFFFu) {
        uint64_t h = Mix64((uint64_t)ok[i]) & mask;
        while (rowidx[h] != 0xFFFFFFFFu) h = (h + 1) & mask;
        keys[h] = ok[i];
        rowidx[h] = orow[i];
      }
  }
  inline uint32_t Find(int64_t fid) const {
    uint64_t h = Mix64((uint64_t)fid) & mask;
    while (true) {
      const uint32_t r = rowidx[h];
      if (r == 0xFFFFFFFFu) return r;
      if (keys[h] == fid) return r;
      h = (h + 1) & mask;
    }
  }
  // find or insert; a new row is initialised like EntryAccessor::Init (initializer, then optimizer Init)
  inline uint32_t Upsert(int64_t fid) {
    if (2 * (n + 1) > keys.size()) Reserve(n + 1 + n / 2);
    uint64_t h = Mix64((uint64_t)fid) & mask;
    while (true) {
      const uint32_t r = rowidx[h];
      if (r == 0xFFFFFFFFu) break;
      if (keys[h] == fid) return r;
      h = (h + 1) & mask;
    }
    const uint32_t r = (uint32_t)n++;
    keys[h] = fid;
    rowidx[h] = r;
    if (rows.size() < (size_t)n * W) rows.resize(std::max(rows.size() * 2, (size_t)n * W));
    if (ts.size() < n) ts.resize(std::max<size_t>(ts.size() * 2, n));
    Row tmp;
    proto->Init(fid, &tmp);
    std::memcpy(rows.data() + (size_t)r * W, tmp.data.data(), sizeof(float) * W);
    ts[r] = 0;
    return r;
  }
};

struct DedupSet {  // scratch first-occurrence set of one shard, reused across steps
  std::vector<int64_t> keys;
  std::vector<int32_t> val;  // -1 = empty
  uint64_t mask = 0;
  void Reset(size_t want) {
    uint64_t cap = 1024;
    while (cap < 2 * want) cap <<= 1;
    if (cap != keys.size()) {
      keys.assign(cap, 0);
      val.assign(cap, -1);
      mask = cap - 1;
    } else {
      std::fill(val.begin(), val.end(), -1);
    }
  }
};

struct PS {
  int T = 1;
  Table proto;
  std::unique_ptr<Pool> pool;
  std::vector<Shard> shards;
  // per-step scratch (kept between steps)
  std::vector<std::vector<std::vector<uint32_t>>> part;  // [thread][shard] -> positions
  std::vector<DedupSet> sets;
  std::vector<std::vector<int64_t>> uniq;      // [shard]
  std::vector<std::vector<uint32_t>> occ_pos;  // [shard] positions in order
  std::vector<std::vector<uint32_t>> occ_loc;  // [shard] local unique index of each of them
  std::vector<std::vector<float>> rows, ugrad; // [shard][U_s * D]
  std::vector<uint32_t> loc;                   // [M] local unique index
  std::vector<uint16_t> sh;                    // [M] shard
};

}  // namespace fastps

extern "C" {

struct orc_fastps : fastps::PS {};

int orc_fastps_create(const mono_table_cfg* cfg, int threads, orc_fastps** out) {
  auto ps = std::make_unique<orc_fastps>();
  orc_mtable* m = nullptr;
  orc_mtable_create(cfg, 1, &m);
  ps->proto = m->tables[0];
  ps->proto.m.clear();
  orc_mtable_destroy(m);
  ps->T = std::max(1, threads);
  ps->pool = std::make_unique<fastps::Pool>(ps->T);
  ps->shards.resize(ps->T);
  for (auto& s : ps->shards) {
    s.dim = ps->proto.dim;
    s.state = ps->proto.state;
    s.W = s.dim + s.state;
    s.proto = &ps->proto;
  }
  ps->part.assign(ps->T, std::vector<std::vector<uint32_t>>(ps->T));
  ps->sets.resize(ps->T);
  ps->uniq.resize(ps->T);
  ps->occ_pos.resize(ps->T);
  ps->occ_loc.resize(ps->T);
  ps->rows.resize(ps->T);
  ps->ugrad.resize(ps->T);
  *out = ps.release();
  return 0;
}
int orc_fastps_destroy(orc_fastps* ps) { delete ps; return 0; }

int orc_fastps_fill_slots(orc_fastps* ps, int n_slots, int64_t keys_per_slot) {
  const int T = ps->T;
  ps->pool->run([&](int s) {
    fastps::Shard& sd = ps->shards[s];
    sd.Reserve((uint64_t)(n_slots * keys_per_slot / T * 1.1) + 16);
    for (int sl = 1; sl <= n_slots; ++sl)
      for (int64_t r = 0; r < keys_per_slot; ++r) {
        const int64_t fid = (int64_t)(((uint64_t)sl << 48) | (uint64_t)r);
        if ((int)((uint64_t)fid % (uint64_t)T) == s) sd.Upsert(fid);
      }
  });
  return 0;
}

int64_t orc_fastps_size(const orc_fastps* ps) {
  int64_t n = 0;
  for (auto& s : ps->shards) n += (int64_t)s.n;
  return n;
}

// raw entry [emb | state] of a FID (zeros when absent) — for the equality test against the oracle tables
int orc_fastps_entry(const orc_fastps* ps, int64_t fid, float* out) {
  const fastps::Shard& sd = ps->shards[(uint64_t)fid % (uint64_t)ps->T];
  const uint32_t r = sd.Find(fid);
  if (r == 0xFFFFFFFFu) {
    std::memset(out, 0, sizeof(float) * sd.W);
    return 0;
  }
  std::memcpy(out, sd.rows.data() + (size_t)r * sd.W, sizeof(float) * sd.W);
  return 1;
}

// One full sparse train step (same contract as orc_ps_train_step); returns the number of unique FIDs.
int64_t orc_fastps_train_step(orc_fastps* ps, const int64_t* fids, int64_t M, const int32_t* row_offsets,
                              int64_t n_rows, int pooling, const float* pooled_grad, float* pooled_out,
                              const float* lr, int64_t update_time) {
  using namespace fastps;
  const int T = ps->T;
  const int D = ps->proto.dim;
  if ((int64_t)ps->loc.size() < M) {
    ps->loc.resize((size_t)M);
    ps->sh.resize((size_t)M);
  }
  std::vector<uint32_t> occ_row;  // occurrence -> pooled row (CSR input only)
  if (row_offsets) {
    occ_row.resize((size_t)M);
    ps->pool->run([&](int t) {
      for (int64_t r = n_rows * t / T; r < n_rows * (t + 1) / T; ++r)
        for (int32_t i = row_offsets[r]; i < row_offsets[r + 1]; ++i) occ_row[i] = (uint32_t)r;
    });
  }
  // 1a. worker-side shard split (FusedReorderByIndices, first half): positions -> per-shard lists
  ps->pool->run([&](int t) {
    auto& mine = ps->part[t];
    for (auto& v : mine) v.clear();
    const int64_t b = M * t / T, e = M * (t + 1) / T;
    for (int64_t i = b; i < e; ++i) {
      const int s = (int)((uint64_t)fids[i] % (uint64_t)T);
      mine[s].push_back((uint32_t)i);
      ps->sh[i] = (uint16_t)s;
    }
  });
  // 1b + 2. per shard: first-occurrence dedup of its positions (chunks in order => position order), then the
  //          PS-side lookup of the distinct FIDs (per-id find, miss -> zeros)
  ps->pool->run([&](int s) {
    size_t cnt = 0;
    for (int t = 0; t < T; ++t) cnt += ps->part[t][s].size();
    DedupSet& ds = ps->sets[s];
    ds.Reset(cnt);
    auto& uq = ps->uniq[s];
    auto& op = ps->occ_pos[s];
    auto& ol = ps->occ_loc[s];
    uq.clear();
    op.clear();
    ol.clear();
    for (int t = 0; t < T; ++t)
      for (uint32_t pos : ps->part[t][s]) {
        const int64_t fid = fids[pos];
        uint64_t h = Mix64((uint64_t)fid * 0x9E3779B97F4A7C15ULL) & ds.mask;
        int32_t u;
        while (true) {
          if (ds.val[h] < 0) {
            u = (int32_t)uq.size();
            ds.keys[h] = fid;
            ds.val[h] = u;
            uq.push_back(fid);
            break;
          }
          if (ds.keys[h] == fid) { u = ds.val[h]; break; }
          h = (h + 1) & ds.mask;
        }
        ps->loc[pos] = (uint32_t)u;
        op.push_back(pos);
        ol.push_back((uint32_t)u);
      }
    const Shard& sd = ps->shards[s];
    auto& rw = ps->rows[s];
    rw.resize(uq.size() * (size_t)D);
    for (size_t u = 0; u < uq.size(); ++u) {
      const uint32_t r = sd.Find(uq[u]);
      if (r == 0xFFFFFFFFu) std::memset(rw.data() + u * D, 0, sizeof(float) * D);
      else std::memcpy(rw.data() + u * D, sd.rows.data() + (size_t)r * sd.W, sizeof(float) * D);
    }
  });
  // 3. worker-side gather + per-row pool, threads over row ranges
  ps->pool->run([&](int t) {
    const int64_t r0 = n_rows * t / T, r1 = n_rows * (t + 1) / T;
    for (int64_t r = r0; r < r1; ++r) {
      const int64_t b = row_offsets ? row_offsets[r] : r, e = row_offsets ? row_offsets[r + 1] : r + 1;
      float* dst = pooled_out + r * D;
      std::memset(dst, 0, sizeof(float) * D);
      bool init = true;
      for (int64_t i = b; i < e; ++i)
        SumPool(ps->rows[ps->sh[i]].data() + (size_t)ps->loc[i] * D, D, &init, dst,
                pooling == MONO_POOL_MEAN ? (int)(e - b) : 0);
    }
  });
  // 4. backward: per shard, scatter the pooled grads of ITS occurrences (position order) to its unique rows,
  //    then the PS-side optimize of those rows (upsert + Adagrad/... + timestamp)
  ps->pool->run([&](int s) {
    auto& ug = ps->ugrad[s];
    const size_t U = ps->uniq[s].size();
    ug.assign(U * (size_t)D, 0.f);
    const auto& op = ps->occ_pos[s];
    const auto& ol = ps->occ_loc[s];
    for (size_t q = 0; q < op.size(); ++q) {
      const uint32_t pos = op[q];
      const int64_t r = row_offsets ? (int64_t)occ_row[pos] : (int64_t)pos;
      const float* g = pooled_grad + r * D;
      float* dst = ug.data() + (size_t)ol[q] * D;
      if (pooling == MONO_POOL_MEAN && row_offsets) {
        const float n = (float)(row_offsets[r + 1] - row_offsets[r]);
        for (int j = 0; j < D; ++j) dst[j] += g[j] / n;
      } else {
        for (int j = 0; j < D; ++j) dst[j] += g[j];
      }
    }
    Shard& sd = ps->shards[s];
    Row tmp;
    tmp.data.resize(sd.W);
    for (size_t u = 0; u < U; ++u) {
      const uint32_t r = sd.Upsert(ps->uniq[s][u]);
      float* row = sd.rows.data() + (size_t)r * sd.W;
      if (ps->proto.segs.size() == 1 && ps->proto.segs[0].opt_type == MONO_OPT_ADAGRAD) {
        AdagradOptimize(row, row + D, ug.data() + u * D, (size_t)D, lr[0], ps->proto.segs[0].opt_p[1]);
      } else {  // any segment mix: through the oracle's CombinedOptimizer restatement
        std::memcpy(tmp.data.data(), row, sizeof(float) * sd.W);
        ps->proto.Optimize(&tmp, ug.data() + u * D, lr);
        std::memcpy(row, tmp.data.data(), sizeof(float) * sd.W);
      }
      sd.ts[r] = (uint32_t)update_time;
    }
  });
  int64_t U = 0;
  for (int s = 0; s < T; ++s) U += (int64_t)ps->uniq[s].size();
  return U;
}

}  // extern "C"
