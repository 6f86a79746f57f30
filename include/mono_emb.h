/*
 * mono_emb.h — C ABI of the H100-native collisionless-embedding engine.
 *
 * This is the drop-in boundary for the hot path of bytedance/monolith:
 *   MultiHashTable.lookup / assign / assign_add / reinitialize / apply_gradients /
 *   fused_lookup / fused_apply_gradient, plus the dedup+shard and pooling ops around them.
 *
 * The reference has no C ABI (its boundary is TF OpKernels over a ResourceBase); every entry
 * point below names the reference op / function it replaces ("ref:" = path under
 * monolith/native_training/, RT = runtime/).  A reference maintainer binds these from a
 * TF custom-op shim (INTEGRATION.md) or from Python ctypes (monolith_b200/_lib.py).
 *
 * Conventions
 *   - plain C types only; no torch / TF types.
 *   - every function returns 0 on success or a negative mono_status code; the message is in
 *     mono_last_error() (thread-local).  No C++ exception crosses this boundary
 *     (ref: RT/ops/embedding_hash_table_tf_bridge.cc:132-134 converts exceptions to Status).
 *   - pointers named *_dev are CUDA device pointers on the table's device; pointers named
 *     *_host are ordinary host memory.  `stream` is a cudaStream_t passed as void*
 *     (NULL = legacy default stream).  Calls on one stream are ordered; the library never
 *     synchronises the device except where documented ("SYNC").
 *   - table order inside a multi-table is sorted-by-name (ref: multi_hash_table_ops.py:72,83).
 *   - there is NO CPU fallback: every compute entry point runs hand-written sm_90a kernels and
 *     fails with MONO_ERR_CUDA if no device is present.
 */
#ifndef MONO_EMB_H_
#define MONO_EMB_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MONO_EMB_ABI_VERSION 1

typedef enum mono_status {
  MONO_OK = 0,
  MONO_ERR_INVALID_ARGUMENT = -1, /* ref: errors::InvalidArgument (lookup / update ops) */
  MONO_ERR_RESOURCE_EXHAUSTED = -2, /* ref: errors::ResourceExhausted (save / restore / alloc) */
  MONO_ERR_CUDA = -3,
  MONO_ERR_INTERNAL = -4
} mono_status;

/* ---- table configuration: plain-struct equivalent of MultiEmbeddingHashTableConfig
 *      (ref: RT/hash_table/embedding_hash_table.proto:23-96, optimizer/optimizer.proto,
 *      initializer/initializer_config.proto) ------------------------------------------------ */

typedef enum mono_opt_type {
  MONO_OPT_SGD = 0,     /* ref: RT/hash_table/optimizer/sgd_optimizer.cc:42-49      */
  MONO_OPT_ADAGRAD = 1, /* ref: optimizer/adagrad_optimizer.cc:54-60, avx_utils.h   */
  MONO_OPT_FTRL = 2,    /* ref: optimizer/ftrl_optimizer.cc:56-76                   */
  MONO_OPT_ADAM = 3,    /* ref: optimizer/adam_optimizer.cc:57-84                   */
  /* further optimizers of RT/hash_table/optimizer/optimizer.proto:210-227 (SURVEY 8(f) row 4): served by the
   * generic per-element apply path (any segment mix), not by the single-segment vector fast paths */
  MONO_OPT_MOMENTUM = 4,  /* ref: optimizer/momentum_optimizer.cc:52-72              */
  MONO_OPT_RMSPROP = 5,   /* ref: optimizer/rmsprop_optimizer.cc:49-68 (double arithmetic, CONFIG learning rate) */
  MONO_OPT_RMSPROPV2 = 6, /* ref: optimizer/rmsprop_optimizer.cc:121-141             */
  MONO_OPT_ADADELTA = 7,  /* ref: optimizer/adadelta_optimizer.cc:51-72              */
  MONO_OPT_AMSGRAD = 8,   /* ref: optimizer/amsgrad_optimizer.cc:58-88               */
  MONO_OPT_MOVING_AVERAGE = 9, /* ref: optimizer/moving_average_optimizer.cc:44-52 (no state, no learning rate) */
  MONO_OPT_GROUP_ADAGRAD = 10  /* ref: optimizer/group_adagrad_optimizer.cc:50-89 (one float of state per segment;
                                  the whole segment is one group: max-gradient accumulator, L2 group shrinkage) */
} mono_opt_type;

typedef enum mono_init_type {
  MONO_INIT_ZEROS = 0,
  MONO_INIT_ONES = 1,
  MONO_INIT_CONSTANT = 2, /* init_a = constant            */
  MONO_INIT_UNIFORM = 3   /* uniform in [init_a, init_b)  */
} mono_init_type;

/* One EntryConfig.Segment: `dim` embedding floats with their own initializer + optimizer.
 * Entry layout follows the reference: all segment embeddings first, then all segment optimizer
 * states (ref: RT/hash_table/entry_accessor.cc:113-223, optimizer/optimizer_combination.cc:58-72).
 * opt_p meaning by optimizer:
 *   SGD      : (none)
 *   ADAGRAD  : [0] initial_accumulator_value, [1] weight_decay_factor
 *   FTRL     : [0] initial_accumulator_value, [1] beta, [2] l1, [3] l2
 *   ADAM     : [0] beta1, [1] beta2, [2] epsilon, [3] weight_decay_factor, [4] use_nesterov(0/1)
 *   MOMENTUM : [0] momentum, [1] weight_decay_factor, [2] use_nesterov(0/1)            state: n[dim]
 *   RMSPROP  : [0] momentum, [1] weight_decay_factor, [2] learning_rate of the CONFIG  state: n[dim]
 *   RMSPROPV2: [0] momentum, [1] weight_decay_factor                                   state: n[dim]
 *   ADADELTA : [0] averaging_ratio, [1] epsilon, [2] weight_decay_factor               state: accum[dim], accum_update[dim]
 *   AMSGRAD  : as ADAM                                                                 state: m, v, vhat [dim each], beta powers
 *   MOVING_AVERAGE: [0] momentum                                                       state: none
 *   GROUP_ADAGRAD : [0] initial_accumulator_value, [1] weight_decay_factor, [2] beta,
 *                   [3] l2_regularization_strength                                     state: grad_square_sum (1 float)
 */
typedef struct mono_segment_cfg {
  int32_t dim;
  int32_t init_type; /* mono_init_type */
  float init_a;
  float init_b;
  int32_t opt_type; /* mono_opt_type */
  float opt_p[6];
} mono_segment_cfg;

typedef struct mono_table_cfg {
  const char* name;
  int32_t n_segments;
  const mono_segment_cfg* segments;
  uint64_t initial_capacity;      /* rows to pre-size for (ref proto field 2)                */
  uint32_t default_expire_days;   /* SlotExpireTimeConfig.default_expire_time (36500)        */
  int32_t n_slot_expire;          /* per-slot overrides                                      */
  const uint32_t* slot_ids;       /* [n_slot_expire]                                         */
  const uint32_t* slot_expire_days; /* [n_slot_expire]                                       */
  uint64_t init_seed;             /* counter-based uniform init keyed by (seed, fid, column) */
} mono_table_cfg;

typedef struct mono_mtable mono_mtable_t; /* opaque; ref: RT/ops/multi_hash_table.h:29-71 */

const char* mono_last_error(void);
int32_t mono_abi_version(void);

/* ref: CreateMultiHashTableOp::CreateResource, RT/ops/multi_hash_table_op.cc:86-103.
 * `device` is the CUDA ordinal that owns the table. */
int mono_mtable_create(const mono_table_cfg* cfgs, int32_t n_tables, int32_t device,
                       mono_mtable_t** out);
int mono_mtable_destroy(mono_mtable_t* t);

int32_t mono_mtable_num_tables(const mono_mtable_t* t);
/* index of `name` in sorted order, or -1 */
int32_t mono_mtable_table_index(const mono_mtable_t* t, const char* name);
const char* mono_mtable_table_name(const mono_mtable_t* t, int32_t k);
/* ref: EmbeddingHashTableInterface::{DimSize,SliceSize,Size} (embedding_hash_table_interface.h:79-133) */
int32_t mono_mtable_dim(const mono_mtable_t* t, int32_t k);
int32_t mono_mtable_slice_size(const mono_mtable_t* t, int32_t k);
int mono_mtable_size(mono_mtable_t* t, int32_t k, int64_t* out_size, void* stream); /* SYNC */
/* ref: EmbeddingHashTableTfBridge::max_update_ts_sec_ (tf_bridge.cc:202-206,262-263) */
int64_t mono_mtable_max_update_ts(const mono_mtable_t* t, int32_t k);

/* ---- lookup ------------------------------------------------------------------------------ */

/* ref: MonolithMultiHashTableLookup, RT/ops/multi_hash_table_lookup_op.cc:37-88,200-209
 * (req_size==1 behaviour).  ids_dev[id_split[k]:id_split[k+1]] are looked up in table k; rows are
 * written contiguously: emb = concat_k (n_k x D_k).  Miss -> zeros, never inserts
 * (ref: cuckoo_embedding_hash_table.cc:161-171). */
int mono_mtable_lookup(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                       float* emb_out_dev, void* stream);

/* ref: MonolithMultiHashTableFusedLookup, multi_hash_table_lookup_op.cc:143-197,229-255 and
 * ComputeFusedOffsets, RT/hash_table/utils.h:28-61.  ids are laid out shard-major / table-minor
 * with fused_slot_size[n*K+k] ids in segment (shard n, table k).
 * mono_fused_offsets fills the three small int32 outputs on the host (no device work) so that the
 * caller can size `emb_out_dev` (= emb_offsets[N*K]) before calling mono_mtable_fused_lookup. */
int mono_mtable_fused_offsets(const mono_mtable_t* t, const int32_t* fused_slot_size_host,
                              int32_t num_shards, int32_t* emb_splits_host /*[N]*/,
                              int32_t* id_offsets_host /*[N*K+1]*/,
                              int32_t* emb_offsets_host /*[N*K+1]*/);
int mono_mtable_fused_lookup(mono_mtable_t* t, const int64_t* ids_dev,
                             const int32_t* fused_slot_size_host, int32_t num_shards,
                             int64_t req_time, float* emb_out_dev, void* stream);

/* Membership test (ref: EmbeddingHashTableInterface::Contains).  out_dev[i] in {0,1}. */
int mono_mtable_contains(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                         uint8_t* out_dev, void* stream);

/* ---- fused lookup + pool (the headline kernel) --------------------------------------------
 * Probe + row gather + per-pooled-row SUM / MEAN pool in ONE kernel, straight from raw FID
 * occurrences (no dedup pass is needed on the forward).  Replaces, for one table,
 *   MultiHashTable.lookup -> embedding_combiners.ReduceSum/ReduceMean
 *   (ref: multi_hash_table_ops.py:382-390, embedding_combiners.py:41-70, RT/ops/reduce_op.cc:29-87)
 * and, in the fused-layout path, lookup -> GatherEmb (ref: RT/ops/fused_embedding_to_layout.h:204-261).
 * fids_dev[row_offsets[r]:row_offsets[r+1]] are the FIDs pooled into output row r
 * (row_offsets_dev == NULL means exactly one FID per pooled row).  Terms are accumulated in FID
 * order (deterministic, no atomics).  MEAN divides each term by n (fused-layout semantics,
 * ref: fused_embedding_to_layout.cc:36-38,47-49).  out_dev is [n_rows, out_stride] floats and row r
 * is written at out_dev + r*out_stride (+ out_col) for dim(k) floats.
 */
typedef enum mono_pooling { MONO_POOL_SUM = 0, MONO_POOL_MEAN = 1, MONO_POOL_FIRSTN = 2 } mono_pooling;

int mono_mtable_lookup_pool(mono_mtable_t* t, int32_t k, const int64_t* fids_dev,
                            const int32_t* row_offsets_dev /*[n_rows+1] or NULL*/, int64_t n_rows,
                            int32_t pooling, float* out_dev, int64_t out_stride, int32_t out_col,
                            void* stream);

/* ---- fused backward of lookup_pool ----------------------------------------------------------
 * Scatter of the pooled-row gradients to the unique FIDs + sparse optimizer step + expiry bump for
 * table k, in one call and without materialising the per-unique-FID gradient buffer.  Replaces
 *   ScatterGrad / BackwardBatchKernel (ref: RT/ops/fused_embedding_to_layout.h:286-347,
 *   fused_embedding_to_layout.cu.cc:337-381: float atomicAdd per occurrence) followed by
 *   MonolithMultiHashTableOptimize (ref: RT/ops/multi_hash_table_update_op.cc:47-100)
 * for the occurrences fids_dev[row_offsets[r]:row_offsets[r+1]] of pooled row r (row_offsets NULL:
 * one FID per row).  Every distinct FID receives ONE optimizer step with the sum (SUM) or the sum
 * of g/n (MEAN) of its occurrences' pooled-row gradients, summed without float atomics (run-to-run
 * bit-stable) in the order described at mono_scatter_grad_rows; absent FIDs are inserted (upsert)
 * exactly like optimize.
 * Needs dim(k) % 4 == 0, dim(k) <= 128 and 16-byte aligned gradient rows.  No host sync. */
int mono_mtable_pool_backward(mono_mtable_t* t, int32_t k, const int64_t* fids_dev, int64_t n_fids,
                              const int32_t* row_offsets_dev, int64_t n_rows, int32_t pooling,
                              const float* pooled_grad_dev, int64_t grad_stride, int32_t grad_col,
                              const float* learning_rate_host /*[slice_size(k)]*/,
                              int64_t update_time, int64_t global_step, void* stream);

/* ---- fused forward and backward over many features and tables in one call ------------------
 * A part is one feature's slice of a step: FIDs of table `table`, pooled by `pooling` into rows
 * (row_offsets_dev as for mono_mtable_lookup_pool, NULL = one FID per row and then n_rows == n_fids);
 * row r is rows_dev + r*stride + col: the forward's output row, the backward's row gradient.
 *
 * FIRSTN parts (pooling == MONO_POOL_FIRSTN; max_seq_len = L >= 1, read for FIRSTN parts only): a
 * sequence feature, as the reference's FirstN combiner and the fused layout's FIRSTN branch (ref:
 * embedding_combiners.py:72-102, RT/ops/fused_embedding_to_layout.h:251-256,334-340).  Row r owns the
 * L*dim floats at rows_dev + r*stride + col, position j at + j*dim (a [B, L, dim] tensor is
 * stride = L*dim, col = 0).  Let n_r be row r's FID count (1 without row offsets).
 *   forward: position j < min(n_r, L) is the row of FID fids[offs[r] + j] (zeros for an absent FID);
 *     positions n_r <= j < L are +0.0; occurrences at j >= L are not read.
 *   backward: exactly the result of a one-FID-per-row SUM part over the same FIDs whose gradient row
 *     for occurrence (r, j) is position j of row r for j < L and a row of +0.0 for j >= L.  So a FID
 *     whose occurrences all lie beyond L is still upserted, bumped and counted by the admission
 *     filter, and gets one optimizer step with a zero gradient (the reference's ScatterGrad leaves its
 *     gradient row at the zero fill, and the FID stays in the ids the optimizer receives).
 * A FIRSTN part needs n_rows * max_seq_len <= 2^31.
 *
 * mono_mtable_lookup_pool_parts: every SUM / MEAN part's output is bit-identical to
 * mono_mtable_lookup_pool on that part alone (any dim up to 512, CSR or one-FID rows, SUM or MEAN, any
 * stride and column; parts may write disjoint columns of one tensor); FIRSTN parts serve any dim up to
 * 512 too.  Kernel launches: one per distinct kernel instantiation among the parts (for SUM / MEAN the
 * kernel mono_mtable_lookup_pool would pick; for FIRSTN one of lookup_seq_kernel's, by the table's
 * lane group and whether misses must be confirmed), not one per part.
 * MONO_ERR_INVALID_ARGUMENT, before any device work: n_parts outside [0, MONO_MAX_POOL_PARTS], a bad
 * table index, dim > 512, pooling other than SUM, MEAN or FIRSTN, a FIRSTN part with max_seq_len < 1
 * or n_rows * max_seq_len > 2^31, n_rows != n_fids without offsets.
 *
 * mono_mtable_pool_backward_parts: for every table named by some part, the occurrences
 * of all its parts are ONE batch, taken in part order and then occurrence order, as the reference's
 * per-table ScatterGrad sees them: each distinct FID of the table gets one upsert, one timestamp bump,
 * one admission-filter count and one optimizer step with the sum of its terms (a term is the part's
 * row gradient, divided by the row's n for a CSR MEAN part; for a FIRSTN part as stated above).  The
 * sum is associated as for
 * mono_mtable_pool_backward, with the tree depth set by the table's occurrence count in the call, so
 * parts of one table with one pooling give exactly the bits of one mono_mtable_pool_backward over
 * their concatenated FIDs, stacked gradient rows and rebased row offsets.  Tables do not interact.
 * learning_rate_host has sum_k slice_size(k) floats for ALL tables, table order (as optimize).
 * Kernel launches: 1 occurrence map + 1 claim + 1 miss + 1 finalize + 3 per radix pass + 3 run list,
 * then per distinct table k of the call 3 + L(k) (reduce, L(k) tree levels, finish, apply), where
 * passes = ceil(bits / 11) for bits = ceil(log2(sum_k claim slots(k))), claim slots(k) = the smallest
 * power of two >= max(1024, 2 M(k)), L(k) = 0 for M(k) <= 16384 occurrences, 1 up to 2^21, else 2.
 * MONO_ERR_INVALID_ARGUMENT, before any device work (no table changes): n_parts outside
 * [0, MONO_MAX_POOL_PARTS], a bad table index, a part whose table breaks the pool_backward conditions
 * (dim % 4 == 0, dim <= 128, 16-byte aligned gradient rows; FIRSTN parts included), pooling other
 * than SUM, MEAN or FIRSTN, a FIRSTN part with max_seq_len < 1 or n_rows * max_seq_len > 2^31,
 * n_rows != n_fids without offsets, or more than 2^30 occurrences in total.  FIRSTN parts add no
 * launch: the occurrence map writes their gradient-row addresses.  No host sync. */
#define MONO_MAX_POOL_PARTS 1024

typedef struct mono_pool_part {
  int32_t table;                    /* k, sorted-name index                                   */
  const int64_t* fids_dev;
  int64_t n_fids;
  const int32_t* row_offsets_dev;   /* [n_rows+1] or NULL = one FID per row                   */
  int64_t n_rows;
  int32_t pooling;                  /* MONO_POOL_SUM | MONO_POOL_MEAN | MONO_POOL_FIRSTN       */
  float* rows_dev;                  /* forward: output rows; backward: pooled-row gradients   */
  int64_t stride;                   /* floats between rows                                    */
  int32_t col;                      /* first column of the table's dim(k) floats in a row     */
  int32_t max_seq_len;              /* FIRSTN only: positions per row (in the trailing padding
                                       of the earlier layout: the struct stays 72 bytes)      */
} mono_pool_part;

int mono_mtable_lookup_pool_parts(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                  void* stream);
int mono_mtable_pool_backward_parts(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                    const float* learning_rate_host /*[sum_k slice_size(k)]*/,
                                    int64_t update_time, int64_t global_step, void* stream);

/* ---- the parts calls with bfloat16 rows ------------------------------------------------------
 * The arguments of mono_mtable_lookup_pool_parts / mono_mtable_pool_backward_parts, but every part's
 * rows_dev points at bfloat16 storage (a cast pointer; the struct is unchanged), and stride and col
 * count bf16 elements (a FIRSTN part's position j sits at + j*dim bf16 elements).  Tables, optimizer
 * state and all arithmetic stay fp32: only the rows handed in or back are bf16.
 *
 * mono_mtable_lookup_pool_parts_bf16: each output element is the fp32 value
 * mono_mtable_lookup_pool_parts writes for the same part (accumulated in fp32 in the same order),
 * rounded once to bf16 to nearest even (__float2bfloat16_rn); absent FIDs and empty FIRSTN
 * positions are +0.0, NaN stays NaN (payload unspecified).  Any dim up to 512, any stride and
 * column, parts writing disjoint columns of one tensor, and the same errors: as the fp32 call.
 * Kernel launches: one per distinct bf16 kernel instantiation among the parts.  A one-FID part
 * never takes the TMA-staged lookup (it moves rows without touching registers, and the conversion
 * needs them): it runs the register-path lookup kernel at every dim.  The lookup_dual option does
 * not apply.
 *
 * mono_mtable_pool_backward_parts_bf16: bit for bit the result of mono_mtable_pool_backward_parts
 * on the same parts with every gradient row widened exactly to fp32 (table entries, optimizer
 * state, timestamps, admission-filter counts, the sum's association and tree depth); the MEAN
 * division and every add happen in fp32 after the widening.  Same launches as the fp32 call.
 * MONO_ERR_INVALID_ARGUMENT, before any device work (no table changes): the fp32 call's conditions,
 * with the row condition dim % 4 == 0, dim <= 128, stride % 4 == 0, col % 4 == 0 and 8-byte
 * aligned rows. */
int mono_mtable_lookup_pool_parts_bf16(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                       void* stream);
int mono_mtable_pool_backward_parts_bf16(mono_mtable_t* t, const mono_pool_part* parts_host, int32_t n_parts,
                                         const float* learning_rate_host /*[sum_k slice_size(k)]*/,
                                         int64_t update_time, int64_t global_step, void* stream);

/* ---- updates ----------------------------------------------------------------------------- */

#define MONO_FLAG_IDS_UNIQUE 1u      /* caller guarantees ids unique per table within this call   */
#define MONO_FLAG_DEDUP_SUM 2u       /* ref: enable_dedup / enable_grad_accumulation (sum grads)  */

/* ref: MonolithMultiHashTableOptimize, RT/ops/multi_hash_table_update_op.cc:47-100 ->
 * EmbeddingHashTableTfBridge::BatchOptimize (tf_bridge.cc:258-341) ->
 * CuckooEmbeddingHashTable::Optimize (cuckoo_embedding_hash_table.cc:239-247): upsert (insert +
 * Init when absent), SetTimestamp(update_time), optimizer step.  learning_rate_host has
 * sum_k slice_size(k) floats, consumed table by table.  Without MONO_FLAG_IDS_UNIQUE duplicate ids
 * are applied sequentially in input order, exactly like the reference's per-id loop (this costs a
 * device sync per round of duplicates). */
int mono_mtable_optimize(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                         const float* grads_dev, const float* learning_rate_host,
                         int64_t update_time, int64_t global_step, uint32_t flags, void* stream);

/* ref: MonolithMultiHashTableFusedOptimize, multi_hash_table_update_op.cc:268-325.
 * Segments as in fused_lookup; id_offsets / grad_offsets are the arrays returned by
 * mono_mtable_fused_offsets.  The same FID may appear once per shard; shards are applied in shard
 * order (the reference's single-thread order). */
int mono_mtable_fused_optimize(mono_mtable_t* t, const int64_t* ids_dev,
                               const int32_t* fused_slot_size_host, const float* grads_dev,
                               const int32_t* id_offsets_host, const int32_t* grad_offsets_host,
                               const float* learning_rate_host, int64_t req_time,
                               int64_t global_step, int32_t num_shards, uint32_t flags,
                               void* stream);

/* ref: MonolithMultiHashTableAssign / AssignAdd, multi_hash_table_update_op.cc:106-190;
 * cuckoo_embedding_hash_table.cc:185-212 (upsert, SetTimestamp, overwrite / +=). */
int mono_mtable_assign(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                       const float* values_dev, int64_t update_time, uint32_t flags, void* stream);
int mono_mtable_assign_add(mono_mtable_t* t, const int64_t* ids_dev, const int64_t* id_split_host,
                           const float* values_dev, int64_t update_time, uint32_t flags,
                           void* stream);

/* ref: MonolithMultiHashTableReinitialize, multi_hash_table_update_op.cc:192-241;
 * cuckoo_embedding_hash_table.cc:214-226.  status_dev[i]: 0 inserted, 1 existed & re-initialised.
 * Unknown table name => k < 0 => every status is -1 and nothing is touched. */
int mono_mtable_reinitialize(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                             int32_t* status_dev, int64_t update_time, void* stream);

/* ref: CuckooEmbeddingHashTable::Evict, cuckoo_embedding_hash_table.cc:251-264: drop rows with
 * max_update_time - row.ts >= expire_days(slot_id_v2(fid)) * 86400.  The reference drives this
 * from a background thread (tf_bridge.cc:73-104); here the caller drives it. */
int mono_mtable_evict(mono_mtable_t* t, int32_t k, int64_t max_update_time, void* stream);

/* Counting admission filter of table k (ref: monolith::hash_filter::HashFilter<uint16_t>, RT/hash_filter/
 * hash_filter.h:34-165; created by hash_filter_ops.create_hash_filters; thresholds from
 * SlotOccurrenceThresholdConfig, embedding_hash_table.proto:100-110).  A FID that is ABSENT from the table is only
 * inserted by optimize / assign / the fused backward once the filter has counted `threshold(slot)` earlier
 * occurrences of it (ref call sites: RT/ops/embedding_hash_table_tf_bridge.cc:181-185,208-240,296-326);
 * assign_add consults the filter for every id, present or not (AssignAdd2, :224-232).  threshold 0 never filters.
 * Tables without a filter behave like the reference's DummyHashFilter.  SYNC (allocates). */
int mono_mtable_set_hash_filter(mono_mtable_t* t, int32_t k, int64_t capacity, uint32_t default_threshold,
                                const uint32_t* slot_ids_host, const uint32_t* slot_thresholds_host,
                                int32_t n_slots, void* stream);

/* Full row access for checkpoint/restore and parity tests (ref: EntryDump,
 * embedding_hash_table.proto:45-50; LookupEntry, cuckoo_embedding_hash_table.cc:173-183).
 * entry_out_dev is [n, dim + state_floats + 2]: emb, optimizer state (reference order), then
 * found flag (0/1) and last_update_ts as floats' bit patterns (uint32). */
int32_t mono_mtable_state_floats(const mono_mtable_t* t, int32_t k);
int mono_mtable_lookup_entry(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                             float* entry_out_dev, void* stream);
/* Export up to `max_n` live (fid, row) pairs of table k starting at bucket cursor *cursor
 * (0 to start; set to -1 when exhausted).  SYNC.  ids_out_dev [max_n], entry_out_dev as above. */
int mono_mtable_export(mono_mtable_t* t, int32_t k, int64_t* cursor, int64_t max_n,
                       int64_t* ids_out_dev, float* entry_out_dev, int64_t* n_out, void* stream);
/* Upsert full rows (emb + optimizer state + ts), ref: Restore, cuckoo_embedding_hash_table.cc:299-320 */
int mono_mtable_restore_rows(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, int64_t n,
                             const float* entry_in_dev, void* stream);
/* Restore side of max_update_ts: the reference's Restore returns the largest last_update_ts_sec it read and
 * the table keeps it (cuckoo_embedding_hash_table.cc:299-321; embedding_hash_table_tf_bridge.cc Restore);
 * the caller reports it here after mono_mtable_restore_rows (max with the current value). */
int mono_mtable_note_update_ts(mono_mtable_t* t, int32_t k, int64_t ts);

/* ---- dedup + shard (requester side) ------------------------------------------------------- */

/* ref: FusedReorderByIndices, RT/ops/fused_reorder_by_indices.cc:38-136.
 * inputs: K id lists concatenated in ids_dev, list m = ids_dev[id_split[m]:id_split[m+1]].
 * Dedup is per list (first occurrence wins); shard = fid % (N - rank0_empty) + rank0_empty.
 * Outputs (bit-exact with the reference for non-negative FIDs):
 *   output_dev        int64[<= M]  unique FIDs, shard-major / list-minor, first-occurrence order
 *   shard_sizes       int32[N]
 *   sharded_slot_sizes int32[N*K]
 *   fused_emb_offset_dev int32[M]  float offset of each occurrence's row in the post-all-to-all
 *                                  buffer (rows laid out in `output` order, list m has dims[m] floats)
 * The two small arrays are produced on the device (sizes_dev, int32[N + N*K]) and also copied to
 * the host pointers when those are non-NULL (SYNC in that case).  n_unique likewise.
 * Limits, checked on the host before the device is selected (MONO_ERR_INVALID_ARGUMENT, nothing launched):
 *   1 <= K <= 2^25 lists, 1 <= N <= 64 shards (N >= 2 with rank0_empty), id_split[0] == 0 and non-decreasing,
 *   M = id_split[K] <= 2^30 ids (the scratch set for more would not fit in 80 GB), every dims[m] > 0
 *   (dims[0] only for K == 1).
 * The float offsets are int32, as in the reference: sum over (shard, list) of sizes x dims must be <= 2^31 - 1.
 * The call checks the exact sum after its synchronisation (K > 1 or any host output requested) and then
 * returns MONO_ERR_INVALID_ARGUMENT; the device outputs are undefined and the host outputs are not written.
 * K == 1 without host outputs does not synchronise and is rejected up front when M * dims[0] > 2^31 - 1.
 */
int mono_reorder_by_indices(int32_t device, const int64_t* ids_dev, const int64_t* id_split_host,
                            int32_t num_lists, int32_t num_shards, const int32_t* dims_host,
                            int32_t rank0_empty, int64_t* output_dev, int32_t* sizes_dev,
                            int32_t* fused_emb_offset_dev, int32_t* shard_sizes_host,
                            int32_t* sharded_slot_sizes_host, int64_t* n_unique_host,
                            void* stream);

/* Single-list dedup used by the fused single-GPU train step: unique FIDs in first-occurrence
 * order + the inverse map (occurrence -> unique ordinal).  n_unique_dev is an int32 on device;
 * n_unique_host (optional) forces a SYNC.  n <= 2^30 (MONO_ERR_INVALID_ARGUMENT otherwise, nothing launched). */
int mono_dedup(int32_t device, const int64_t* ids_dev, int64_t n, int64_t* unique_out_dev,
               int32_t* inverse_out_dev, int32_t* n_unique_dev, int64_t* n_unique_host,
               void* stream);

/* ---- owner grouping: one grouping per batch shared by the sharded forward and backward -------
 * Replaces FusedReorderByIndices (ref: RT/ops/fused_reorder_by_indices.cc:38-123) + the float-atomic
 * FusedGatherGrad scatter (ref: RT/ops/map_id_to_embedding.cu.cc:75-118) for ONE id list on the
 * sharded fast path.  build(): the M occurrences are grouped by FID (scratch set + stable radix sort)
 * and the distinct FIDs are bucketed by owner = (uint64)fid % num_shards.  Outputs on the device:
 *   uniq_out_dev[<= M]     distinct FIDs, shard-major (order inside a shard is the engine's; use
 *                          mono_reorder_by_indices when the reference's first-occurrence order is needed)
 *   occ_offset_out_dev[M]  float offset (index in uniq_out * dim) of every occurrence's row in the
 *                          post-all-to-all row buffer  (== fused_emb_offset of the reference op)
 * and on the host (SYNC): shard_counts_host[num_shards], n_unique_host.
 * reduce(): with the grouping built last, out_rows_dev[u*dim : +dim] = sum (SUM) / sum of g/n (MEAN)
 * of the pooled-row gradients of FID u's occurrences, without float atomics, in the order described
 * at mono_scatter_grad_rows. */
typedef struct mono_grouping mono_grouping_t;
int mono_grouping_create(int32_t device, mono_grouping_t** out);
int mono_grouping_destroy(mono_grouping_t* g);
int mono_grouping_build(mono_grouping_t* g, const int64_t* fids_dev, int64_t n_fids, int32_t num_shards,
                        int32_t dim, int64_t* uniq_out_dev, int32_t* occ_offset_out_dev,
                        int32_t* shard_counts_host, int64_t* n_unique_host, void* stream);
int mono_grouping_reduce(mono_grouping_t* g, const float* pooled_grad_dev, int64_t grad_stride,
                         int32_t grad_col, const int32_t* row_offsets_dev, int64_t n_rows,
                         int32_t pooling, float* out_rows_dev, void* stream);

/* ---- pooling from a looked-up buffer (sync all-to-all path) ------------------------------- */

/* ref: FusedGatherKernel, RT/ops/map_id_to_embedding.cu.cc:30-74 (forward) and
 * FusedGatherGradKernel :75-118 (backward) fused with the per-row SUM/MEAN pool:
 * out[r, out_col:out_col+dim] = pool_{m in row r} fused_emb[offsets[m] : +dim].
 * row_offsets_dev == NULL => one occurrence per row (pure gather, == FusedGatherKernel). */
int mono_gather_pool(int32_t device, const float* fused_emb_dev, const int32_t* emb_offset_dev,
                     const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim, int32_t pooling,
                     float* out_dev, int64_t out_stride, int32_t out_col, void* stream);
/* Backward: grad_fused[offsets[m] : +dim] += pooled_grad[r] (SUM) or /n (MEAN).
 * grad_fused_dev must be zero-filled by the caller (ref zero-fills at cu.cc:397-400). */
int mono_gather_pool_grad(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                          int32_t grad_col, const int32_t* emb_offset_dev,
                          const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                          int32_t pooling, float* grad_fused_dev, void* stream);

/* Deterministic variant of mono_gather_pool_grad (no float atomics): occurrences are radix-sorted
 * by destination offset and each destination row is written once with the sum of its occurrences'
 * pooled-row gradients (run-to-run bit-stable; the reference GPU kernel uses atomicAdd,
 * map_id_to_embedding.cu.cc:75-118).  Summation order: a row with at most 64 occurrences is summed
 * sequentially in occurrence order (the CPU reference's order); a longer run is summed in 32-occurrence
 * blocks aligned to its first occurrence, and the blocks are combined by a fixed tree whose shape
 * depends on the run length, the row width (dim picks the lane group) and the call's occurrence count
 * (which picks the tree depth: none up to 16 384 occurrences, one level up to 2^21, two above).  emb_offset_dev[m] is the float offset of
 * occurrence m's row inside grad_fused_dev (multiples of dim; total_floats = buffer length).
 * Destination rows that no occurrence refers to are left untouched.  dim % 4 == 0, dim <= 128. */
int mono_scatter_grad_rows(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                           int32_t grad_col, const int32_t* emb_offset_dev, int64_t n_occurrences,
                           const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                           int32_t pooling, float* grad_fused_dev, int64_t total_floats,
                           void* stream);

/* ---- the gather calls with bfloat16 pooled rows ----------------------------------------------
 * The arguments of their fp32 twins above, but the tower-side rows are bfloat16: out_dev /
 * pooled_grad_dev point at bf16 storage (cast pointers) and out_stride / out_col, grad_stride /
 * grad_col count bf16 elements.  fused_emb_dev and grad_fused_dev stay fp32, as does all arithmetic.
 *
 * mono_gather_pool_bf16: each output element is the fp32 value mono_gather_pool writes (accumulated in
 * fp32 in the same order), rounded once to nearest even (__float2bfloat16_rn); NaN stays NaN (payload
 * unspecified).  One kernel launch: the row copy when row_offsets_dev is NULL, dim % 4 == 0,
 * dim <= 4 * lane-group width, out_stride % 4 == 0, out_col % 4 == 0, fused_emb_dev 16-byte and out_dev
 * 8-byte aligned; the pooling kernel otherwise.
 *
 * mono_gather_pool_grad_bf16 / mono_scatter_grad_rows_bf16: bit for bit the fp32 twin's result on the
 * pooled gradients widened exactly to fp32 (the MEAN division and every add happen in fp32 after the
 * widening).  gather_pool_grad: one kernel launch.  scatter_grad_rows: the fp32 twin's launches
 * (3 per radix pass and 3 for the run list, 1 occurrence -> row map when row_offsets_dev is given, the
 * reduce, one per tree level and the finish, then the emit); MONO_ERR_INVALID_ARGUMENT before any
 * device work unless dim % 4 == 0, dim <= 128, grad_stride % 4 == 0, grad_col % 4 == 0, pooled_grad_dev
 * 8-byte and grad_fused_dev 16-byte aligned. */
int mono_gather_pool_bf16(int32_t device, const float* fused_emb_dev, const int32_t* emb_offset_dev,
                          const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim, int32_t pooling,
                          float* out_dev, int64_t out_stride, int32_t out_col, void* stream);
int mono_gather_pool_grad_bf16(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                               int32_t grad_col, const int32_t* emb_offset_dev,
                               const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                               int32_t pooling, float* grad_fused_dev, void* stream);
int mono_scatter_grad_rows_bf16(int32_t device, const float* pooled_grad_dev, int64_t grad_stride,
                                int32_t grad_col, const int32_t* emb_offset_dev, int64_t n_occurrences,
                                const int32_t* row_offsets_dev, int64_t n_rows, int32_t dim,
                                int32_t pooling, float* grad_fused_dev, int64_t total_floats,
                                void* stream);

/* ---- generic fused layout op -------------------------------------------------------------- */

/* ref: MonolithEmbeddingToLayoutV3/V4/V5 and its grad, RT/ops/fused_embedding_to_layout.{h,cc,cu.cc}.
 * The proto FeatureConfigs/OutConfig/SliceConfig (idl/matrix/proto/example.proto:177-220) is
 * flattened by the host wrapper into slice tasks: */
typedef struct mono_slice_task {
  int32_t nfl_idx;     /* feature index into nfl_offset (sorted feature names)             */
  int32_t slice_start; /* first float of the slice inside the feature's row               */
  int32_t dim;         /* slice_end - slice_start                                          */
  int32_t pooling;     /* mono_pooling                                                      */
  int32_t max_seq_len; /* FIRSTN only                                                       */
  int32_t out_tensor;  /* which output tensor                                               */
  int32_t out_row_stride; /* floats between consecutive samples of that tensor             */
  int32_t out_col;     /* float offset of this slice inside a sample's row                 */
  int32_t accumulate;  /* 1 for ADDN outputs: add into the row instead of overwriting      */
} mono_slice_task;

/* emb_ptrs_dev: device array of `n_emb` device pointers (one per (table, shard) list, index1 of
 * fid_offset); emb_strides_dev[n_emb] = PtrWrapper.offset of each list (1 in v3/v4/v5).
 * nfl_offset_dev holds the reference's uint32 words (bit 31 = shared feature), one per entry;
 * fid_offset_dev the reference's uint64 words.
 * out_ptrs_dev: device array of output tensor pointers.  The output sizes are not passed: the
 * forward writes exactly the elements its tasks cover (for every sample b < batch_size, floats
 * out_col .. out_col + dim of row b, out_col + max_seq_len * dim for FIRSTN, zeros where a sample
 * has no FIDs or a FIRSTN row is shorter than max_seq_len) and leaves every other element as it
 * was.  The grad call accumulates into emb_grad_ptrs_dev with float atomics: those buffers must
 * arrive zero-filled, and elements no FID refers to are left as they are.
 * Both calls return MONO_ERR_INVALID_ARGUMENT, before any device work, for a task with nfl_idx
 * outside [0, total_nfl), dim <= 0, a negative slice_start, out_col or out_tensor, an unknown
 * pooling, FIRSTN with max_seq_len <= 0 or accumulate set, out_row_stride < out_col + dim
 * (out_col + max_seq_len * dim for FIRSTN); and, once the device is selected, for ADDN members of
 * one output slice with unequal dims. */
int mono_embedding_to_layout(int32_t device, const float* const* emb_ptrs_dev,
                             const int32_t* emb_strides_dev, int32_t n_emb,
                             const uint64_t* fid_offset_dev, int64_t total_fid,
                             const int32_t* feature_offset_dev, int32_t total_feature,
                             const uint32_t* nfl_offset_dev, int32_t total_nfl, int32_t batch_size,
                             const mono_slice_task* tasks_host, int32_t n_tasks,
                             float* const* out_ptrs_dev, void* stream);
int mono_embedding_to_layout_grad(int32_t device, float* const* emb_grad_ptrs_dev,
                                  const int32_t* emb_strides_dev, int32_t n_emb,
                                  const uint64_t* fid_offset_dev, int64_t total_fid,
                                  const int32_t* feature_offset_dev, int32_t total_feature,
                                  const uint32_t* nfl_offset_dev, int32_t total_nfl,
                                  int32_t batch_size, const mono_slice_task* tasks_host,
                                  int32_t n_tasks, const float* const* out_grad_ptrs_dev,
                                  void* stream);

/* The layout calls with bfloat16 tower-side tensors: the arguments of mono_embedding_to_layout /
 * _grad, but out_ptrs_dev / out_grad_ptrs_dev point at bf16 tensors and every task's out_row_stride
 * and out_col count bf16 elements.  The embedding inputs and the embedding gradients stay fp32.
 * Forward: every covered element is the fp32 call's value (accumulated in fp32 in the same order)
 * rounded once to nearest even; NaN stays NaN (payload unspecified); absent rows and empty FIRSTN
 * positions are +0.0; uncovered elements keep their bits.  Grad: bit for bit the fp32 call on the
 * gradients widened exactly to fp32 (MEAN division and atomics in fp32).  The same task validation and
 * error codes as the fp32 calls, in the same order.  One kernel launch per call, as the fp32 calls. */
int mono_embedding_to_layout_bf16(int32_t device, const float* const* emb_ptrs_dev,
                                  const int32_t* emb_strides_dev, int32_t n_emb,
                                  const uint64_t* fid_offset_dev, int64_t total_fid,
                                  const int32_t* feature_offset_dev, int32_t total_feature,
                                  const uint32_t* nfl_offset_dev, int32_t total_nfl, int32_t batch_size,
                                  const mono_slice_task* tasks_host, int32_t n_tasks,
                                  float* const* out_ptrs_dev, void* stream);
int mono_embedding_to_layout_grad_bf16(int32_t device, float* const* emb_grad_ptrs_dev,
                                       const int32_t* emb_strides_dev, int32_t n_emb,
                                       const uint64_t* fid_offset_dev, int64_t total_fid,
                                       const int32_t* feature_offset_dev, int32_t total_feature,
                                       const uint32_t* nfl_offset_dev, int32_t total_nfl,
                                       int32_t batch_size, const mono_slice_task* tasks_host,
                                       int32_t n_tasks, const float* const* out_grad_ptrs_dev,
                                       void* stream);

/* ---- NVLink peer window: the exchange steps of the sharded path as peer stores ---------------
 * ref: the all-to-alls of the reference's synchronous multi-GPU path (distributed_ps_sync.py:92-118
 * forward ids + embeddings, :531-573 backward gradients; SURVEY.md §8e).  One window per rank
 * (device memory, mapped into every peer process of the node through CUDA IPC); the producing kernel
 * stores its result where the consuming rank reads it, and a flag barrier orders the ranks.
 * All offsets are relative to the window's data region; `world` values per array, indexed by rank.
 *   create  : allocates `bytes` of window on `device` (world <= 16).
 *   handle  : writes this rank's 64-byte IPC handle; the caller all-gathers the handles ...
 *   attach  : ... and passes all `world` of them (64 bytes each, rank order).
 *   detach  : unmaps the peers' windows; teardown = detach on every rank, rank barrier, destroy.
 *   local   : device pointer of this rank's data region (what the peers write into).
 *   barrier : stream-ordered; returns immediately.  Every rank must call it the same number of times.
 *   put     : nbytes[r] bytes from src_dev + src_off[r] into rank r's window at region_off + dst_off[r]
 *             (multiples of 8 bytes).
 *   get     : the mirror of put: nbytes[r] bytes of rank r's window at region_off + src_off[r] are read
 *             into dst_dev + dst_off[r] (multiples of 16 bytes).
 *   lookup_push       : fused lookup + row exchange.  ids_dev = counts[0] ids of rank 0, then counts[1]
 *             of rank 1, ...; the row of rank r's i-th id is stored into rank r's window at
 *             region_off + (dst_row_off[r] + i) * dim * 4.  Absent ids give zero rows.  dim % 4 == 0.
 *   reduce_push       : mono_grouping_reduce whose output rows (owner-bucketed: shard_counts[r] rows for
 *             rank r, in mono_grouping_build's order) are stored into rank r's window at
 *             region_off + dst_row_off[r] * dim * 4. */
typedef struct mono_peer mono_peer_t;
int mono_peer_create(int32_t device, int32_t world, int32_t rank, int64_t bytes, mono_peer_t** out);
int mono_peer_destroy(mono_peer_t* p);
int mono_peer_detach(mono_peer_t* p);
int mono_peer_handle(mono_peer_t* p, void* handle_out_64);
int mono_peer_attach(mono_peer_t* p, const void* handles, int32_t n_handles);
int mono_peer_local(mono_peer_t* p, void** data_dev_out);
int mono_peer_barrier(mono_peer_t* p, void* stream);
int mono_peer_put(mono_peer_t* p, int64_t region_off, const int64_t* dst_off, const void* src_dev,
                  const int64_t* src_off, const int64_t* nbytes, void* stream);
int mono_peer_get(mono_peer_t* p, int64_t region_off, const int64_t* src_off, void* dst_dev,
                  const int64_t* dst_off, const int64_t* nbytes, void* stream);
int mono_mtable_lookup_push(mono_mtable_t* t, int32_t k, const int64_t* ids_dev, const int64_t* counts,
                            mono_peer_t* p, int64_t region_off, const int64_t* dst_row_off, void* stream);
int mono_grouping_reduce_push(mono_grouping_t* g, const float* pooled_grad_dev, int64_t grad_stride,
                              int32_t grad_col, const int32_t* row_offsets_dev, int64_t n_rows,
                              int32_t pooling, const int64_t* shard_counts, mono_peer_t* p,
                              int64_t region_off, const int64_t* dst_row_off, void* stream);

/* ---- host-buffer entry points (what a CPU-resident caller such as the reference's TF op shim
 *      would call: ids / grads in host memory, results back in host memory).  These stage through
 *      pinned memory and include the H2D / D2H copies; they return after the result is on the host.
 *      ref: same ops as mono_mtable_lookup / lookup_pool / optimize. ------------------------- */
int mono_mtable_lookup_host(mono_mtable_t* t, const int64_t* ids_host, const int64_t* id_split_host,
                            float* emb_out_host);
int mono_mtable_lookup_pool_host(mono_mtable_t* t, int32_t k, const int64_t* fids_host,
                                 const int32_t* row_offsets_host, int64_t n_rows, int64_t n_fids,
                                 int32_t pooling, float* out_host);
int mono_mtable_optimize_host(mono_mtable_t* t, const int64_t* ids_host,
                              const int64_t* id_split_host, const float* grads_host,
                              const float* learning_rate_host, int64_t update_time,
                              int64_t global_step, uint32_t flags);

/* ---- checkpoint files in the reference's on-disk format (host-only; SURVEY §8(f) row 1) -------
 * ref: MonolithMultiHashTableSave / Restore, RT/ops/multi_hash_table_save_restore_ops.cc:105-388.
 *   <basename>-%05d-of-%05d      TFRecord stream, Snappy block compression: per table, one serialized
 *                                EntryDump (embedding_hash_table.proto:45-50) per live entry
 *   <basename>.meta-%05d-of-%05d TFRecord stream: one MultiHashTableMetadata {table_name, num_entries}
 *                                per table, in the order the tables were written
 * Rows cross this boundary in mono_mtable_export / mono_mtable_restore_rows layout:
 * n x (dim + state_floats + 2) floats = [num | optimizer state | found | last_update_ts (u32 bits)].
 * writer: open -> (begin_table -> add* -> end_table)* -> close(commit = 1 renames the temporary files).
 *   add drops expired entries like the reference's save (max_update_ts - ts >= expire_days(slot) * 86400);
 *   expire_days_by_slot has 32768 entries (slot = (id >> 48) & 0x7fff) or is NULL (keep everything).
 * reader: open -> (next_table -> read*)* -> close; read decodes against the caller's segment list.
 * snappy = 1: the reference's data-file container; 0: plain TFRecord (the metadata file is always plain).
 * encode_entry / decode_entry / crc32c / snappy_* expose the building blocks to the tests. */
typedef struct mono_ckpt_writer mono_ckpt_writer_t;
typedef struct mono_ckpt_reader mono_ckpt_reader_t;
const char* mono_ckpt_last_error(void);
int mono_ckpt_writer_open(const char* data_path, const char* meta_path, int32_t snappy,
                          mono_ckpt_writer_t** out);
int mono_ckpt_writer_begin_table(mono_ckpt_writer_t* w, const char* name, const mono_segment_cfg* segs,
                                 int32_t nsegs);
int mono_ckpt_writer_add(mono_ckpt_writer_t* w, const int64_t* ids_host, const float* rows_host, int64_t n,
                         int64_t max_update_ts, const int64_t* expire_days_by_slot, int64_t* n_written);
int mono_ckpt_writer_end_table(mono_ckpt_writer_t* w);
int mono_ckpt_writer_close(mono_ckpt_writer_t* w, int32_t commit);
int mono_ckpt_reader_open(const char* data_path, const char* meta_path, int32_t snappy,
                          mono_ckpt_reader_t** out);
int mono_ckpt_reader_next_table(mono_ckpt_reader_t* r, char* name_out, int32_t cap, int64_t* num_entries,
                                int32_t* has);
int mono_ckpt_reader_read(mono_ckpt_reader_t* r, const mono_segment_cfg* segs, int32_t nsegs,
                          int64_t* ids_out_host, float* rows_out_host, int64_t max_n, int64_t* n_read);
int mono_ckpt_reader_close(mono_ckpt_reader_t* r);
int64_t mono_ckpt_encode_entry(const mono_segment_cfg* segs, int32_t nsegs, int64_t id, const float* row,
                               void* out, int64_t out_cap);
int mono_ckpt_decode_entry(const mono_segment_cfg* segs, int32_t nsegs, const void* rec, int64_t n,
                           int64_t* id_out, float* row_out);
uint32_t mono_ckpt_crc32c(const void* data, int64_t n);
uint32_t mono_ckpt_masked_crc32c(const void* data, int64_t n);
int64_t mono_ckpt_snappy_compress(const void* in, int64_t n, void* out, int64_t out_cap);
int64_t mono_ckpt_snappy_uncompress(const void* in, int64_t n, void* out, int64_t out_cap);

/* ---- device-driven sharded step (replaces the orchestration of NT/distributed_ps.py:1501-2001 and
 *      NT/distributed_ps_sync.py:95-512 for ONE table on the GPUs of one NVSwitch box) ------------------------------
 * A whole sparse train step sharded by fid mod N with nothing returning to the host: FID buckets, rows and summed
 * gradient rows travel through fixed per-source regions of the ranks' peer windows, arrival is signalled by
 * directional flags (no all-rank barrier, no host count exchange), every loop is sized by device-side counts
 * (csrc/xstep.cu).  Same results as mono_grouping_* + mono_peer_* + mono_mtable_fused_optimize driven from the host.
 *   mono_xstep_window_bytes  bytes the window of every rank must have for capacity `cap_pair` (max FID occurrences
 *                            of one rank's batch) — create the windows with mono_peer_create and attach them first
 *   mono_xstep_forward       group the batch, exchange, pool: out[r] = pool of the rows of fids (CSR row_offsets or
 *                            one FID per row), as mono_mtable_lookup_pool on the global table
 *   mono_xstep_backward      gradient of that forward: per-FID sums to the owners, owners upsert + optimize, the
 *                            requesters applied in rank order (ref: multi_hash_table_update_op.cc:286-300)
 * Every rank must call forward / backward the same number of times; a forward must be followed by its backward. */
typedef struct mono_xstep mono_xstep_t;
int64_t mono_xstep_window_bytes(int32_t world, int64_t cap_pair, int32_t dim);
int mono_xstep_create(mono_mtable_t* t, int32_t k, mono_peer_t* window, int64_t cap_pair, mono_xstep_t** out);
int mono_xstep_destroy(mono_xstep_t* x);
/* Optional: build the grouping of the NEXT batch on `stream2` while the step in flight runs on its own stream (the
 * grouping depends on the batch only; ref pipelining: NT/distributed_ps_sync.py:199-204,270-275).  The next
 * mono_xstep_forward must get the same fids pointer and count, otherwise it regroups inline. */
int mono_xstep_prepare(mono_xstep_t* x, const int64_t* fids_next_dev, int64_t n_fids, void* stream2);
int mono_xstep_forward(mono_xstep_t* x, const int64_t* fids_dev, int64_t n_fids, const int32_t* row_offsets_dev,
                       int64_t n_rows, int32_t pooling, float* out_dev, int64_t out_stride, int32_t out_col,
                       void* stream);
int mono_xstep_backward(mono_xstep_t* x, const float* pooled_grad_dev, int64_t grad_stride, int32_t grad_col,
                        const int32_t* row_offsets_dev, int32_t pooling, const float* lr_host, int64_t update_time,
                        void* stream);

/* Number of kernel launches issued by this library since load (for bench.py's gpu_launches). */
int64_t mono_kernel_launch_count(void);

/* Stand-in dense tower of bench.py's end-to-end step (NOT part of the reference's embedding interface; dense layers
 * are out of scope): pooled[batch][64] fp32 (device) -> relu(x W1) -> . w2 -> mean BCE-with-logits against labels[batch];
 * writes d loss / d pooled into grad_out[batch][64] fp32 and the loss into *loss_out (device scalar).  w1: bf16 [64 in][64
 * out] row-major, w2: bf16 [64].  scratch: device floats, at least mono_bench_tower_scratch_floats().  One fused kernel
 * (bf16 tensor-core MMA, fp32 accumulate) + a 1-block loss reduction, asynchronous on `stream`. */
int64_t mono_bench_tower_scratch_floats(void);
int mono_bench_tower_grad(const float* pooled, int64_t batch, const float* labels, const void* w1_bf16,
                          const void* w2_bf16, float* grad_out, float* loss_out, float* scratch,
                          int64_t scratch_floats, void* stream);

/* Engine tuning knobs (process-wide; no reference counterpart).  Known names:
 *   "lookup_tma"  1 (default) / 0: single-table lookups with packed 128- or 256-byte output rows use the TMA-staged kernel (bulk row copies
 *                 global -> shared -> global) instead of the register-path kernel.  Results are identical.
 *   "claim_pf" "apply_pf" "lookup_pf" (L2 prefetch of the next item's lines), "seg_vpl" (1 | 2), "seg_ahead",
 *   "claim_dual" "lookup_dual" (both candidate buckets requested together): A/B switches between two implementations
 *   of the same result; defaults are the measured winners (`bench.py --ab` times the alternatives).
 * Returns MONO_ERR_INVALID_ARGUMENT for an unknown name.  mono_get_option returns the current value (or -1). */
int mono_set_option(const char* name, int64_t value);
int64_t mono_get_option(const char* name);

#ifdef __cplusplus
}
#endif
#endif /* MONO_EMB_H_ */
