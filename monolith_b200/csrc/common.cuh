// common.cuh — device data structures and primitives of the H100-native collisionless table.
//
// HBM layout of one table (see DESIGN.md §3):
//   buckets : Entry[num_buckets][4]   64-byte bucket = 4 x {fid:int64, row:u32, ts:u32}; the 16-byte
//                                      entry is read with one 128-bit load and mutated with one
//                                      128-bit atomic (atom.cas.b128 / exch.b128, sm_90+), so
//                                      inserts are lock-free (the reference takes two spinlocks per
//                                      id: RT/hash_table/cuckoohash/cuckoohash_map.hpp:489-499).
//   emb     : float[row_cap][emb_stride]   embedding rows, 16-byte aligned, dense (row ids are
//                                      handed out by a bump allocator + free list, the GPU analogue
//                                      of RT/allocator/block_allocator.h:40-120)
//   state   : float[row_cap][state_stride] optimizer state rows in the reference's order
//                                      (RT/hash_table/optimizer/optimizer_combination.cc:58-72)
//   stash   : Entry[stash_cap]         overflow for cuckoo chains that exceed kMaxEvictions
// The expiry timestamp lives in the bucket entry (u32 seconds, RT/hash_table/entry_defs.h:31-39),
// so the TTL scan streams the bucket array only.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mono_emb.h"

namespace mono {

struct __align__(16) Entry {
  int64_t key;
  uint32_t row;
  uint32_t ts;
};
static_assert(sizeof(Entry) == 16, "entry must be 16 bytes");

constexpr uint32_t kEmptyRow = 0xFFFFFFFFu;  // all-ones entry == empty (cudaMemset 0xFF)
constexpr uint32_t kTombRow = 0xFFFFFFFEu;   // deleted stash slot (keeps probe chains intact)
// Bit 31 of a LIVE entry's row marks "being moved by a cuckoo displacement" (cuckoo_insert): the entry is still valid
// (readers strip the bit), other inserters leave it alone.  Row indices are < 2^31.
constexpr uint32_t kMovingBit = 0x80000000u;
constexpr uint32_t kRowMask = 0x7FFFFFFFu;
constexpr int kBucketSlots = 4;
constexpr int kMaxEvictions = 48;
constexpr int kMaxSegs = 8;
constexpr int kThreads = 256;

// counters (uint32) kept in device memory per table
enum Ctr {
  kCtrBump = 0,      // rows ever handed out by the bump allocator
  kCtrFree = 1,      // entries on the free list
  kCtrSize = 2,      // live keys
  kCtrStash = 3,     // live + tomb entries in the stash
  kCtrError = 4,     // sticky error bits (1 = stash overflow, 2 = row slab overflow, 4 = lost a marked slot)
  kCtrMiss = 5,      // scratch: misses of the current upsert call
  kCtrAux = 6,       // scratch
  kCtrMaxTs = 7,     // max update time seen (low 32 bits; ref tf_bridge.cc:202-206 truncates to int)
  kCtrMoves = 8,     // cuckoo displacements ever made (readers on other streams use it to confirm a miss)
  kCtrInflight = 9,  // entries currently carried in a register by the exchange fallback of cuckoo_insert
  kNumCtrs = 16
};

struct SegDev {  // one EntryConfig.Segment (ref: embedding_hash_table.proto:23-33)
  int32_t col_begin;
  int32_t dim;
  int32_t state_off;  // float offset of this segment's optimizer state inside the state row
  int32_t opt_type;
  int32_t init_type;
  float init_a, init_b;
  float p[6];
};

struct TableDev {
  Entry* buckets;
  Entry* stash;
  uint32_t* ctrs;
  uint32_t* free_list;
  float* emb;
  float* state;
  uint32_t num_buckets;
  uint32_t stash_cap;  // power of two
  uint32_t row_cap;
  uint32_t emb_stride;    // floats, multiple of 4
  uint32_t state_stride;  // floats, multiple of 4 (0 when no state)
  int32_t dim;
  int32_t state_dim;
  int32_t num_segs;
  uint32_t default_expire_days;
  int32_t n_slot_expire;
  const uint32_t* slot_expire;  // pairs (slot, days)
  uint64_t seed;
  // counting admission filter (null = the dummy filter: never filters); see filter_add below
  uint32_t* flt_cells;           // uint16 cells packed two per word, [flt_total + 64] cells
  uint32_t flt_total;            // capacity * 1.5
  uint32_t flt_default_thr;
  int32_t n_slot_thr;
  const uint32_t* slot_thr;      // pairs (slot, threshold)
  SegDev segs[kMaxSegs];
};

// One contiguous run of ids of a call that belongs to one table.
struct CallSeg {
  int64_t id_begin;  // first id (inclusive) in the call's id array
  int64_t id_end;    // exclusive
  int64_t val_off;   // float offset of the run's first row in the value / grad / output buffer
  int32_t table;
  int32_t lr_off;    // offset into the call's learning-rate array
};

// ---------------------------------------------------------------------------------------------
// hashing
// ---------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {  // splitmix64 finalizer
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
  x ^= x >> 27; x *= 0x94d049bb133111ebULL;
  x ^= x >> 31;
  return x;
}

__device__ __forceinline__ void bucket_pair(int64_t key, uint32_t nb, uint32_t& b1, uint32_t& b2) {
  uint64_t h = mix64((uint64_t)key);
  b1 = __umulhi((uint32_t)h, nb);
  b2 = __umulhi((uint32_t)(h >> 32), nb);
  if (b2 == b1) b2 = (b1 + 1 == nb) ? 0u : b1 + 1;
}

// Counter-based uniform initializer keyed by (seed, fid, column): reproducible and shard-invariant
// (the reference's thread_local mt19937 is not: RT/hash_table/initializer/
// random_uniform_initializer.cc:31-37).  Mirrored bit-for-bit by oracle/oracle.cc UniformInit.
__host__ __device__ __forceinline__ float uniform_init(uint64_t seed, int64_t fid, int col, float lo,
                                                       float hi) {
  uint64_t h = mix64(mix64(seed ^ 0x9E3779B97F4A7C15ULL) + (uint64_t)fid);
  h = mix64(h + (uint64_t)col * 0xD1B54A32D192ED03ULL);
  float u = (float)(h >> 40) * (1.0f / 16777216.0f);
  return lo + (hi - lo) * u;
}

// ref: NT/data/training_instance/cc/reader_util.h:36-38
__host__ __device__ __forceinline__ uint32_t slot_id_v2(int64_t fid) {
  return (uint32_t)(((uint64_t)fid >> 48) & 0x7FFFu);
}

// ---------------------------------------------------------------------------------------------
// 128-bit entry access
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ Entry ld_entry_nc(const Entry* p) {  // read-only kernels
  uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
  Entry e;
  e.key = (int64_t)(((uint64_t)v.y << 32) | v.x);
  e.row = v.z;
  e.ts = v.w;
  return e;
}
__device__ __forceinline__ Entry ld_entry_cg(const Entry* p) {  // coherent at L2 (insert loops)
  uint4 v = __ldcg(reinterpret_cast<const uint4*>(p));
  Entry e;
  e.key = (int64_t)(((uint64_t)v.y << 32) | v.x);
  e.row = v.z;
  e.ts = v.w;
  return e;
}
__device__ __forceinline__ Entry ld_entry(const Entry* p) {
  uint4 v = *reinterpret_cast<const uint4*>(p);
  Entry e;
  e.key = (int64_t)(((uint64_t)v.y << 32) | v.x);
  e.row = v.z;
  e.ts = v.w;
  return e;
}

__device__ __forceinline__ Entry empty_entry() {
  Entry e;
  e.key = -1;
  e.row = kEmptyRow;
  e.ts = 0xFFFFFFFFu;
  return e;
}

__device__ __forceinline__ bool cas_entry(Entry* addr, const Entry& cmp, const Entry& val) {
  unsigned long long c0 = (unsigned long long)cmp.key, c1 = ((unsigned long long)cmp.ts << 32) | cmp.row;
  unsigned long long v0 = (unsigned long long)val.key, v1 = ((unsigned long long)val.ts << 32) | val.row;
  unsigned long long o0, o1;
  asm volatile(
      "{\n\t.reg .b128 c, v, o;\n\t"
      "mov.b128 c, {%2, %3};\n\tmov.b128 v, {%4, %5};\n\t"
      "atom.global.cas.b128 o, [%6], c, v;\n\t"
      "mov.b128 {%0, %1}, o;\n\t}"
      : "=l"(o0), "=l"(o1)
      : "l"(c0), "l"(c1), "l"(v0), "l"(v1), "l"(addr)
      : "memory");
  return o0 == c0 && o1 == c1;
}

// compare-and-swap that returns the value found (== cmp on success)
__device__ __forceinline__ Entry cas_entry_old(Entry* addr, const Entry& cmp, const Entry& val) {
  unsigned long long c0 = (unsigned long long)cmp.key, c1 = ((unsigned long long)cmp.ts << 32) | cmp.row;
  unsigned long long v0 = (unsigned long long)val.key, v1 = ((unsigned long long)val.ts << 32) | val.row;
  unsigned long long o0, o1;
  asm volatile(
      "{\n\t.reg .b128 c, v, o;\n\t"
      "mov.b128 c, {%2, %3};\n\tmov.b128 v, {%4, %5};\n\t"
      "atom.global.cas.b128 o, [%6], c, v;\n\t"
      "mov.b128 {%0, %1}, o;\n\t}"
      : "=l"(o0), "=l"(o1)
      : "l"(c0), "l"(c1), "l"(v0), "l"(v1), "l"(addr)
      : "memory");
  Entry e;
  e.key = (long long)o0;
  e.row = (uint32_t)o1;
  e.ts = (uint32_t)(o1 >> 32);
  return e;
}

__device__ __forceinline__ Entry exch_entry(Entry* addr, const Entry& val) {
  unsigned long long v0 = (unsigned long long)val.key, v1 = ((unsigned long long)val.ts << 32) | val.row;
  unsigned long long o0, o1;
  asm volatile(
      "{\n\t.reg .b128 v, o;\n\t"
      "mov.b128 v, {%2, %3};\n\t"
      "atom.global.exch.b128 o, [%4], v;\n\t"
      "mov.b128 {%0, %1}, o;\n\t}"
      : "=l"(o0), "=l"(o1)
      : "l"(v0), "l"(v1), "l"(addr)
      : "memory");
  Entry e;
  e.key = (long long)o0;
  e.row = (uint32_t)o1;
  e.ts = (uint32_t)(o1 >> 32);
  return e;
}

// ---------------------------------------------------------------------------------------------
// first-occurrence set: the lowest position of every distinct (key, tag) of a call, in a scratch
// open-addressing set of power-of-two size memset to 0xFF (tag -1 = empty; tags are >= 0).  Which
// slot a key lands in decides no output: first_pos alone does.
// ---------------------------------------------------------------------------------------------
struct FirstOcc {  // viewed as an Entry for the 128-bit CAS: row = tag, ts = first_pos
  int64_t key;
  int32_t tag;
  int32_t first_pos;
};
static_assert(sizeof(FirstOcc) == sizeof(Entry), "a set entry is one 128-bit word");

__device__ __forceinline__ uint32_t first_occ_slot(int64_t key, int tag, uint32_t mask) {
  return (uint32_t)(mix64((uint64_t)key * 0x9E3779B97F4A7C15ULL + (uint64_t)tag) >> 20) & mask;
}

// Position pos claims or joins the slot of (key, tag), probing linearly from slot s; returns that slot.
__device__ __forceinline__ uint32_t claim_first_occ(FirstOcc* set, uint32_t mask, uint32_t s, int64_t key, int tag,
                                                    int32_t pos) {
  while (true) {
    const Entry e = ld_entry_cg(reinterpret_cast<Entry*>(set + s));
    if ((int32_t)e.row == -1) {  // empty
      Entry v;
      v.key = key;
      v.row = (uint32_t)tag;
      v.ts = (uint32_t)pos;
      if (cas_entry(reinterpret_cast<Entry*>(set + s), empty_entry(), v)) return s;
      continue;  // lost the race: re-read the same slot
    }
    if (e.key == key && (int32_t)e.row == tag) {
      // first_pos only ever decreases: skip the atomic when the value just read is already
      // lower (this removes the same-address atomic storm of hot keys in Zipf batches)
      if ((int32_t)e.ts > pos) atomicMin(&set[s].first_pos, pos);
      return s;
    }
    s = (s + 1) & mask;
  }
}

// ---------------------------------------------------------------------------------------------
// lane groups: G lanes (4, 8, 16 or 32) cooperate on one id / one pooled row.  All 32 lanes of a
// warp stay converged (inactive groups run with `active == false`), so full-mask warp votes are legal.
// ---------------------------------------------------------------------------------------------
template <int G>
struct Group {
  static_assert(G == 4 || G == 8 || G == 16 || G == 32, "group size");
  static __device__ __forceinline__ int lane() { return threadIdx.x & 31; }
  static __device__ __forceinline__ int gl() { return threadIdx.x & (G - 1); }
  static __device__ __forceinline__ int base() { return (threadIdx.x & 31) & ~(G - 1); }
  static __device__ __forceinline__ uint32_t mask() {  // lane mask of this thread's group
    if (G == 32) return 0xffffffffu;
    return ((1u << G) - 1u) << base();
  }
  static __device__ __forceinline__ uint32_t bits(uint32_t ballot) {
    if (G == 32) return ballot;
    return (ballot >> base()) & ((1u << G) - 1u);
  }
};

struct Probe {
  uint32_t row;  // kEmptyRow when absent
  Entry* slot;   // address of the matching entry (valid in every lane of the group when found)
};

// Find `key` of table t.  Called by all 32 lanes; `active` is group-uniform.
// LD: 0 = ld.global.nc (read-only kernels), 1 = plain ld (kernels that also write ts).
// Probe order: bucket 1, then bucket 2 for the groups that missed, then the stash if non-empty.
// Warp-ballot compaction: a second / third round is issued only when some group of the warp still
// misses, and only those groups' lanes issue loads.
template <int G, int LD>
__device__ __forceinline__ Probe probe_key(const TableDev* __restrict__ t, int64_t key, bool active,
                                           uint32_t stash_count) {
  const int gl = Group<G>::gl();
  Probe r;
  r.row = kEmptyRow;
  r.slot = nullptr;
  uint32_t b1 = 0, b2 = 0;
  Entry* buckets = t->buckets;
  if (active) bucket_pair(key, t->num_buckets, b1, b2);
  bool pending = active;
#pragma unroll
  for (int round = 0; round < 2; ++round) {
    if (round == 1 && !__any_sync(0xffffffffu, pending)) break;
    uint32_t b = round == 0 ? b1 : b2;
    Entry e;
    e.row = kEmptyRow;
    e.key = 0;
    Entry* p = buckets + (size_t)b * kBucketSlots + (gl & 3);
    if (pending && gl < kBucketSlots) e = LD == 0 ? ld_entry_nc(p) : ld_entry(p);
    bool hit = pending && gl < kBucketSlots && e.key == key && e.row < kTombRow;
    uint32_t bal = Group<G>::bits(__ballot_sync(0xffffffffu, hit));
    int src = Group<G>::base() + (bal ? (__ffs(bal) - 1) : 0);
    uint32_t row = __shfl_sync(0xffffffffu, e.row, src) & kRowMask;
    unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)p, src);
    if (pending && bal) {
      r.row = row;
      r.slot = reinterpret_cast<Entry*>(pp);
      pending = false;
    }
  }
  if (stash_count != 0 && __any_sync(0xffffffffu, pending)) {
    // rare: linear probe of the stash by lane 0 of each pending group
    uint32_t row = kEmptyRow;
    Entry* sp = nullptr;
    if (pending && gl == 0) {
      uint32_t mask = t->stash_cap - 1;
      uint32_t s = (uint32_t)(mix64((uint64_t)key) >> 17) & mask;
      for (uint32_t i = 0; i <= mask; ++i) {
        Entry* p = t->stash + ((s + i) & mask);
        Entry e = ld_entry_cg(p);
        if (e.row == kEmptyRow) break;
        if (e.key == key && e.row < kTombRow) { row = e.row & kRowMask; sp = p; break; }
      }
    }
    int src = Group<G>::base();
    row = __shfl_sync(0xffffffffu, row, src);
    unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)sp, src);
    if (pending && row != kEmptyRow) {
      r.row = row;
      r.slot = reinterpret_cast<Entry*>(pp);
    }
  }
  return r;
}

// Lock-free cuckoo insert of a key known to be ABSENT (callers resolve hits first and keys are
// unique within a call).  One thread per key.  Bucketised (4-slot) 2-choice cuckoo, as libcuckoo
// (ref: cuckoohash_map.hpp:574-588 uprase_fn, :1432 BFS depth) but with 128-bit CAS/EXCH instead of
// bucket locks: claim an empty slot with CAS; when both buckets are full, move a victim to its alternate
// bucket (copy-first, below).  A chain longer than kMaxEvictions parks the carried entry in the stash.
__device__ __forceinline__ bool same_entry(const Entry& a, const Entry& b) {
  return a.key == b.key && a.row == b.row && a.ts == b.ts;
}

// Lock-free insert of a key that is NOT in the table (callers guarantee one inserter per key).
// Displacement is COPY-FIRST and exclusive per victim:
//   1. the victim's slot is MARKED (kMovingBit in its row, one 128-bit CAS): readers strip the bit and still find the
//      entry; other inserters leave a marked entry alone, so exactly one mover works on a victim at a time;
//   2. the victim (unmarked) is CAS-copied into a free slot of ITS alternate bucket — for a moment it is present twice,
//      with the same row;
//   3. the displacement counter is bumped (a reader that probed the alternate bucket before the copy and the old slot
//      after step 4 sees the counter change between its two reads and probes again: rowops.cuh probe_lane_confirm_miss);
//   4. the marked slot is overwritten with `e` (CAS; only a concurrent timestamp bump can make it retry).
// A lookup running at the same time on another stream therefore never misses a key that is in the table (the
// reference's readers hold bucket locks for the same guarantee: cuckoohash_map.hpp find / uprase under lock), and no
// interleaving of movers can leave a key in the table twice: the original stays until ITS mover replaces it, and only
// that mover creates a copy.  If the alternate bucket has no free slot the mark is taken back and the next victim is
// tried; only when all four fail does the insert fall back to the classic step — swap `e` with an (unmarked) victim
// and carry it to its alternate bucket (at <= 60 % load a ~1e-5 event).  While an entry is carried it is in no bucket:
// ctrs[kCtrInflight] counts such entries, and a reader that misses a key while the count is non-zero probes again.
__device__ __forceinline__ bool same_key_row(const Entry& a, const Entry& b) {
  return a.key == b.key && ((a.row ^ b.row) & kRowMask) == 0;
}
__device__ __forceinline__ void cuckoo_insert(const TableDev* __restrict__ t, Entry e) {
  const uint32_t nb = t->num_buckets;
  Entry* buckets = t->buckets;
  const Entry empty = empty_entry();
  uint32_t b1, b2;
  bucket_pair(e.key, nb, b1, b2);
  uint32_t cur = b1;
  bool carrying = false;   // `e` is a displaced RESIDENT entry held in this register (exchange fallback): readers must wait
  auto placed = [&]() {   // the carried entry is in the table again: bump the move counter FIRST, then leave the in-flight
    if (carrying) {       // count — a reader that sees the count at zero then also sees the counter changed and probes again
      __threadfence();
      atomicAdd(t->ctrs + kCtrMoves, 1u);
      __threadfence();
      atomicSub(t->ctrs + kCtrInflight, 1u);
    }
  };
  for (int it = 0; it < kMaxEvictions; ++it) {
    // try every empty slot of `cur`, and on the first iteration of the alternate bucket too
    for (int which = 0; which < (it == 0 ? 2 : 1); ++which) {
      uint32_t b = which == 0 ? cur : (cur == b1 ? b2 : b1);
      Entry* base = buckets + (size_t)b * kBucketSlots;
#pragma unroll
      for (int s = 0; s < kBucketSlots; ++s) {
        Entry o = ld_entry_cg(base + s);
        if (o.row == kEmptyRow && cas_entry(base + s, empty, e)) { placed(); return; }
      }
    }
    // ---- copy-first displacement of one entry of `cur` ----
    const uint32_t v0 = (uint32_t)(mix64((uint64_t)e.key + it) >> 7) & (kBucketSlots - 1);  // deterministic first victim
    bool rescan = false;
    for (int k = 0; k < kBucketSlots && !rescan; ++k) {
      Entry* vp = buckets + (size_t)cur * kBucketSlots + ((v0 + k) & (kBucketSlots - 1));
      const Entry v = ld_entry_cg(vp);
      if (v.row == kEmptyRow) {  // freed meanwhile
        if (cas_entry(vp, empty, e)) { placed(); return; }
        rescan = true;
        break;
      }
      if (v.row & kMovingBit) continue;       // another mover owns this victim
      Entry marked = v;
      marked.row |= kMovingBit;
      if (!cas_entry(vp, v, marked)) {        // changed under us (timestamp bump, another mover, ...): look again
        rescan = true;
        break;
      }
      uint32_t a1, a2;
      bucket_pair(v.key, nb, a1, a2);
      const uint32_t va = cur == a1 ? a2 : a1;
      Entry* ab = buckets + (size_t)va * kBucketSlots;
      bool copied = false;
      for (int s = 0; s < kBucketSlots && !copied; ++s) {
        const Entry o = ld_entry_cg(ab + s);
        if (o.row == kEmptyRow && cas_entry(ab + s, empty, v)) copied = true;
      }
      if (copied) {
        __threadfence();
        atomicAdd(t->ctrs + kCtrMoves, 1u);
        __threadfence();
      }
      // replace the marked original with `e` (copied) or take the mark back (alternate bucket full); nobody but a
      // timestamp bump touches a marked entry, so the loop ends after a retry or two
      Entry seen = marked;
      bool done = false;
      for (int tries = 0; tries < 64 && !done; ++tries) {
        Entry want = e;
        if (!copied) {
          want = seen;
          want.row &= kRowMask;
        }
        const Entry old = cas_entry_old(vp, seen, want);
        if (same_entry(old, seen)) done = true;
        else if (same_key_row(old, seen)) seen = old;   // its timestamp moved
        else break;                                      // cannot happen while the mark is ours (structural ops are stream-ordered)
      }
      if (copied && done) { placed(); return; }   // placed; the victim lives on in its alternate bucket
      if (copied) atomicOr(t->ctrs + kCtrError, 4u);  // lost a marked slot: table changed structurally under an insert
    }
    if (rescan) continue;  // the bucket changed under us: rescan it
    // ---- every victim is owned or its alternate bucket is full: classic step on an unmarked victim ----
    Entry* vp = buckets + (size_t)cur * kBucketSlots + v0;
    Entry victim = ld_entry_cg(vp);
    if (victim.row != kEmptyRow && (victim.row & kMovingBit)) continue;   // wait for its mover (costs an iteration)
    // the victim will be in this register only until it is placed again: announce it (a reader that misses a key while
    // the in-flight count is non-zero probes again, rowops.cuh probe_lane_confirm_miss), then take it out
    const bool first_carry = !carrying && victim.row != kEmptyRow;
    if (first_carry) atomicAdd(t->ctrs + kCtrInflight, 1u);
    atomicAdd(t->ctrs + kCtrMoves, 1u);
    __threadfence();
    if (!cas_entry(vp, victim, e)) {          // changed meanwhile: rescan
      if (first_carry) atomicSub(t->ctrs + kCtrInflight, 1u);
      continue;
    }
    if (victim.row == kEmptyRow) { placed(); return; }   // slot was freed meanwhile: we just filled it
    carrying = true;
    e = victim;
    bucket_pair(e.key, nb, b1, b2);
    cur = (cur == b1) ? b2 : b1;
  }
  // stash.  The count goes up BEFORE the entry appears there: a reader that could see the entry must not skip the stash
  // because it still read a zero count (the count is only ever used as "the stash may be non-empty").
  atomicAdd(t->ctrs + kCtrStash, 1u);
  __threadfence();
  uint32_t mask = t->stash_cap - 1;
  uint32_t s = (uint32_t)(mix64((uint64_t)e.key) >> 17) & mask;
  for (uint32_t i = 0; i <= mask; ++i) {
    Entry* p = t->stash + ((s + i) & mask);
    Entry o = ld_entry_cg(p);
    if (o.row == kEmptyRow && cas_entry(p, empty, e)) {
      placed();
      return;
    }
  }
  atomicOr(t->ctrs + kCtrError, 1u);
  placed();
}

// ---------------------------------------------------------------------------------------------
// fresh rows: every inserter of an upsert call (resolve_miss_kernel, claim_miss_kernel, xmiss_insert_kernel) takes its
// row here.  Ticket k of the call's kCtrMiss count takes the k-th row from the top of the free list, the tickets past
// its end take the bump allocator's next rows in order.  kCtrFree and kCtrBump stay put during the call:
// upsert_finalize_kernel (ops.cu), the other half of this protocol, folds the tickets into them after the call.
// ---------------------------------------------------------------------------------------------
// `key` is absent and admitted, and has exactly one inserter in the call.  Publishes {key, row, ts} with cuckoo_insert
// and returns the row (kFreshBit clear), or kEmptyRow with error bit 2 when the row slab is full.
__device__ __forceinline__ uint32_t insert_new_row(const TableDev* __restrict__ t, int64_t key, uint32_t ts) {
  const uint32_t ticket = atomicAdd(t->ctrs + kCtrMiss, 1u);
  const uint32_t fc = t->ctrs[kCtrFree];
  const uint32_t row = ticket < fc ? t->free_list[fc - 1 - ticket] : t->ctrs[kCtrBump] + (ticket - fc);
  if (row >= t->row_cap) {
    atomicOr(t->ctrs + kCtrError, 2u);
    return kEmptyRow;
  }
  Entry e;
  e.key = key;
  e.row = row;
  e.ts = ts;
  cuckoo_insert(t, e);
  return row;
}

// ---------------------------------------------------------------------------------------------
// epoch-versioned claim set (engine.h ClaimSet, which allocates it): entry key = FID, ts = epoch of the call that
// claimed the slot (any other ts = empty, so the set is never cleared between calls), row = kEmptyRow at the claim,
// then whatever the caller parks there.  A key's slot is found by linear probing from epoch_slot.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t epoch_slot(int64_t key, uint32_t R) {
  return __umulhi((uint32_t)(mix64((uint64_t)key) >> 24), R);
}

// Finds or claims the slot of `key` in the region set[base, base + R), probing linearly from set[base + start]; returns
// its index in set.  BOUNDED gives up after R probes and returns kNoSlot; a caller whose region always has a free slot
// passes false and keeps no probe count.  *won tells whether this thread's CAS claimed the slot (one thread per key and
// call).  LOAD reads each slot first: a stale read only costs a failed CAS, which returns the true entry.
template <Entry (*LOAD)(const Entry*), bool BOUNDED>
__device__ __forceinline__ uint32_t claim_epoch_slot(Entry* set, uint32_t base, uint32_t R, uint32_t start, int64_t key,
                                                     uint32_t epoch, bool* won) {
  uint32_t idx = start;
  *won = false;
  for (uint32_t probes = 0; !BOUNDED || probes < R; ++probes) {
    Entry* p = set + base + idx;
    Entry e = LOAD(p);
    while (e.ts != epoch) {  // empty as far as we can see: claim it (CAS against what we saw)
      Entry ne;
      ne.key = key;
      ne.row = kEmptyRow;
      ne.ts = epoch;
      const Entry old = cas_entry_old(p, e, ne);
      if (same_entry(old, e)) {
        *won = true;
        e = ne;
      } else {
        e = old;  // somebody else changed it: the true entry (claimed this epoch, or a different stale one)
      }
    }
    if (e.key == key) return base + idx;
    idx = idx + 1 == R ? 0 : idx + 1;
  }
  return kNoSlot;
}

// ---------------------------------------------------------------------------------------------
// warp-aggregated append: every lane with `pred` set appends `value` to list, with one atomicAdd on *ctr per warp.
// All 32 lanes of the warp must call it converged (full-mask ballot and shuffle).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_append(bool pred, uint32_t* ctr, uint32_t* list, uint32_t value) {
  const int lane = threadIdx.x & 31;
  const uint32_t bal = __ballot_sync(0xffffffffu, pred);
  if (bal) {
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd(ctr, (uint32_t)__popc(bal));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (pred) list[base + __popc(bal & ((1u << lane) - 1u))] = value;
  }
}

// Batched probe: U independent keys per lane group.  All U bucket loads are issued back to back
// before the first ballot consumes one, so a group keeps U random 64-byte reads in flight instead
// of one (the kernels are latency-bound on dependent HBM round trips, not on bytes).
template <int G, int LD, int U>
__device__ __forceinline__ void probe_keys(const TableDev* __restrict__ t, const int64_t (&key)[U],
                                           const bool (&active)[U], uint32_t stash_count,
                                           uint32_t (&row)[U], Entry* (&slot)[U]) {
  const int gl = Group<G>::gl();
  Entry* buckets = t->buckets;
  const uint32_t nb = t->num_buckets;
  uint32_t b1[U], b2[U];
  bool pending[U];
#pragma unroll
  for (int q = 0; q < U; ++q) {
    b1[q] = b2[q] = 0;
    if (active[q]) bucket_pair(key[q], nb, b1[q], b2[q]);
    pending[q] = active[q];
    row[q] = kEmptyRow;
    slot[q] = nullptr;
  }
#pragma unroll
  for (int round = 0; round < 2; ++round) {
    if (round == 1) {
      bool any = false;
#pragma unroll
      for (int q = 0; q < U; ++q) any |= pending[q];
      if (!__any_sync(0xffffffffu, any)) break;
    }
    Entry e[U];
    Entry* p[U];
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const uint32_t b = round == 0 ? b1[q] : b2[q];
      p[q] = buckets + (size_t)b * kBucketSlots + (gl & 3);
      e[q].row = kEmptyRow;
      e[q].key = 0;
      if (pending[q] && gl < kBucketSlots) e[q] = LD == 0 ? ld_entry_nc(p[q]) : ld_entry(p[q]);
    }
#pragma unroll
    for (int q = 0; q < U; ++q) {
      const bool hit = pending[q] && gl < kBucketSlots && e[q].key == key[q] && e[q].row < kTombRow;
      const uint32_t bal = Group<G>::bits(__ballot_sync(0xffffffffu, hit));
      const int src = Group<G>::base() + (bal ? (__ffs(bal) - 1) : 0);
      const uint32_t r = __shfl_sync(0xffffffffu, e[q].row, src) & kRowMask;
      const unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)p[q], src);
      if (pending[q] && bal) {
        row[q] = r;
        slot[q] = reinterpret_cast<Entry*>(pp);
        pending[q] = false;
      }
    }
  }
  if (stash_count != 0) {
#pragma unroll
    for (int q = 0; q < U; ++q) {
      if (!__any_sync(0xffffffffu, pending[q])) continue;
      uint32_t r = kEmptyRow;
      Entry* sp = nullptr;
      if (pending[q] && gl == 0) {
        const uint32_t mask = t->stash_cap - 1;
        const uint32_t s = (uint32_t)(mix64((uint64_t)key[q]) >> 17) & mask;
        for (uint32_t i = 0; i <= mask; ++i) {
          Entry* pq = t->stash + ((s + i) & mask);
          Entry e = ld_entry_cg(pq);
          if (e.row == kEmptyRow) break;
          if (e.key == key[q] && e.row < kTombRow) { r = e.row & kRowMask; sp = pq; break; }
        }
      }
      r = __shfl_sync(0xffffffffu, r, Group<G>::base());
      const unsigned long long pp = __shfl_sync(0xffffffffu, (unsigned long long)sp, Group<G>::base());
      if (pending[q] && r != kEmptyRow) {
        row[q] = r;
        slot[q] = reinterpret_cast<Entry*>(pp);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Counting admission filter — monolith::hash_filter::HashFilter<uint16_t> (ref: RT/hash_filter/hash_filter.h:34-165,
// filter.h:60-61) on the device: open addressing over total = capacity * 1.5 (+ 64 spill) 16-bit cells, cell =
// 12-bit signature << 4 | 4-bit saturating count, at most 64 probes.  filter_add returns the count BEFORE the
// addition (0 for a new FID, 15 when the probe window is exhausted), like the reference's iterator add (:40-62).
// Cells are updated with a 32-bit CAS on the word that holds them, so concurrent adds of different FIDs are safe;
// the cell a FID lands in depends on the hash (the reference's absl::Hash is salted per process: unpinned there
// too), the counts do not.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t filter_add(const TableDev* __restrict__ t, int64_t fid_, uint32_t count) {
  constexpr uint32_t kMaxCount = 15, kMaxStep = 64;
  const uint64_t fid = (uint64_t)fid_;
  const uint32_t sign = (uint32_t)(((fid >> 17) | (fid << 15)) & 0x0FFFu);  // hash_filter.h:128
  const uint32_t ncell = t->flt_total + kMaxStep;
  uint32_t pos = (uint32_t)(mix64(fid) % (uint64_t)t->flt_total);
  if (count > kMaxCount) count = kMaxCount;
  for (uint32_t step = 0; step < kMaxStep; ++step) {
    uint32_t* wp = t->flt_cells + (pos >> 1);
    const uint32_t shift = (pos & 1u) * 16u;
    uint32_t w = *reinterpret_cast<volatile uint32_t*>(wp);
    while (true) {
      const uint32_t v = (w >> shift) & 0xFFFFu;
      if (v != 0 && (v >> 4) != sign) break;  // somebody else's cell: next probe
      const uint32_t c = v & kMaxCount;
      const uint32_t nv = v == 0 ? ((sign << 4) + count) : (c + count >= kMaxCount ? (v | kMaxCount) : v + count);
      const uint32_t nw = (w & ~(0xFFFFu << shift)) | (nv << shift);
      const uint32_t old = atomicCAS(wp, w, nw);
      if (old == w) return v == 0 ? 0u : c;
      w = old;  // the word changed under us (either half): look again
    }
    if (++pos == ncell) pos = 0;
  }
  return kMaxCount;
}

// ref: HashFilter::ShouldBeFiltered (hash_filter.h:137-144) with the per-slot occurrence thresholds
// (SlotOccurrenceThresholdConfig, embedding_hash_table.proto:100-110): threshold 0 never filters
__device__ __forceinline__ bool should_be_filtered(const TableDev* __restrict__ t, int64_t fid, uint32_t count) {
  if (t->flt_cells == nullptr) return false;
  uint32_t thr = t->flt_default_thr;
  const uint32_t slot = slot_id_v2(fid);
  for (int i = 0; i < t->n_slot_thr; ++i)
    if (t->slot_thr[2 * i] == slot) thr = t->slot_thr[2 * i + 1];
  if (thr == 0) return false;
  return filter_add(t, fid, count) < thr;
}

// binary search: last segment with id_begin <= i (segments are sorted, non-overlapping)
__device__ __forceinline__ int find_seg(const CallSeg* __restrict__ segs, int nsegs, int64_t i) {
  int lo = 0, hi = nsegs - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (segs[mid].id_begin <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

}  // namespace mono
