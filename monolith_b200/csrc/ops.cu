// ops.cu — the hot-path kernels: lookup, fused lookup+pool, and the upsert family
// (optimize / assign / assign_add / reinitialize / restore) with the fused sparse optimizers.
//
// Work decomposition: G lanes (G = 4..32, picked from the row width: one 16-byte vector per lane)
// cooperate on one id.  4 lanes fetch the 64-byte bucket with one 128-bit load each; the match is
// found with a warp ballot; all G lanes then move the row with 128-bit loads/stores.
//
// Why no TMA here: a row is 32..512 bytes at a data-dependent address.  cp.async.bulk needs one
// elected thread + an mbarrier round trip per row and pays off from ~1 KB per copy; at dim 32 a row is
// a single 128-byte line that 8 lanes fetch with one LDG.128 each.  The kernels are bound by random
// 64 B + 128 B HBM accesses in flight, so occupancy (memory-level parallelism), not staging, is the
// lever (DESIGN.md §4).
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "rowops.cuh"

namespace mono {

// ------------------------------------------------------------------------------------------
// lookup
// ------------------------------------------------------------------------------------------
// ref: MultiHashTableLookupOp::Compute / FusedLookupOp (multi_hash_table_lookup_op.cc:37-88,143-197)
// One launch serves every (shard, table) segment of the call.
//
// Two phases per warp-tile of 32 ids (rowops.cuh lookup_tiles): a lane-per-key probe, then a group-per-row copy.
// Used by lookup / fused_lookup (multi-segment) and by lookup_pool when every pooled row has exactly
// one FID (the per-slot case of Criteo/MovieLens/DCN-shaped inputs, where pooling is the identity).
// store one 4-element vector of a row (vector store when the row base is aligned to 4 elements)
template <typename T>
__device__ __forceinline__ void store_vec(T* dst, int c, int D, const float4& x, bool vec_ok) {
  if (c >= D) return;
  if (vec_ok) {
    stcs_row4(dst + c, x);  // streaming: written once, consumed later
  } else {
    const float a[4] = {x.x, x.y, x.z, x.w};
    for (int w = 0; w < 4 && c + w < D; ++w) dst[c + w] = to_row_elem(a[w], dst);
  }
}

// lookup_tiles sink: row ir at base + ir * rs, streaming stores (store_vec)
template <typename T>
struct StreamRows {
  T* base;
  int64_t rs;
  int D;
  bool vec;
  __device__ __forceinline__ T* row(int64_t ir, uint32_t) const { return base + ir * rs; }
  __device__ __forceinline__ void store(T* dst, int c, const float4& x) const { store_vec(dst, c, D, x, vec); }
};

// SINGLE: the call has one segment (one table): table fields and the output base are warp-uniform
// and hoisted, which keeps the kernel at ~40 registers => 6 resident blocks (48 warps) per SM.
// CONFIRM: the call may run beside inserts of another stream (mono_mtable::lookup_must_confirm): misses are confirmed.
// One part of a multi-feature forward (lookup_pool_parts): the one-table forward kernels take an optional array of
// these and then serve part blockIdx.y, with exactly the arguments a single-part launch would have passed.
// A FIRSTN part's sequence length rides in seg.lr_off (a forward has no learning rate): a field of its own would
// change the struct's size and with it the code of every kernel that indexes the array.
struct FwdPart {
  CallSeg seg;                  // lookup_kernel: the part's one segment; lookup_seq_kernel: seg.lr_off = L
  const TableDev* t;
  const int64_t* fids;
  const int32_t* row_offsets;
  int64_t n_rows;
  float* out;
  int64_t out_stride;
  int32_t out_col, pooling;
};

// The kernel bodies below are templates on the output row element T (float, or __nv_bfloat16 for the parts calls'
// bf16 forms, whose FwdPart::out is then a cast pointer); the __global__ kernels instantiate them.
template <typename T, int G, bool SINGLE, bool DUAL, bool CONFIRM>
__device__ __forceinline__ void
lookup_rows(const TableDev* __restrict__ tables, const CallSeg* __restrict__ segs, int nsegs,
            const int64_t* __restrict__ ids, int64_t n_total, T* __restrict__ out,
            int64_t out_stride /* <= 0: rows packed at dim elements */, int out_col, int prefetch,
            const FwdPart* __restrict__ parts) {
  if (SINGLE && parts) {
    const FwdPart& p = parts[blockIdx.y];
    segs = &p.seg;
    ids = p.fids;
    n_total = p.n_rows;
    out = reinterpret_cast<T*>(p.out);
    out_stride = p.out_stride;
    out_col = p.out_col;
  }
  if constexpr (SINGLE) {  // hoisted table / output description
    const TileLanes<G> ln;
    const TableRows tab = table_rows(tables + segs[0].table);
    const int64_t rs0 = out_stride > 0 ? out_stride : tab.D;
    T* const base0 = out + segs[0].val_off - segs[0].id_begin * rs0 + out_col;
    const bool vec0 = (tab.D & 3) == 0 && (rs0 & 3) == 0 && (reinterpret_cast<uintptr_t>(base0) & (4 * sizeof(T) - 1)) == 0;
    lookup_tiles<T, G, DUAL, CONFIRM>(ln, IdKeys<true>{tab, n_total, ids, prefetch}, StreamRows<T>{base0, rs0, tab.D, vec0});
    return;
  }
  // several segments: the tile loop of lookup_tiles with the table, output base and stride of each position's segment
  constexpr int RPI = 32 / G;
  constexpr int ITERS = G;
  constexpr int UNR = 4;
  const int lane = threadIdx.x & 31, gl = Group<G>::gl(), grp = lane / G;
  const int c = gl * 4;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * 32;
  const int64_t wfirst = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * 32;
  int64_t key_next = wfirst + lane < n_total ? __ldg(ids + wfirst + lane) : 0;
  for (int64_t wbase = wfirst; wbase < n_total; wbase += wstride) {
    const int64_t i = wbase + lane;
    const int64_t key = key_next;
    if (i + wstride < n_total) key_next = __ldg(ids + i + wstride);
    int si = 0;
    uint32_t row = kEmptyRow;
    if (i < n_total) {
      si = find_seg(segs, nsegs, i);
      const TableDev* tk = tables + segs[si].table;
      row = probe_lane<DUAL>(tk, key);
      if (CONFIRM && row == kEmptyRow) row = probe_lane_confirm_miss(tk, key);  // inserts on another stream
    }
#pragma unroll
    for (int it0 = 0; it0 < ITERS; it0 += UNR) {
      float4 x[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int src_lane = (it0 + u) * RPI + grp;
        const uint32_t r = __shfl_sync(0xffffffffu, row, src_lane);
        x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int s_r = __shfl_sync(0xffffffffu, si, src_lane);
        if (r != kEmptyRow) {
          const TableDev* t = tables + segs[s_r].table;
          if (c < t->dim) x[u] = __ldg(reinterpret_cast<const float4*>(t->emb + (size_t)r * t->emb_stride + c));
        }
      }
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        const int src_lane = (it0 + u) * RPI + grp;
        const int64_t ir = wbase + src_lane;
        // shuffles read lanes outside the group: all 32 lanes take part, before any divergence
        const uint32_t r_st = __shfl_sync(0xffffffffu, row, src_lane);
        const int s_st = __shfl_sync(0xffffffffu, si, src_lane);
        if (ir >= n_total) continue;
        const CallSeg sg = segs[s_st];
        const TableDev* t = tables + sg.table;
        const int D = t->dim;
        const int64_t rs = out_stride > 0 ? out_stride : D;
        T* dst = out + sg.val_off + (ir - sg.id_begin) * rs + out_col;
        const bool vec_ok = (D & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & (4 * sizeof(T) - 1)) == 0;
        store_vec(dst, c, D, x[u], vec_ok);
        if (D > 4 * G) {
          for (int cc = c + 4 * G; cc < D; cc += 4 * G) {
            float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r_st != kEmptyRow) y = __ldg(reinterpret_cast<const float4*>(t->emb + (size_t)r_st * t->emb_stride + cc));
            store_vec(dst, cc, D, y, vec_ok);
          }
        }
      }
    }
  }
}

template <int G, bool SINGLE, bool DUAL = false, bool CONFIRM = true>
__global__ void __launch_bounds__(kThreads, SINGLE && !DUAL ? 6 : 4)
lookup_kernel(const TableDev* __restrict__ tables, const CallSeg* __restrict__ segs, int nsegs,
              const int64_t* __restrict__ ids, int64_t n_total, float* __restrict__ out,
              int64_t out_stride /* <= 0: rows packed at dim floats */, int out_col, int prefetch,
              const FwdPart* __restrict__ parts = nullptr) {
  lookup_rows<float, G, SINGLE, DUAL, CONFIRM>(tables, segs, nsegs, ids, n_total, out, out_stride, out_col, prefetch,
                                               parts);
}

// mono_mtable_lookup_f16: lookup_kernel with fp16 output rows, each element rounded once where it is stored (a miss
// stores +0.0).  The same arguments as lookup_kernel; parts is always null here.
template <int G, bool SINGLE, bool DUAL = false, bool CONFIRM = true>
__global__ void __launch_bounds__(kThreads, SINGLE && !DUAL ? 6 : 4)
f16_lookup_kernel(const TableDev* __restrict__ tables, const CallSeg* __restrict__ segs, int nsegs,
                  const int64_t* __restrict__ ids, int64_t n_total, __half* __restrict__ out, int64_t out_stride,
                  int out_col, int prefetch, const FwdPart* __restrict__ parts = nullptr) {
  lookup_rows<__half, G, SINGLE, DUAL, CONFIRM>(tables, segs, nsegs, ids, n_total, out, out_stride, out_col, prefetch,
                                                parts);
}

// one-FID parts of lookup_pool_parts_bf16 (lookup_kernel<G, true, false, CONFIRM> with bf16 rows)
template <int G, bool CONFIRM>
__global__ void __launch_bounds__(kThreads, 6)
bf16_lookup_kernel(const TableDev* __restrict__ tables, int prefetch, const FwdPart* __restrict__ parts) {
  lookup_rows<__nv_bfloat16, G, true, false, CONFIRM>(tables, nullptr, 1, nullptr, 0, nullptr, 0, 0, prefetch, parts);
}

// lookup_tiles source: slot q -> its row r (the tag), and its FID when position j = q - r*L holds one
struct SeqKeys {
  static constexpr bool kAhead = false, kTag = true;
  TableRows tab;
  int64_t n;
  const int64_t* __restrict__ fids;
  const int32_t* __restrict__ offs;
  uint32_t L;
  __device__ __forceinline__ bool key(int64_t q, int64_t& key, uint32_t& r) const {
    r = (uint32_t)q / L;
    const uint32_t j = (uint32_t)q - r * L;
    int64_t b = r, e = (int64_t)r + 1;
    if (offs) {
      b = __ldg(offs + r);
      e = __ldg(offs + r + 1);
    }
    if ((int64_t)j >= e - b) return false;
    key = __ldg(fids + b + j);
    return true;
  }
};

// lookup_tiles sink: position j of row r at base + r * rs + j * D
template <typename T>
struct SeqRows : StreamRows<T> {
  uint32_t L;
  __device__ __forceinline__ T* row(int64_t ir, uint32_t r) const {
    return this->base + (int64_t)r * this->rs + (int64_t)((uint32_t)ir - r * L) * this->D;
  }
};

// FIRSTN parts of lookup_pool_parts (ref: GatherEmb's FIRSTN branch, fused_embedding_to_layout.h:251-256): part
// blockIdx.y writes n_rows x L positions of dim floats, position j of row r at out + r*out_stride + out_col + j*dim.
// lookup_kernel<G, true>'s two phases over position slots q = r*L + j instead of ids: a slot with j < n_r probes
// FID fids[offs[r] + j] (lane per key), a slot with j >= n_r probes nothing; phase B copies a found row and stores
// zeros for the rest.  n_rows * L <= 2^31 (checked by the launcher), so slots divide in 32 bits.  4 blocks per SM
// (64 registers): at 6 (40 registers) it spills, and so it does with lookup_kernel's next-tile FID prefetch.
template <typename T, int G, bool CONFIRM>
__device__ __forceinline__ void seq_rows(const FwdPart* __restrict__ parts) {
  const FwdPart& p = parts[blockIdx.y];
  const uint32_t L = (uint32_t)p.seg.lr_off;
  const int64_t n_total = p.n_rows * L;
  const int32_t* __restrict__ offs = p.row_offsets;
  const int64_t* __restrict__ fids = p.fids;
  const TileLanes<G> ln;
  const TableRows tab = table_rows(p.t);
  const int64_t rs0 = p.out_stride;
  T* const base0 = reinterpret_cast<T*>(p.out) + p.out_col;
  const bool vec0 = (tab.D & 3) == 0 && (rs0 & 3) == 0 && (reinterpret_cast<uintptr_t>(base0) & (4 * sizeof(T) - 1)) == 0;
  lookup_tiles<T, G, false, CONFIRM>(ln, SeqKeys{tab, n_total, fids, offs, L}, SeqRows<T>{{base0, rs0, tab.D, vec0}, L});
}

template <int G, bool CONFIRM>
__global__ void __launch_bounds__(kThreads, 4)
lookup_seq_kernel(const FwdPart* __restrict__ parts) {
  seq_rows<float, G, CONFIRM>(parts);
}

template <int G, bool CONFIRM>
__global__ void __launch_bounds__(kThreads, 4)
bf16_seq_kernel(const FwdPart* __restrict__ parts) {
  seq_rows<__nv_bfloat16, G, CONFIRM>(parts);
}

// lookup_tiles sink: row ir into the window of the part that holds ir
struct PeerRows : PlainStore {
  const int64_t* start;  // the part boundaries (shared memory)
  const PeerOut& po;
  __device__ __forceinline__ float* row(int64_t ir, uint32_t) const {
    const int pr = peer_part(start, po.n, ir);
    return reinterpret_cast<float*>(po.base[pr]) + (ir - start[pr]) * D;
  }
};

// Owner lookup fused with the row exchange of the sharded forward (replaces FusedLookup + the
// embedding all-to-all, ref: distributed_ps_sync.py:100-118): ids[] is the concatenation of the FID
// buckets the requesters stored into this rank's window; the row of id i is written straight into the
// window of the requester that asked for it (one 128-bit NVLink store per lane, a whole row per group).
// Same two phases as lookup_kernel<G, true>, every miss confirmed.
template <int G>
__global__ void __launch_bounds__(kThreads, 6)
lookup_push_kernel(const TableDev* __restrict__ t0, const int64_t* __restrict__ ids, int64_t n_total,
                   const PeerOut po) {
  __shared__ int64_t s_start[kMaxPeers + 1];
  peer_starts(po, s_start);
  const TileLanes<G> ln;
  const TableRows tab = table_rows(t0);
  lookup_tiles<float, G, false, true>(ln, IdKeys<false>{tab, n_total, ids, 0}, PeerRows{{tab.D}, s_start, po});
}

// ------------------------------------------------------------------------------------------
// TMA-staged lookup (single table, packed output rows): the north-star's "TMA to stage rows through shared memory".
// Per warp tile of 32 FIDs:
//   A. lane-per-key probe (as above) -> 32 row indices;
//   B. every lane that found its FID issues ONE bulk copy global -> shared of its whole row
//      (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes, 64..512 B, SASS UBLKCP): 32 row
//      fetches in flight per warp at zero register cost; absent FIDs get zeros written by their lane;
//   C. while the copies fly the warp probes its NEXT tile (software pipeline: the FID -> bucket -> row chain of
//      tile t+1 hides behind the row traffic of tile t);
//   D. mbarrier wait, then ONE bulk store shared -> global of the tile's 32 contiguous output rows
//      (cp.async.bulk.global.shared::cta, 2..16 KB).
// The rows never touch registers.  Two tile buffers per warp, so the store of tile t drains while tile t+1 loads.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(mbar), "r"(parity)
        : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t mbar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(mbar)
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

template <int ROWB>  // bytes per row: dim * 4, a multiple of 16
__global__ void __launch_bounds__(kThreads)
lookup_tma_kernel(const TableDev* __restrict__ t0, const int64_t* __restrict__ ids, int64_t n_total,
                  float* __restrict__ out, const FwdPart* __restrict__ parts = nullptr) {
  if (parts) {
    const FwdPart& p = parts[blockIdx.y];
    t0 = p.t;
    ids = p.fids;
    n_total = p.n_rows;
    out = p.out;
  }
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int NW = kThreads / 32;
  constexpr int TILEB = 32 * ROWB;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned char* buf0 = smem_raw + (size_t)(w * 2) * TILEB;
  const uint32_t buf_s0 = smem_u32(buf0);
  uint64_t* mb = reinterpret_cast<uint64_t*>(smem_raw + (size_t)NW * 2 * TILEB) + w * 2;
  const uint32_t mbar0 = smem_u32(mb);
  if (lane == 0) {
    mbar_init(mbar0, 1);
    mbar_init(mbar0 + 8, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const float* __restrict__ emb0 = t0->emb;
  const uint32_t stride0 = t0->emb_stride;
  const int64_t ntiles = (n_total + 31) / 32;
  const int64_t tstride = (int64_t)gridDim.x * NW;
  int64_t tile = (int64_t)blockIdx.x * NW + w;
  uint32_t row = kEmptyRow;
  if (tile < ntiles && tile * 32 + lane < n_total) {
    const int64_t key0 = __ldg(ids + tile * 32 + lane);
    row = probe_lane(t0, key0);
    if (row == kEmptyRow) row = probe_lane_confirm_miss(t0, key0);
  }
  // FIDs of the tile after this one: requested one iteration before they are probed (off the dependent chain)
  int64_t key_next = (tile + tstride < ntiles && (tile + tstride) * 32 + lane < n_total) ? __ldg(ids + (tile + tstride) * 32 + lane) : 0;
  for (uint32_t it = 0; tile < ntiles; ++it) {
    const int b = it & 1;
    const uint32_t parity = (it >> 1) & 1u;
    const uint32_t buf_s = buf_s0 + (uint32_t)b * TILEB, mbar = mbar0 + (uint32_t)b * 8;
    if (it >= 2) {  // buffer b was read by the bulk store of iteration it - 2
      if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      __syncwarp();
    }
    const int nvalid = (int)min((int64_t)32, n_total - tile * 32);
    const uint32_t found = __ballot_sync(0xffffffffu, row != kEmptyRow);
    if (lane == 0) mbar_expect_tx(mbar, (uint32_t)__popc(found) * ROWB);
    __syncwarp();
    if (row != kEmptyRow) {
      bulk_g2s(buf_s + lane * ROWB, emb0 + (size_t)row * stride0, ROWB, mbar);
    } else if (lane < nvalid) {
      uint4* z = reinterpret_cast<uint4*>(buf0 + (size_t)b * TILEB + (size_t)lane * ROWB);
#pragma unroll
      for (int q = 0; q < ROWB / 16; ++q) z[q] = make_uint4(0u, 0u, 0u, 0u);
    }
    // ---- the next tile's probe chain runs while this tile's rows are in flight ----
    const int64_t next = tile + tstride;
    const int64_t key_cur = key_next;
    if (next + tstride < ntiles && (next + tstride) * 32 + lane < n_total) key_next = __ldg(ids + (next + tstride) * 32 + lane);
    uint32_t row_next = kEmptyRow;
    if (next < ntiles && next * 32 + lane < n_total) {
      row_next = probe_lane(t0, key_cur);
      if (row_next == kEmptyRow) row_next = probe_lane_confirm_miss(t0, key_cur);
    }
    mbar_wait(mbar, parity);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the zero rows (generic proxy) before the bulk store reads them
    __syncwarp();
    if (lane == 0) bulk_s2g(out + (size_t)tile * 32 * (ROWB / 4), buf_s, (uint32_t)nvalid * ROWB);
    tile = next;
    row = row_next;
  }
  if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // shared memory must outlive the reads
  __syncwarp();
}

__global__ void __launch_bounds__(kThreads)
contains_kernel(const TableDev* __restrict__ t, const int64_t* __restrict__ ids, int64_t n,
                uint8_t* __restrict__ out) {
  constexpr int G = 4, GPW = 8;
  const int lane = threadIdx.x & 31;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * GPW;
  for (int64_t wbase = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * GPW; wbase < n;
       wbase += wstride) {
    const int64_t i = wbase + lane / G;
    const bool active = i < n;
    int64_t key = active ? ids[i] : 0;
    Probe pr = probe_key<G, 0>(t, key, active, t->ctrs[kCtrStash]);
    if (active && Group<G>::gl() == 0) out[i] = pr.row != kEmptyRow;
  }
}

// flat entry dump [emb | state | found | ts]
__global__ void __launch_bounds__(kThreads)
lookup_entry_kernel(const TableDev* __restrict__ t, const int64_t* __restrict__ ids, int64_t n,
                    float* __restrict__ out) {
  constexpr int G = 8, GPW = 4;
  const int lane = threadIdx.x & 31, gl = Group<G>::gl();
  const int W = t->dim + t->state_dim + 2;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * GPW;
  for (int64_t wbase = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * GPW; wbase < n;
       wbase += wstride) {
    const int64_t i = wbase + lane / G;
    const bool active = i < n;
    int64_t key = active ? ids[i] : 0;
    Probe pr = probe_key<G, 1>(t, key, active, t->ctrs[kCtrStash]);
    if (!active) continue;
    float* dst = out + i * W;
    if (pr.row == kEmptyRow) {
      for (int c = gl; c < W; c += G) dst[c] = 0.0f;
    } else {
      const float* w = t->emb + (size_t)pr.row * t->emb_stride;
      const float* s = t->state + (size_t)pr.row * t->state_stride;
      for (int c = gl; c < t->dim; c += G) dst[c] = w[c];
      for (int c = gl; c < t->state_dim; c += G) dst[t->dim + c] = s[c];
      if (gl == 0) {
        dst[t->dim + t->state_dim] = __uint_as_float(1u);
        dst[t->dim + t->state_dim + 1] = __uint_as_float(ld_entry(pr.slot).ts);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// fused lookup + pool (forward headline kernel)
// ------------------------------------------------------------------------------------------
// One lane group per pooled output row: walk the row's FIDs in order, probe, gather the 16-byte
// vectors of the embedding row and accumulate in registers; one coalesced store per output row.
// Terms are added in FID order => bit-exact with the CPU reference's pooling
// (ref: OptimizedSumpooling, fused_embedding_to_layout.cc:26-59; ReduceSumOp, reduce_op.cc:29-51).
template <typename T, int G, int NV, int U>  // NV = 16-byte vectors per lane (dim <= 4*G*NV); U = rows in flight
__device__ __forceinline__ void
pool_rows(const TableDev* __restrict__ t, const int64_t* __restrict__ fids, const int32_t* __restrict__ row_offsets,
          int64_t n_rows, int pooling, T* __restrict__ out, int64_t out_stride, int out_col,
          const FwdPart* __restrict__ parts) {
  if (parts) {
    const FwdPart& p = parts[blockIdx.y];
    t = p.t;
    fids = p.fids;
    row_offsets = p.row_offsets;
    n_rows = p.n_rows;
    pooling = p.pooling;
    out = reinterpret_cast<T*>(p.out);
    out_stride = p.out_stride;
    out_col = p.out_col;
  }
  constexpr int GPW = 32 / G;
  const int lane = threadIdx.x & 31, gl = Group<G>::gl();
  const int D = t->dim;
  const uint32_t stash = t->ctrs[kCtrStash];
  const float* __restrict__ emb = t->emb;
  const uint32_t stride = t->emb_stride;
  // a warp owns GPW*U consecutive pooled rows per iteration; group g takes rows g, g+GPW, ...
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * GPW * U;
  for (int64_t wbase = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * GPW * U;
       wbase < n_rows; wbase += wstride) {
    int64_t r[U], b[U];
    int n[U];
    int nloc = 0;
#pragma unroll
    for (int q = 0; q < U; ++q) {
      r[q] = wbase + q * GPW + lane / G;
      b[q] = 0;
      n[q] = 0;
      if (r[q] < n_rows) {
        b[q] = row_offsets ? row_offsets[r[q]] : r[q];
        n[q] = row_offsets ? (int)(row_offsets[r[q] + 1] - b[q]) : 1;
      }
      nloc = max(nloc, n[q]);
    }
    const int nmax = row_offsets ? __reduce_max_sync(0xffffffffu, nloc) : 1;
    float4 acc[U][NV];
#pragma unroll
    for (int q = 0; q < U; ++q)
#pragma unroll
      for (int v = 0; v < NV; ++v) acc[q][v] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < nmax; ++j) {
      int64_t key[U];
      bool active[U];
      uint32_t row[U];
      Entry* slot[U];
#pragma unroll
      for (int q = 0; q < U; ++q) {
        active[q] = j < n[q];
        key[q] = active[q] ? __ldg(fids + b[q] + j) : 0;
      }
      probe_keys<G, 0, U>(t, key, active, stash, row, slot);
#pragma unroll
      for (int q = 0; q < U; ++q) {  // misses are confirmed against inserts running on another stream
        const bool miss = active[q] && row[q] == kEmptyRow;
        if (!__any_sync(0xffffffffu, miss)) continue;
        uint32_t r2 = kEmptyRow;
        if (miss && gl == 0) r2 = probe_lane_confirm_miss(t, key[q]);
        r2 = __shfl_sync(0xffffffffu, r2, Group<G>::base());
        if (miss) row[q] = r2;
      }
      float4 x[U][NV];
#pragma unroll
      for (int q = 0; q < U; ++q)
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          const int c = (v * G + gl) * 4;
          x[q][v] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (active[q] && row[q] != kEmptyRow && c < D)
            x[q][v] = __ldg(reinterpret_cast<const float4*>(emb + (size_t)row[q] * stride + c));
        }
#pragma unroll
      for (int q = 0; q < U; ++q) {
        if (!active[q]) continue;
        const float fn = (float)n[q];
#pragma unroll
        for (int v = 0; v < NV; ++v) {
          float4 xv = x[q][v];
          if (pooling == MONO_POOL_MEAN) {
            xv.x = __fdiv_rn(xv.x, fn); xv.y = __fdiv_rn(xv.y, fn);
            xv.z = __fdiv_rn(xv.z, fn); xv.w = __fdiv_rn(xv.w, fn);
          }
          if (j == 0) {
            acc[q][v] = xv;
          } else {
            acc[q][v].x = __fadd_rn(acc[q][v].x, xv.x); acc[q][v].y = __fadd_rn(acc[q][v].y, xv.y);
            acc[q][v].z = __fadd_rn(acc[q][v].z, xv.z); acc[q][v].w = __fadd_rn(acc[q][v].w, xv.w);
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < U; ++q) {
      if (r[q] >= n_rows) continue;
      T* dst = out + r[q] * out_stride + out_col;
      const bool vec_ok = (D & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & (4 * sizeof(T) - 1)) == 0;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int c = (v * G + gl) * 4;
        if (c >= D) continue;
        if (vec_ok) {
          stcs_row4(dst + c, acc[q][v]);  // streaming: written once, read later
        } else {
          const float a[4] = {acc[q][v].x, acc[q][v].y, acc[q][v].z, acc[q][v].w};
          for (int w = 0; w < 4 && c + w < D; ++w) dst[c + w] = to_row_elem(a[w], dst);
        }
      }
    }
  }
}

template <int G, int NV, int U>
__global__ void __launch_bounds__(kThreads)
lookup_pool_kernel(const TableDev* __restrict__ t, const int64_t* __restrict__ fids,
                   const int32_t* __restrict__ row_offsets, int64_t n_rows, int pooling,
                   float* __restrict__ out, int64_t out_stride, int out_col,
                   const FwdPart* __restrict__ parts = nullptr) {
  pool_rows<float, G, NV, U>(t, fids, row_offsets, n_rows, pooling, out, out_stride, out_col, parts);
}

template <int G, int NV, int U>
__global__ void __launch_bounds__(kThreads)
bf16_pool_kernel(const FwdPart* __restrict__ parts) {
  pool_rows<__nv_bfloat16, G, NV, U>(nullptr, nullptr, nullptr, 0, 0, nullptr, 0, 0, parts);
}

// CSR pooling, staged: the round-1 kernel above walks a pooled row's FIDs one at a time (FID -> bucket -> row per step:
// 2-3 dependent HBM round trips per FID, 0.16 of the roofline at 4 FIDs per row).  Here a lane group takes U = 4 pooled
// rows at once and treats their FIDs as ONE flat list of up to kStage = 16 entries: every lane probes its share of the
// list (lane per key, the whole 64-byte bucket per lane), then ALL rows of the list are requested together with cp.async
// into per-thread shared-memory slots (this lane's 16-byte slice of each row), and the sums run in FID order out of
// shared memory: three round trips per 16 FIDs instead of two per FID.  Longer lists are walked in chunks of 16 with
// the accumulators carried.  Terms are added in FID order: bit-exact with the CPU reference's pooling.
// T = __nv_bfloat16: the output base only needs 8-byte alignment (4 elements), as the fp32 form's 16.
template <typename T, int G, int U>  // U: pooled rows per lane group
__device__ __forceinline__ void
pool_staged_rows(const TableDev* __restrict__ t, const int64_t* __restrict__ fids,
                 const int32_t* __restrict__ row_offsets, int64_t n_rows, int pooling, T* __restrict__ out,
                 int64_t out_stride, int out_col, const FwdPart* __restrict__ parts) {
  if (parts) {
    const FwdPart& p = parts[blockIdx.y];
    t = p.t;
    fids = p.fids;
    row_offsets = p.row_offsets;
    n_rows = p.n_rows;
    pooling = p.pooling;
    out = reinterpret_cast<T*>(p.out);
    out_stride = p.out_stride;
    out_col = p.out_col;
  }
  constexpr int GPW = 32 / G;
  constexpr int KPL = kStage / G > 0 ? kStage / G : 1;  // keys probed per lane and chunk
  extern __shared__ float4 stage_raw[];  // [kStage][kThreads]
  float4 (*stage)[kThreads] = reinterpret_cast<float4 (*)[kThreads]>(stage_raw);
  const int lane = threadIdx.x & 31, gl = Group<G>::gl();
  const uint32_t gmask = Group<G>::mask();
  const int gb = Group<G>::base();
  const int c = gl * 4;
  const int D = t->dim;
  const float* __restrict__ emb = t->emb;
  const uint32_t stride = t->emb_stride;
  const bool in = c < D;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / 32) * GPW * U;
  for (int64_t r0 = (((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * GPW + lane / G) * U; r0 < n_rows;
       r0 += gstride) {
    // the group's U rows cover the flat FID range [f_begin, f_end)
    int32_t ro[U + 1];
#pragma unroll
    for (int q = 0; q <= U; ++q) ro[q] = row_offsets[min(r0 + q, n_rows)];
    const int64_t f_begin = ro[0], f_end = ro[U];
    float4 acc[U];
#pragma unroll
    for (int q = 0; q < U; ++q) acc[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int64_t f0 = f_begin; f0 < f_end; f0 += kStage) {
      const int cnt = (int)min((int64_t)kStage, f_end - f0);
      // ---- probe: lane gl takes flat entries gl, gl + G, ... ----
      // (all key loads first, then all first-bucket loads: the KPL probe chains of a lane overlap instead of queueing)
      uint32_t rk[KPL];
      int64_t key[KPL];
      const Entry* bk[KPL];
      Entry e0[KPL], e1[KPL], e2[KPL], e3[KPL];
#pragma unroll
      for (int s = 0; s < KPL; ++s) {
        const int k = s * G + gl;
        key[s] = (k < cnt && k < kStage) ? __ldg(fids + f0 + k) : 0;
      }
#pragma unroll
      for (int s = 0; s < KPL; ++s) {
        uint32_t b1, b2;
        bucket_pair(key[s], t->num_buckets, b1, b2);
        bk[s] = t->buckets + (size_t)b1 * kBucketSlots;
        e0[s] = ld_entry_nc(bk[s]); e1[s] = ld_entry_nc(bk[s] + 1); e2[s] = ld_entry_nc(bk[s] + 2); e3[s] = ld_entry_nc(bk[s] + 3);
      }
#pragma unroll
      for (int s = 0; s < KPL; ++s) {
        const int k = s * G + gl;
        uint32_t row = kEmptyRow;
        if (e0[s].key == key[s] && e0[s].row < kTombRow) row = e0[s].row & kRowMask;
        if (e1[s].key == key[s] && e1[s].row < kTombRow) row = e1[s].row & kRowMask;
        if (e2[s].key == key[s] && e2[s].row < kTombRow) row = e2[s].row & kRowMask;
        if (e3[s].key == key[s] && e3[s].row < kTombRow) row = e3[s].row & kRowMask;
        const bool live = k < cnt && k < kStage;
        if (live && row == kEmptyRow) row = probe_lane(t, key[s]);  // second bucket / stash: the full probe
        if (live && row == kEmptyRow) row = probe_lane_confirm_miss(t, key[s]);  // inserts on another stream
        rk[s] = live ? row : kEmptyRow;
      }
      // ---- request every row of the chunk ----
#pragma unroll
      for (int k = 0; k < kStage; ++k) {
        uint32_t mine = rk[0];
#pragma unroll
        for (int s = 1; s < KPL; ++s)
          if (k / G == s) mine = rk[s];
        const uint32_t row = __shfl_sync(gmask, mine, gb + (k % G));
        if (k < cnt && row != kEmptyRow && in) cp_async16(&stage[k][threadIdx.x], emb + (size_t)row * stride + c);
        else if (in) stage[k][threadIdx.x] = make_float4(0.f, 0.f, 0.f, 0.f);  // absent FID -> zeros
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      // ---- pool in FID order ----
#pragma unroll
      for (int k = 0; k < kStage; ++k) {
        if (k >= cnt) break;
        const int64_t f = f0 + k;
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in) x = stage[k][threadIdx.x];
#pragma unroll
        for (int qq = 0; qq < U; ++qq) {  // which of the U rows owns flat entry f (compile-time indices: no local arrays)
          if (f < ro[qq] || f >= ro[qq + 1]) continue;
          float4 y = x;
          if (pooling == MONO_POOL_MEAN) {
            const float fn = (float)(ro[qq + 1] - ro[qq]);
            y.x = __fdiv_rn(y.x, fn); y.y = __fdiv_rn(y.y, fn); y.z = __fdiv_rn(y.z, fn); y.w = __fdiv_rn(y.w, fn);
          }
          if (f == ro[qq]) {
            acc[qq] = y;
          } else {
            acc[qq].x = __fadd_rn(acc[qq].x, y.x); acc[qq].y = __fadd_rn(acc[qq].y, y.y);
            acc[qq].z = __fadd_rn(acc[qq].z, y.z); acc[qq].w = __fadd_rn(acc[qq].w, y.w);
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < U; ++q) {
      if (r0 + q >= n_rows || !in) continue;
      T* dst = out + (r0 + q) * out_stride + out_col;
      stcs_row4(dst + c, acc[q]);  // an empty row pools to zeros
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads, 2)
lookup_pool_staged_kernel(const TableDev* __restrict__ t, const int64_t* __restrict__ fids,
                          const int32_t* __restrict__ row_offsets, int64_t n_rows, int pooling,
                          float* __restrict__ out, int64_t out_stride, int out_col,
                          const FwdPart* __restrict__ parts = nullptr) {
  constexpr int U = 4;
  pool_staged_rows<float, G, U>(t, fids, row_offsets, n_rows, pooling, out, out_stride, out_col, parts);
}

template <int G>
__global__ void __launch_bounds__(kThreads, 2)
bf16_pool_staged_kernel(const FwdPart* __restrict__ parts) {
  constexpr int U = 4;
  pool_staged_rows<__nv_bfloat16, G, U>(nullptr, nullptr, nullptr, 0, 0, nullptr, 0, 0, parts);
}

// ------------------------------------------------------------------------------------------
// upsert family
// ------------------------------------------------------------------------------------------
struct UpsertArgs {
  const TableDev* tables;
  const CallSeg* segs;
  int nsegs;
  const int64_t* ids;
  const uint32_t* idx_list = nullptr;  // optional indirection: item j is ids[idx_list[j]]
  int64_t n;                           // number of items to process
  const uint32_t* n_dev = nullptr;     // optional: item count on device (overrides n when non-null)
  const float* vals;
  const float* lr;           // device copy of the call's learning rates
  uint32_t update_ts;
  uint32_t* miss_ctr;        // global miss counter of the call
  uint32_t* miss_list;       // item indices j that missed
  uint32_t* rowidx;          // per item j: resolved row (bit 31 = freshly inserted)
  int32_t* status = nullptr; // reinitialize only
  int64_t pos0 = 0;          // apply pass without idx_list: item j is position pos0 + j
  // admission filter (tables without one never filter): 0 = not consulted (reinitialize, restore); 1 = ids ABSENT
  // from the table consult it (optimize: tf_bridge.cc:296-326; assign: :181-185); 2 = every id does (AssignAdd2
  // has no Contains check, tf_bridge.cc:224-232)
  int filter_mode = 0;
  const uint32_t* occ_extra = nullptr;  // dedup path: occurrences of id position i beyond the first (count = 1 + occ_extra[i])
  // duplicate rounds with filter_mode 1: absent0[i] = id position i was absent from the table at call start
  const uint8_t* absent0 = nullptr;
  // apply pass of the device-driven sharded step: do not start before *wait_flag >= wait_seq (the requester's
  // gradient rows have landed in this rank's window; acquire at system scope)
  const uint64_t* wait_flag = nullptr;
  uint64_t wait_seq = 0;
};
__device__ __forceinline__ uint32_t restore_ts(const UpsertArgs& a, const CallSeg& sg, const TableDev* t,
                                               int64_t i) {
  const int width = t->dim + t->state_dim + 2;
  return __float_as_uint(a.vals[sg.val_off + (i - sg.id_begin) * width + t->dim + t->state_dim + 1]);
}

// Pass 1 — resolve present keys, lane per key (32 independent probe chains per warp): row index to
// rowidx[j], expiry timestamp bumped in the bucket entry (ref: entry.SetTimestamp(update_time),
// cuckoo_embedding_hash_table.cc:243); misses are compacted with a warp ballot + one atomic per warp.
template <bool RESTORE>
__global__ void __launch_bounds__(kThreads) resolve_hit_kernel(UpsertArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t n = a.n_dev ? (int64_t)*a.n_dev : a.n;
  const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * 32;
  for (int64_t wbase = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * 32; wbase < n;
       wbase += wstride) {
    const int64_t j = wbase + lane;
    bool miss = false;
    if (j < n) {
      const int64_t i = a.idx_list ? (int64_t)a.idx_list[j] : j;
      const CallSeg sg = a.segs[a.nsegs > 1 ? find_seg(a.segs, a.nsegs, i) : 0];
      const TableDev* t = a.tables + sg.table;
      Entry* slot = nullptr;
      const uint32_t row = probe_lane_slot(t, a.ids[i], &slot);
      if (row == kEmptyRow) {
        miss = true;
      } else if (a.filter_mode == 2 && should_be_filtered(t, a.ids[i], 1)) {
        a.rowidx[j] = kEmptyRow;  // AssignAdd2: filtered although present — the op is skipped for this id
      } else {
        // an id absent at call start adds 1 per occurrence, also once an earlier round has admitted it: the reference
        // filters the whole id list before it writes a row (tf_bridge.cc:179-190, 312-326).  It stays admitted.
        if (a.absent0 && a.absent0[i]) (void)should_be_filtered(t, a.ids[i], 1);
        slot->ts = RESTORE ? restore_ts(a, sg, t, i) : a.update_ts;
        a.rowidx[j] = row;
      }
    }
    warp_append(miss, a.miss_ctr, a.miss_list, (uint32_t)j);
  }
}

// Pass 2 — absent keys (unique within the call), thread per key: take a row and publish {fid, row, ts}
// (insert_new_row).  The row contents are written by the apply pass (fresh bit set).
template <bool RESTORE>
__global__ void __launch_bounds__(kThreads) resolve_miss_kernel(UpsertArgs a) {
  const int64_t n = (int64_t)*a.miss_ctr;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n;
       q += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = a.miss_list[q];
    const int64_t i = a.idx_list ? (int64_t)a.idx_list[j] : j;
    const CallSeg sg = a.segs[a.nsegs > 1 ? find_seg(a.segs, a.nsegs, i) : 0];
    const TableDev* t = a.tables + sg.table;
    if (a.filter_mode != 0 && should_be_filtered(t, a.ids[i], a.occ_extra ? 1u + a.occ_extra[i] : 1u)) {
      a.rowidx[j] = kEmptyRow;  // not admitted yet: no row, the apply pass skips it
      continue;
    }
    const uint32_t row = insert_new_row(t, a.ids[i], RESTORE ? restore_ts(a, sg, t, i) : a.update_ts);
    a.rowidx[j] = row == kEmptyRow ? row : row | kFreshBit;  // kEmptyRow: row slab overflow, the apply skips it
  }
}

// Before the duplicate rounds of a filtered optimize / assign: which id positions are absent from the table.
__global__ void __launch_bounds__(kThreads) absent_at_start_kernel(UpsertArgs a, uint8_t* __restrict__ absent0) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * blockDim.x) {
    const CallSeg sg = a.segs[a.nsegs > 1 ? find_seg(a.segs, a.nsegs, i) : 0];
    Entry* slot;
    absent0[i] = probe_lane_slot(a.tables + sg.table, a.ids[i], &slot) == kEmptyRow;
  }
}

// Fold the call's per-table miss tickets into the allocator counters.
__global__ void upsert_finalize_kernel(const TableDev* tables, const int32_t* table_ids, int ntab,
                                       uint32_t* miss_ctr, uint32_t update_ts) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q == 0) *miss_ctr = 0;
  if (q >= ntab) return;
  const TableDev* t = tables + table_ids[q];
  uint32_t m = t->ctrs[kCtrMiss];
  uint32_t fc = t->ctrs[kCtrFree];
  if (m <= fc) {
    t->ctrs[kCtrFree] = fc - m;
  } else {
    t->ctrs[kCtrFree] = 0;
    t->ctrs[kCtrBump] += m - fc;
  }
  t->ctrs[kCtrSize] += m;
  t->ctrs[kCtrMiss] = 0;
  if (update_ts > t->ctrs[kCtrMaxTs]) t->ctrs[kCtrMaxTs] = update_ts;
}

// Pass 3 — apply the op to the resolved rows, lane group per row (pure streaming over w / state /
// value rows: no hash logic left here).
template <int G, int OP>
__global__ void __launch_bounds__(kThreads) upsert_apply_kernel(UpsertArgs a) {
  if (a.wait_flag) {
    if (threadIdx.x == 0) {
      uint64_t v;
      do {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(a.wait_flag) : "memory");
      } while (v < a.wait_seq);
    }
    __syncthreads();
  }
  const int gl = Group<G>::gl();
  const int64_t n = a.n_dev ? (int64_t)*a.n_dev : a.n;
  const int64_t gstride = (int64_t)gridDim.x * (kThreads / G);
  for (int64_t j = (int64_t)blockIdx.x * (kThreads / G) + threadIdx.x / G; j < n; j += gstride) {
    const uint32_t ri = a.rowidx[j];
    if (ri == kEmptyRow) continue;  // row slab overflow was flagged
    const int64_t i = a.idx_list ? (int64_t)a.idx_list[j] : j + a.pos0;
    const CallSeg sg = a.segs[a.nsegs > 1 ? find_seg(a.segs, a.nsegs, i) : 0];
    const TableDev* t = a.tables + sg.table;
    const bool fresh = (ri & kFreshBit) != 0;
    const int width = OP == kOpRestore ? t->dim + t->state_dim + 2 : t->dim;
    const float* v = a.vals ? a.vals + sg.val_off + (i - sg.id_begin) * width : nullptr;
    if (OP == kOpReinit && gl == 0) a.status[i] = fresh ? 0 : 1;
    apply_row<G, OP>(t, ri & ~kFreshBit, a.ids[i], v, a.lr + sg.lr_off, fresh);
  }
}

// ---- duplicate handling (ids not guaranteed unique) ------------------------------------------
// every pending position claims / joins the set slot of its (table, fid) and lowers first_pos
__global__ void __launch_bounds__(kThreads)
dup_claim_kernel(const CallSeg* __restrict__ segs, int nsegs, const int64_t* __restrict__ ids,
                 const uint32_t* __restrict__ pending, int64_t n, FirstOcc* set, uint32_t mask,
                 uint32_t* __restrict__ slot_of, const uint32_t* __restrict__ n_dev = nullptr) {
  if (n_dev) n = (int64_t)*n_dev;
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n;
       j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = pending ? (int64_t)pending[j] : j;
    const int table = segs[nsegs > 1 ? find_seg(segs, nsegs, i) : 0].table;
    const int64_t key = ids[i];
    slot_of[j] = claim_first_occ(set, mask, first_occ_slot(key, table, mask), key, table, (int32_t)i);
  }
}

// split pending into leaders (lowest pending position of their key) and the rest
__global__ void __launch_bounds__(kThreads)
dup_split_kernel(const uint32_t* __restrict__ pending, int64_t n, const FirstOcc* __restrict__ set,
                 const uint32_t* __restrict__ slot_of, uint32_t* leaders, uint32_t* rest,
                 uint32_t* ctr /*[0]=leaders,[1]=rest*/, uint32_t* leader_of /*optional, by position*/) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n;
       j += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t i = pending ? pending[j] : (uint32_t)j;
    const int32_t fp = set[slot_of[j]].first_pos;
    if (leader_of) leader_of[i] = (uint32_t)fp;
    if ((uint32_t)fp == i) leaders[atomicAdd(ctr, 1u)] = i;
    else rest[atomicAdd(ctr + 1, 1u)] = i;
  }
}

// Misses of a call whose segments are each duplicate-free but may share FIDs with one another (the
// owner side of the sharded backward: one segment per requesting rank).  The lowest position of a
// missing FID inserts it (leaders -> resolve_miss_kernel); the others take the leader's row, not fresh.
__global__ void __launch_bounds__(kThreads)
miss_split_kernel(const uint32_t* __restrict__ miss_list, const uint32_t* __restrict__ n_miss,
                  const FirstOcc* __restrict__ set, const uint32_t* __restrict__ slot_of,
                  uint32_t* __restrict__ leaders, uint32_t* __restrict__ followers,
                  uint32_t* __restrict__ fol_leader, uint32_t* ctr /*[1] = leaders, [2] = followers*/) {
  const int64_t n = *n_miss;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t i = miss_list[q];
    const uint32_t fp = (uint32_t)set[slot_of[q]].first_pos;
    if (fp == i) {
      leaders[atomicAdd(ctr + 1, 1u)] = i;
    } else {
      const uint32_t k = atomicAdd(ctr + 2, 1u);
      followers[k] = i;
      fol_leader[k] = fp;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
miss_follow_kernel(const uint32_t* __restrict__ followers, const uint32_t* __restrict__ fol_leader,
                   const uint32_t* __restrict__ n_fol, uint32_t* __restrict__ rowidx) {
  const int64_t n = *n_fol;
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t r = rowidx[fol_leader[k]];
    rowidx[followers[k]] = r == kEmptyRow ? r : (r & ~kFreshBit);
  }
}

// acc_row(leader_of[i]) += vals_row(i) for this round's items (one item per key per round)
template <int G>
__global__ void __launch_bounds__(kThreads)
dup_accumulate_kernel(const TableDev* __restrict__ tables, const CallSeg* __restrict__ segs, int nsegs,
                      const uint32_t* __restrict__ items, const uint32_t* n_dev,
                      const uint32_t* __restrict__ leader_of, const float* __restrict__ vals,
                      float* __restrict__ acc, uint32_t* __restrict__ occ_extra /* optional */) {
  const int64_t n = *n_dev;
  const int gl = Group<G>::gl();
  for (int64_t j = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / G; j < n;
       j += (int64_t)gridDim.x * blockDim.x / G) {
    const int64_t i = items[j];
    const int64_t l = leader_of[i];
    const int si = nsegs > 1 ? find_seg(segs, nsegs, i) : 0;
    const CallSeg sg = segs[si];
    const int D = tables[sg.table].dim;
    const float* src = vals + sg.val_off + (i - sg.id_begin) * D;
    float* dst = acc + sg.val_off + (l - sg.id_begin) * D;  // leader is in the same segment? see host
    for (int c = gl; c < D; c += G) dst[c] = __fadd_rn(dst[c], src[c]);
    if (occ_extra && gl == 0) occ_extra[l] += 1u;  // one item per key and round: no race
  }
}

// ------------------------------------------------------------------------------------------
// host launchers
// ------------------------------------------------------------------------------------------
int pick_group(int max_dim) {
  int v = (max_dim + 3) / 4;
  int g = 4;
  while (g < v && g < 32) g <<= 1;
  return g;
}

CallBlob stage_call(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const float* lr_host, int n_lr,
                    cudaStream_t s) {
  size_t seg_bytes = sizeof(CallSeg) * (size_t)nsegs;
  size_t lr_bytes = sizeof(float) * (size_t)std::max(n_lr, 1);
  std::vector<int32_t> tabs;
  for (int i = 0; i < nsegs; ++i)
    if (std::find(tabs.begin(), tabs.end(), h_segs[i].table) == tabs.end())
      tabs.push_back(h_segs[i].table);
  size_t lr_off = (seg_bytes + 15) & ~(size_t)15;
  size_t tab_off = (lr_off + lr_bytes + 15) & ~(size_t)15;
  size_t total = tab_off + sizeof(int32_t) * tabs.size();
  if (total > StageRing::kBlockBytes) throw ArgError("too many segments in one call");
  int b = mt->ring.acquire();
  char* h = mt->ring.h(b);
  std::memcpy(h, h_segs, seg_bytes);
  if (n_lr > 0) std::memcpy(h + lr_off, lr_host, sizeof(float) * n_lr);
  std::memcpy(h + tab_off, tabs.data(), sizeof(int32_t) * tabs.size());
  mt->ring.commit(b, total, s);
  CallBlob cb;
  cb.segs = reinterpret_cast<const CallSeg*>(mt->ring.d(b));
  cb.lr = reinterpret_cast<const float*>(mt->ring.d(b) + lr_off);
  cb.table_ids = reinterpret_cast<const int32_t*>(mt->ring.d(b) + tab_off);
  cb.ntab = (int)tabs.size();
  return cb;
}

static int max_dim_of(mono_mtable* mt, const CallSeg* h_segs, int nsegs) {
  int m = 1;
  for (int i = 0; i < nsegs; ++i) m = std::max(m, mt->tables[h_segs[i].table].dim);
  return m;
}

// whether the TMA variant serves a one-FID-per-row lookup of table k into out_dev.  fp32 rows only: it copies rows
// unchanged, so fp16 output rows (mono_mtable_lookup_f16) always take the register path (f16_lookup_kernel).
static bool tma_applies(mono_mtable* mt, int k, const float* out_dev, int64_t out_stride, int out_col) {
  static const int env_mode = [] {  // MONO_LOOKUP_TMA=0/1 presets mono_set_option("lookup_tma")
    const char* e = std::getenv("MONO_LOOKUP_TMA");
    if (e) g_opt_lookup_tma.store(std::atoi(e) != 0);
    return 0;
  }();
  (void)env_mode;
  if (g_opt_lookup_tma.load(std::memory_order_relaxed) == 0) return false;
  const HostTable& ht = mt->tables[k];
  const int D = ht.dim;
  const int rowb = D * 4;
  // 128- and 256-byte rows only: on an H100 the staged copy wins at dim 32 and 64, while at dim 16 (64-byte rows, one
  // sector pair per lane group) the register path is faster with Zipf-skewed FIDs (bench.py --workload c5)
  if ((D & 3) || (rowb != 128 && rowb != 256)) return false;
  if (out_col != 0 || (out_stride > 0 && out_stride != D) || (reinterpret_cast<uintptr_t>(out_dev) & 15)) return false;
  if (ht.dev.emb_stride != (uint32_t)D) return false;  // rows are 16-byte aligned and contiguous when dim % 4 == 0
  return true;
}

// TMA lookup of rows of `rowb` bytes; parts != null: one grid row (blockIdx.y) per part, n_total = the largest
static void launch_tma(int rowb, const TableDev* t, const int64_t* ids_dev, int64_t n_total, float* out_dev,
                       const FwdPart* parts, int n_parts, cudaStream_t s) {
  constexpr int NW = kThreads / 32;
  auto launch = [&](auto rb) {
    constexpr int RB = decltype(rb)::value;
    constexpr size_t smem = (size_t)NW * 2 * 32 * RB + NW * 2 * 8;
    set_max_dynamic_smem<lookup_tma_kernel<RB>>(smem);
    const int grid = resident_grid(lookup_tma_kernel<RB>, (n_total + 31) / 32, NW, kThreads, smem);
    lookup_tma_kernel<RB><<<dim3(grid, n_parts), kThreads, smem, s>>>(t, ids_dev, n_total, out_dev, parts);
  };
  if (rowb == 128) launch(Int<128>{});
  else launch(Int<256>{});
  MONO_CHECK_LAUNCH();
}

// launcher: returns false when the TMA variant does not apply (the caller falls back to lookup_kernel)
static bool try_lookup_tma(mono_mtable* mt, int k, const int64_t* ids_dev, int64_t n_total, float* out_dev,
                           int64_t out_stride, int out_col, cudaStream_t s) {
  if (!tma_applies(mt, k, out_dev, out_stride, out_col)) return false;
  launch_tma(mt->tables[k].dim * 4, mt->d_tables + k, ids_dev, n_total, out_dev, nullptr, 1, s);
  return true;
}

static void launch_lookup_staged(mono_mtable* mt, const CallSeg* d_segs, int nsegs, int G,
                                 const int64_t* ids_dev, int64_t n_total, float* out_dev,
                                 int64_t out_stride, int out_col, cudaStream_t s) {
  const int pf = knob(KNOB_LOOKUP_PF);
  by_group(G, [&](auto g) {
    constexpr int GG = decltype(g)::value;
    const auto kern = nsegs == 1 && knob(KNOB_LOOKUP_DUAL) ? lookup_kernel<GG, true, true>
                      : nsegs == 1 && !mt->lookup_must_confirm(s) ? lookup_kernel<GG, true, false, false>
                      : nsegs == 1 ? lookup_kernel<GG, true>
                      : lookup_kernel<GG, false>;
    kern<<<resident_grid(kern, n_total, kThreads), kThreads, 0, s>>>(mt->d_tables, d_segs, nsegs, ids_dev, n_total,
                                                                     out_dev, out_stride, out_col, pf, nullptr);
  });
  MONO_CHECK_LAUNCH();
}

// fp16 output rows: the same selection over f16_lookup_kernel
static void launch_lookup_staged(mono_mtable* mt, const CallSeg* d_segs, int nsegs, int G,
                                 const int64_t* ids_dev, int64_t n_total, __half* out_dev,
                                 int64_t out_stride, int out_col, cudaStream_t s) {
  const int pf = knob(KNOB_LOOKUP_PF);
  by_group(G, [&](auto g) {
    constexpr int GG = decltype(g)::value;
    const auto kern = nsegs == 1 && knob(KNOB_LOOKUP_DUAL) ? f16_lookup_kernel<GG, true, true>
                      : nsegs == 1 && !mt->lookup_must_confirm(s) ? f16_lookup_kernel<GG, true, false, false>
                      : nsegs == 1 ? f16_lookup_kernel<GG, true>
                      : f16_lookup_kernel<GG, false>;
    kern<<<resident_grid(kern, n_total, kThreads), kThreads, 0, s>>>(mt->d_tables, d_segs, nsegs, ids_dev, n_total,
                                                                     out_dev, out_stride, out_col, pf, nullptr);
  });
  MONO_CHECK_LAUNCH();
}

template <typename T>
void launch_lookup(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const int64_t* ids_dev,
                   int64_t n_total, T* out_dev, cudaStream_t s) {
  if (n_total <= 0) return;
  upload_tables(mt, s);
  // merge adjacent segments of the same table whose ids and output rows are contiguous (fused_lookup
  // of a single table: N shard segments collapse into one -> hoisted single-table kernel)
  std::vector<CallSeg> merged;
  for (int i = 0; i < nsegs; ++i) {
    if (!merged.empty()) {
      CallSeg& b = merged.back();
      const int D = mt->tables[b.table].dim;
      if (b.table == h_segs[i].table && b.id_end == h_segs[i].id_begin &&
          b.val_off + (b.id_end - b.id_begin) * D == h_segs[i].val_off) {
        b.id_end = h_segs[i].id_end;
        continue;
      }
    }
    merged.push_back(h_segs[i]);
  }
  h_segs = merged.data();
  nsegs = (int)merged.size();
  if constexpr (std::is_same_v<T, float>) {
    if (nsegs == 1 && h_segs[0].id_begin == 0 &&
        try_lookup_tma(mt, h_segs[0].table, ids_dev, n_total, out_dev + h_segs[0].val_off, 0, 0, s))
      return;
  }
  CallBlob cb = stage_call(mt, h_segs, nsegs, nullptr, 0, s);
  launch_lookup_staged(mt, cb.segs, nsegs, pick_group(max_dim_of(mt, h_segs, nsegs)), ids_dev, n_total,
                       out_dev, 0, 0, s);
}
template void launch_lookup<float>(mono_mtable*, const CallSeg*, int, const int64_t*, int64_t, float*, cudaStream_t);
template void launch_lookup<__half>(mono_mtable*, const CallSeg*, int, const int64_t*, int64_t, __half*, cudaStream_t);

void launch_lookup_push(mono_mtable* mt, int k, const int64_t* ids_dev, int64_t n_total, const PeerOut& po,
                        cudaStream_t s) {
  if (n_total <= 0) return;
  const int D = mt->tables[k].dim;
  if (D & 3) throw ArgError("lookup_push needs dim % 4 == 0 (16-byte peer stores)");
  if (po.start[po.n] != n_total) throw ArgError("lookup_push: counts do not add up to the id count");
  upload_tables(mt, s);
  const TableDev* t = mt->d_tables + k;
  by_group(pick_group(D), [&](auto g) {
    constexpr int GG = decltype(g)::value;
    lookup_push_kernel<GG><<<resident_grid(lookup_push_kernel<GG>, n_total, kThreads), kThreads, 0, s>>>(t, ids_dev,
                                                                                                         n_total, po);
  });
  MONO_CHECK_LAUNCH();
}

// The kernel that serves a lookup_pool of one table (lookup_pool_parts launches each distinct one once)
struct PoolPlan {
  enum Kind { kTma, kLookup, kStaged, kPool, kSeq } kind;
  int a, b, c;  // kTma: row bytes; kLookup: G, variant (0 dual, 1 no miss confirm, 2 confirm); kStaged: G; kPool: G, nv;
                // kSeq (FIRSTN, parts only): G, whether misses are confirmed
  bool bf16;    // bf16 output rows (lookup_pool_parts_bf16): the bf16_* kernels
  bool operator==(const PoolPlan& o) const {
    return kind == o.kind && a == o.a && b == o.b && c == o.c && bf16 == o.bf16;
  }
};

// bf16 output rows (lookup_pool_parts_bf16: the bf16_* kernels) take the register-path kernels only: the TMA lookup
// never touches registers, and the conversion needs them, so a one-FID part takes the lookup kernel at any dim; the
// lookup_dual knob does not apply; and the staged kernel's 4-element output vectors are 8 bytes, not 16.
static PoolPlan plan_lookup_pool(mono_mtable* mt, const FwdPart& p, bool bf16, cudaStream_t s) {
  const int k = p.seg.table;
  const int D = mt->tables[k].dim;
  const int G = pick_group(D);
  const bool confirm = mt->lookup_must_confirm(s);
  if (p.pooling == MONO_POOL_FIRSTN) return {PoolPlan::kSeq, G, confirm ? 1 : 0, 0, bf16};
  const int nv = (D + 4 * G - 1) / (4 * G);
  const int64_t n_rows = p.n_rows, out_stride = p.out_stride;
  const int out_col = p.out_col;
  const float* out = p.out;
  const uintptr_t out_align = bf16 ? 7 : 15;
  if (p.row_offsets == nullptr) {
    // one FID per pooled row: SUM and MEAN are the identity (x / 1 == x): probe + gather only
    if (!bf16 && tma_applies(mt, k, p.out, p.out_stride, p.out_col)) return {PoolPlan::kTma, D * 4, 0, 0, false};
    return {PoolPlan::kLookup, G, !bf16 && knob(KNOB_LOOKUP_DUAL) ? 0 : !confirm ? 1 : 2, 0, bf16};
  }
  if ((D & 3) == 0 && D <= 128 && (out_stride & 3) == 0 && (out_col & 3) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & out_align) == 0 && n_rows < ((int64_t)1 << 31))
    return {PoolPlan::kStaged, G, 0, 0, bf16};
  return {PoolPlan::kPool, G, nv <= 2 ? nv : 4, 0, bf16};  // nv 3 and 4 share an instantiation
}

// a: the arguments of a single-table call (parts == null), or of any part of a parts launch whose kernels then serve
// part blockIdx.y of `parts` (n_rows: the largest part's pool_work, sizes the grid).  A bf16 plan's kernels read every
// argument from `parts`.
static void launch_pool_plan(mono_mtable* mt, const PoolPlan& pl, const FwdPart& a, const FwdPart* parts,
                             int n_parts, cudaStream_t s) {
  const int64_t n_rows = a.n_rows;
  if (pl.kind == PoolPlan::kTma) {
    launch_tma(pl.a, a.t, a.fids, n_rows, a.out, parts, n_parts, s);
    return;
  }
  // one resident wave of `per` rows per block, one grid row per part
  auto launch = [&](auto kern, int per, size_t smem, auto... args) {
    kern<<<dim3(resident_grid(kern, n_rows, per, kThreads, smem), n_parts), kThreads, smem, s>>>(args...);
  };
  by_group(pl.a, [&](auto g) {
    constexpr int G = decltype(g)::value;
    if (pl.kind == PoolPlan::kSeq) {
      if (pl.bf16) launch(pl.b ? bf16_seq_kernel<G, true> : bf16_seq_kernel<G, false>, kThreads, 0, parts);
      else launch(pl.b ? lookup_seq_kernel<G, true> : lookup_seq_kernel<G, false>, kThreads, 0, parts);
    } else if (pl.kind == PoolPlan::kLookup) {
      const int pf = knob(KNOB_LOOKUP_PF);
      if (pl.bf16) {
        launch(pl.b == 2 ? bf16_lookup_kernel<G, true> : bf16_lookup_kernel<G, false>, kThreads, 0, mt->d_tables, pf,
               parts);
      } else {
        const CallSeg* d_seg = parts ? &parts[0].seg : stage_call(mt, &a.seg, 1, nullptr, 0, s).segs;
        launch(pl.b == 0 ? lookup_kernel<G, true, true> : pl.b == 1 ? lookup_kernel<G, true, false, false>
                                                                    : lookup_kernel<G, true>,
               kThreads, 0, mt->d_tables, d_seg, 1, a.fids, n_rows, a.out, a.out_stride, a.out_col, pf, parts);
      }
    } else if (pl.kind == PoolPlan::kStaged) {
      constexpr size_t kStageBytes = sizeof(float4) * kStage * kThreads;
      if (pl.bf16) {
        set_max_dynamic_smem<bf16_pool_staged_kernel<G>>(kStageBytes);
        launch(bf16_pool_staged_kernel<G>, (kThreads / G) * 4, kStageBytes, parts);
      } else {
        set_max_dynamic_smem<lookup_pool_staged_kernel<G>>(kStageBytes);
        launch(lookup_pool_staged_kernel<G>, (kThreads / G) * 4, kStageBytes, a.t, a.fids, a.row_offsets, n_rows,
               a.pooling, a.out, a.out_stride, a.out_col, parts);
      }
    } else {
      // U rows in flight per lane group: enough independent HBM round trips per warp to cover latency
      auto pool = [&](auto nv, auto u) {
        constexpr int NV = decltype(nv)::value, U = decltype(u)::value;
        if (pl.bf16) launch(bf16_pool_kernel<G, NV, U>, (kThreads / G) * U, 0, parts);
        else launch(lookup_pool_kernel<G, NV, U>, (kThreads / G) * U, 0, a.t, a.fids, a.row_offsets, n_rows, a.pooling,
                    a.out, a.out_stride, a.out_col, parts);
      };
      const int nv = pl.b;
      if constexpr (G < 32) pool(Int<1>{}, Int<4>{});
      else if (nv == 1) pool(Int<1>{}, Int<4>{});
      else if (nv == 2) pool(Int<2>{}, Int<2>{});
      else pool(Int<4>{}, Int<1>{});
    }
  });
  MONO_CHECK_LAUNCH();
}

static FwdPart fwd_part(mono_mtable* mt, int k, const int64_t* fids_dev, const int32_t* row_offsets, int64_t n_rows,
                        int pooling, float* out, int64_t out_stride, int out_col) {
  FwdPart p;
  p.seg.id_begin = 0;
  p.seg.id_end = n_rows;
  p.seg.val_off = 0;
  p.seg.table = k;
  p.seg.lr_off = 0;
  p.t = mt->d_tables + k;
  p.fids = fids_dev;
  p.row_offsets = row_offsets;
  p.n_rows = n_rows;
  p.out = out;
  p.out_stride = out_stride;
  p.out_col = out_col;
  p.pooling = pooling;
  return p;
}

void launch_lookup_pool(mono_mtable* mt, int k, const int64_t* fids_dev, const int32_t* row_offsets,
                        int64_t n_rows, int pooling, float* out, int64_t out_stride, int out_col,
                        cudaStream_t s) {
  if (n_rows <= 0) return;
  if (pooling != MONO_POOL_SUM && pooling != MONO_POOL_MEAN)
    throw ArgError("lookup_pool supports SUM and MEAN pooling");
  upload_tables(mt, s);
  const int D = mt->tables[k].dim;
  if (D > 512) throw ArgError("lookup_pool supports dim <= 512");
  const FwdPart a = fwd_part(mt, k, fids_dev, row_offsets, n_rows, pooling, out, out_stride, out_col);
  launch_pool_plan(mt, plan_lookup_pool(mt, a, false, s), a, nullptr, 1, s);
}

// The grid work of a part: its rows, or for FIRSTN its n_rows * L position slots
static int64_t pool_work(const FwdPart& f) {
  return f.pooling == MONO_POOL_FIRSTN ? f.n_rows * f.seg.lr_off : f.n_rows;
}

// Every SUM / MEAN part exactly as lookup_pool would serve it alone, every FIRSTN part by lookup_seq_kernel, and the
// parts served by the same kernel share one launch: one grid row per part, the parts' arguments in one staged array.
// bf16: rows_dev of every part is bf16 storage (stride and col in bf16 elements), served by the bf16_* kernels.
void run_lookup_pool_parts(mono_mtable* mt, const mono_pool_part* parts, int n_parts, cudaStream_t s, bool bf16) {
  const int K = (int)mt->tables.size();
  if (n_parts < 0 || n_parts > MONO_MAX_POOL_PARTS) throw ArgError("lookup_pool_parts: bad part count");
  if (n_parts > 0 && !parts) throw ArgError("lookup_pool_parts: null argument");
  for (int i = 0; i < n_parts; ++i) {
    const mono_pool_part& p = parts[i];
    if (p.table < 0 || p.table >= K) throw ArgError("lookup_pool_parts: bad table index");
    if (p.pooling != MONO_POOL_SUM && p.pooling != MONO_POOL_MEAN && p.pooling != MONO_POOL_FIRSTN)
      throw ArgError("lookup_pool_parts: SUM, MEAN or FIRSTN");
    if (p.n_rows < 0 || p.n_fids < 0) throw ArgError("lookup_pool_parts: negative count");
    check_firstn("lookup_pool_parts", p);
    if (!p.row_offsets_dev && p.n_rows != p.n_fids)
      throw ArgError("lookup_pool_parts: n_rows must equal n_fids without offsets");
    if (p.n_rows > 0 && (!p.rows_dev || (p.n_fids > 0 && !p.fids_dev))) throw ArgError("lookup_pool_parts: null argument");
    if (mt->tables[p.table].dim > 512) throw ArgError("lookup_pool_parts supports dim <= 512");
  }
  upload_tables(mt, s);
  // group the parts by the kernel that serves them, in order of first use
  std::vector<PoolPlan> plans;
  std::vector<std::vector<FwdPart>> groups;
  for (int i = 0; i < n_parts; ++i) {
    const mono_pool_part& p = parts[i];
    if (p.n_rows == 0) continue;
    FwdPart f = fwd_part(mt, p.table, p.fids_dev, p.row_offsets_dev, p.n_rows, p.pooling, p.rows_dev, p.stride, p.col);
    if (p.pooling == MONO_POOL_FIRSTN) f.seg.lr_off = p.max_seq_len;
    const PoolPlan pl = plan_lookup_pool(mt, f, bf16, s);
    size_t g = 0;
    while (g < plans.size() && !(plans[g] == pl)) ++g;
    if (g == plans.size()) {
      plans.push_back(pl);
      groups.emplace_back();
    }
    groups[g].push_back(f);
  }
  if (plans.empty()) return;
  const int rb = mt->ring.acquire();
  char* h = mt->ring.h(rb);
  size_t off = 0;
  for (const auto& g : groups) {
    std::memcpy(h + off, g.data(), sizeof(FwdPart) * g.size());
    off += sizeof(FwdPart) * g.size();
  }
  static_assert(sizeof(FwdPart) * MONO_MAX_POOL_PARTS <= StageRing::kBlockBytes, "the parts fit one staged block");
  mt->ring.commit(rb, off, s);
  const FwdPart* d = reinterpret_cast<const FwdPart*>(mt->ring.d(rb));
  for (size_t g = 0; g < plans.size(); ++g) {
    FwdPart a = groups[g][0];
    for (const FwdPart& f : groups[g]) a.n_rows = std::max(a.n_rows, pool_work(f));
    launch_pool_plan(mt, plans[g], a, d, (int)groups[g].size(), s);
    d += groups[g].size();
  }
}

void launch_contains(mono_mtable* mt, int k, const int64_t* ids, int64_t n, uint8_t* out,
                     cudaStream_t s) {
  if (n <= 0) return;
  upload_tables(mt, s);
  contains_kernel<<<grid_for(n, kThreads / 4), kThreads, 0, s>>>(mt->d_tables + k, ids, n, out);
  MONO_CHECK_LAUNCH();
}

void launch_lookup_entry(mono_mtable* mt, int k, const int64_t* ids, int64_t n, float* out,
                         cudaStream_t s) {
  if (n <= 0) return;
  upload_tables(mt, s);
  lookup_entry_kernel<<<grid_for(n, kThreads / 8), kThreads, 0, s>>>(mt->d_tables + k, ids, n, out);
  MONO_CHECK_LAUNCH();
}

template <int G, int OP>
static void launch_upsert_pair(const UpsertArgs& a, int64_t n_upper, cudaStream_t s) {
  constexpr bool R = OP == kOpRestore;
  resolve_hit_kernel<R><<<resident_grid(resolve_hit_kernel<R>, n_upper, kThreads), kThreads, 0, s>>>(a);
  MONO_CHECK_LAUNCH();
  resolve_miss_kernel<R><<<resident_grid(resolve_miss_kernel<R>, n_upper, kThreads), kThreads, 0, s>>>(a);
  MONO_CHECK_LAUNCH();
  upsert_apply_kernel<G, OP>
      <<<resident_grid(upsert_apply_kernel<G, OP>, n_upper, kThreads / G), kThreads, 0, s>>>(a);
  MONO_CHECK_LAUNCH();
}

template <int OP>
static void launch_upsert_g(int G, const UpsertArgs& a, int64_t n_upper, cudaStream_t s) {
  by_group(G, [&](auto g) { launch_upsert_pair<decltype(g)::value, OP>(a, n_upper, s); });
}

// the optimize pass alone, over ids whose rows are already resolved in a.rowidx
static void launch_optimize_apply(int G, const UpsertArgs& a, int64_t n_upper, cudaStream_t s) {
  by_group(G, [&](auto g) {
    constexpr int GG = decltype(g)::value;
    upsert_apply_kernel<GG, kOpOptimize>
        <<<resident_grid(upsert_apply_kernel<GG, kOpOptimize>, n_upper, kThreads / GG), kThreads, 0, s>>>(a);
  });
  MONO_CHECK_LAUNCH();
}

void note_issued(mono_mtable* mt, int k, uint64_t n, int64_t update_time, cudaStream_t s) {
  HostTable& t = mt->tables[k];
  t.issued_total += n;
  t.max_update_ts = std::max<int64_t>(t.max_update_ts, update_time);
  request_snapshot(mt, k, s);
}

static void launch_upsert(UpsertOp op, int G, const UpsertArgs& a, int64_t n_upper, cudaStream_t s) {
  switch (op) {
    case kOpOptimize: launch_upsert_g<kOpOptimize>(G, a, n_upper, s); break;
    case kOpAssign: launch_upsert_g<kOpAssign>(G, a, n_upper, s); break;
    case kOpAssignAdd: launch_upsert_g<kOpAssignAdd>(G, a, n_upper, s); break;
    case kOpReinit: launch_upsert_g<kOpReinit>(G, a, n_upper, s); break;
    case kOpRestore: launch_upsert_g<kOpRestore>(G, a, n_upper, s); break;
  }
}

// The fields every upsert launch fills alike; the caller sets idx_list, n_dev, pos0, wait_flag, filter_mode and status.
static UpsertArgs upsert_args(const mono_mtable* mt, const CallBlob& cb, int nsegs, const int64_t* ids, int64_t n,
                              const float* vals, uint32_t update_ts, uint32_t* miss_ctr, uint32_t* miss_list,
                              uint32_t* rowidx) {
  UpsertArgs a;
  a.tables = mt->d_tables;
  a.segs = cb.segs;
  a.nsegs = nsegs;
  a.ids = ids;
  a.n = n;
  a.vals = vals;
  a.lr = cb.lr;
  a.update_ts = update_ts;
  a.miss_ctr = miss_ctr;
  a.miss_list = miss_list;
  a.rowidx = rowidx;
  return a;
}

// The setup run_upsert and run_upsert_groups share: room for the call's ids in every table it touches (may rehash or
// grow, so it precedes the descriptor upload), the staged segments and learning rates, the lane-group width of the
// widest table and whether any of the tables has an admission filter.  issued() closes the call.
struct UpsertCall {
  std::vector<uint64_t> per_table;  // ids of the call per table
  CallBlob cb;
  int G;
  bool any_filter = false;

  UpsertCall(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const float* lr_host, int n_lr, cudaStream_t s)
      : per_table(mt->tables.size(), 0) {
    for (int i = 0; i < nsegs; ++i)
      per_table[h_segs[i].table] += (uint64_t)(h_segs[i].id_end - h_segs[i].id_begin);
    for (size_t k = 0; k < per_table.size(); ++k)
      if (per_table[k]) ensure_capacity(mt, (int)k, per_table[k], s);
    upload_tables(mt, s);
    cb = stage_call(mt, h_segs, nsegs, lr_host, n_lr, s);
    G = pick_group(max_dim_of(mt, h_segs, nsegs));
    for (size_t k = 0; k < per_table.size(); ++k)
      if (per_table[k] && mt->tables[k].dev.flt_cells) any_filter = true;
  }

  void issued(mono_mtable* mt, int64_t update_time, cudaStream_t s) const {
    for (size_t k = 0; k < per_table.size(); ++k)
      if (per_table[k]) note_issued(mt, (int)k, per_table[k], update_time, s);
  }
};

void run_upsert(mono_mtable* mt, UpsertOp op, const CallSeg* h_segs, int nsegs,
                const int64_t* ids_dev, int64_t n_total, const float* vals_dev,
                const float* lr_host, int n_lr, int64_t update_time, bool unique, bool dedup_sum,
                int32_t* status_dev, cudaStream_t s) {
  mt->note_insert(s);
  if (n_total <= 0 || nsegs <= 0) return;
  // The kernels walk positions [0, n): rebase the call on the id range its segments cover
  // (fused_optimize passes one shard's segments of a larger id array).
  std::vector<CallSeg> rebased(h_segs, h_segs + nsegs);
  {
    const int64_t i0 = rebased.front().id_begin;
    for (int i = 0; i < nsegs; ++i) {
      if (i > 0 && rebased[i].id_begin != h_segs[i - 1].id_end)
        throw ArgError("call segments must be contiguous");
      rebased[i].id_begin -= i0;
      rebased[i].id_end -= i0;
    }
    ids_dev += i0;
    if (status_dev) status_dev += i0;
    n_total = rebased.back().id_end;
    h_segs = rebased.data();
  }
  if (n_total >= (int64_t)1 << 31) throw ArgError("more than 2^31 ids in one call");
  const UpsertCall call(mt, h_segs, nsegs, lr_host, n_lr, s);
  const CallBlob& cb = call.cb;
  const int G = call.G;
  const bool any_filter = call.any_filter;

  // scratch: [miss_ctr (64 B) | miss_list u32[n_total] | rowidx u32[n_total]]
  char* ws = (char*)mt->ws_miss.get(64 + 2 * sizeof(uint32_t) * (size_t)n_total, s);
  uint32_t* miss_ctr = reinterpret_cast<uint32_t*>(ws);
  uint32_t* miss_list = reinterpret_cast<uint32_t*>(ws + 64);
  uint32_t* rowidx = miss_list + n_total;
  MONO_CUDA(cudaMemsetAsync(miss_ctr, 0, 64, s));

  UpsertArgs a = upsert_args(mt, cb, nsegs, ids_dev, n_total, vals_dev, (uint32_t)update_time, miss_ctr, miss_list,
                             rowidx);
  a.status = status_dev;
  a.filter_mode = !any_filter ? 0 : (op == kOpOptimize || op == kOpAssign) ? 1 : (op == kOpAssignAdd ? 2 : 0);
  uint32_t* occ_extra = nullptr;

  if (unique) {
    launch_upsert(op, G, a, n_total, s);
    launch_upsert_finalize(mt, cb, miss_ctr, (uint32_t)update_time, s);
  } else {
    // Sequential semantics for duplicates (ref: per-id loops in BatchOptimize / AssignAdd):
    // round r applies the r-th occurrence of every key; within a round keys are unique.
    if (n_total > ((int64_t)1 << 30)) throw ArgError("more than 2^30 non-unique ids in one call");
    const uint32_t cap = claim_set_slots(n_total);  // <= 2^31: n_total <= 2^30 checked above
    FirstOcc* set = (FirstOcc*)mt->ws_a.get(sizeof(FirstOcc) * (size_t)cap, s);
    uint32_t* slot_of = (uint32_t*)mt->ws_b.get(sizeof(uint32_t) * (size_t)n_total, s);
    uint32_t* lists = (uint32_t*)mt->ws_c.get(sizeof(uint32_t) * (size_t)n_total * 3 + 64, s);
    uint32_t* ctr = lists;  // [0] leaders [1] rest
    uint32_t* leaders = lists + 16;
    uint32_t* bufA = leaders + n_total;
    uint32_t* bufB = bufA + n_total;
    uint32_t* leader_of = nullptr;
    float* acc = nullptr;
    uint32_t* round0_leaders = nullptr;
    uint32_t n_round0 = 0;
    size_t val_floats = 0;
    if (dedup_sum) {
      if (op != kOpOptimize) throw ArgError("dedup_sum applies to optimize only");
      {  // the reference dedups per BatchOptimize call = per segment: one segment per table here
        std::vector<int> seen(mt->tables.size(), 0);
        for (int i = 0; i < nsegs; ++i)
          if (h_segs[i].id_end > h_segs[i].id_begin && seen[h_segs[i].table]++)
            throw ArgError("dedup_sum needs at most one segment per table per call");
      }
      for (int i = 0; i < nsegs; ++i)
        val_floats = std::max<size_t>(val_floats, (size_t)h_segs[i].val_off +
                                                     (size_t)(h_segs[i].id_end - h_segs[i].id_begin) *
                                                         mt->tables[h_segs[i].table].dim);
      leader_of = (uint32_t*)mt->ws_d.get(sizeof(uint32_t) * (size_t)n_total * 2, s);
      round0_leaders = leader_of + n_total;
      acc = (float*)mt->ws_e.get(sizeof(float) * val_floats + (any_filter ? 4 * (size_t)n_total + 256 : 0), s);
      MONO_CUDA(cudaMemcpyAsync(acc, vals_dev, sizeof(float) * val_floats, cudaMemcpyDeviceToDevice, s));
      if (any_filter) {  // the dedup path hands the filter each id's occurrence count (tf_bridge.cc:296-310)
        occ_extra = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(acc) + ((sizeof(float) * val_floats + 255) & ~(size_t)255));
        MONO_CUDA(cudaMemsetAsync(occ_extra, 0, 4 * (size_t)n_total, s));
      }
    } else if (a.filter_mode == 1) {
      uint8_t* absent0 = (uint8_t*)mt->ws_d.get((size_t)n_total, s);
      absent_at_start_kernel<<<grid_for(n_total, kThreads), kThreads, 0, s>>>(a, absent0);
      MONO_CHECK_LAUNCH();
      a.absent0 = absent0;
    }
    const uint32_t* pending = nullptr;
    int64_t n_pending = n_total;
    uint32_t* rest = bufA;
    int round = 0;
    while (n_pending > 0) {
      MONO_CUDA(cudaMemsetAsync(set, 0xFF, sizeof(FirstOcc) * (size_t)cap, s));
      MONO_CUDA(cudaMemsetAsync(ctr, 0, 64, s));
      dup_claim_kernel<<<grid_for(n_pending, kThreads), kThreads, 0, s>>>(
          cb.segs, nsegs, ids_dev, pending, n_pending, set, cap - 1, slot_of);
      MONO_CHECK_LAUNCH();
      dup_split_kernel<<<grid_for(n_pending, kThreads), kThreads, 0, s>>>(
          pending, n_pending, set, slot_of, leaders, rest, ctr,
          (dedup_sum && round == 0) ? leader_of : nullptr);
      MONO_CHECK_LAUNCH();
      MONO_CUDA(cudaMemcpyAsync(mt->h_flag, ctr, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
      MONO_CUDA(cudaStreamSynchronize(s));
      const uint32_t n_lead = mt->h_flag[0], n_rest = mt->h_flag[1];
      if (dedup_sum) {
        if (round == 0) {
          MONO_CUDA(cudaMemcpyAsync(round0_leaders, leaders, sizeof(uint32_t) * n_lead,
                                    cudaMemcpyDeviceToDevice, s));
          n_round0 = n_lead;
        } else {
          by_group(G, [&](auto g) {
            constexpr int GG = decltype(g)::value;
            dup_accumulate_kernel<GG><<<grid_for(n_lead, kThreads / GG), kThreads, 0, s>>>(
                mt->d_tables, cb.segs, nsegs, leaders, ctr, leader_of, vals_dev, acc, occ_extra);
          });
          MONO_CHECK_LAUNCH();
          // ctr is reused next round: the kernel above must finish reading it first (same stream)
        }
      } else {
        a.idx_list = leaders;
        a.n = n_lead;
        launch_upsert(op, G, a, n_lead, s);
        launch_upsert_finalize(mt, cb, miss_ctr, (uint32_t)update_time, s);
      }
      pending = rest;
      rest = (rest == bufA) ? bufB : bufA;
      n_pending = n_rest;
      ++round;
    }
    if (dedup_sum) {
      a.idx_list = round0_leaders;
      a.n = n_round0;
      a.vals = acc;
      a.occ_extra = occ_extra;
      launch_upsert(op, G, a, n_round0, s);
      launch_upsert_finalize(mt, cb, miss_ctr, (uint32_t)update_time, s);
    }
  }
  call.issued(mt, update_time, s);
}


// Optimize over several groups of segments (the shards of a fused call) where the ids are unique inside
// a group but a FID may appear once per group: group g is applied after group g-1 (the reference's
// shard-by-shard order, multi_hash_table_update_op.cc:286-300).  One resolve pass serves all groups and
// nothing returns to the host; only the apply pass runs once per group.
void run_upsert_groups(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const int64_t* group_begin,
                       int ngroups, const int64_t* ids_dev, const float* vals_dev, const float* lr_host,
                       int n_lr, int64_t update_time, cudaStream_t s) {
  mt->note_insert(s);
  if (nsegs <= 0 || ngroups <= 0) return;
  const int64_t n_total = h_segs[nsegs - 1].id_end;
  if (n_total <= 0) return;
  if (h_segs[0].id_begin != 0) throw ArgError("grouped optimize: segments must start at id 0");
  for (int i = 1; i < nsegs; ++i)
    if (h_segs[i].id_begin != h_segs[i - 1].id_end) throw ArgError("call segments must be contiguous");
  if (n_total >= (int64_t)1 << 31) throw ArgError("more than 2^31 ids in one call");
  const UpsertCall call(mt, h_segs, nsegs, lr_host, n_lr, s);
  const CallBlob& cb = call.cb;

  if (n_total > ((int64_t)1 << 30)) throw ArgError("more than 2^30 ids in one grouped optimize call");
  const uint32_t cap = claim_set_slots(n_total);
  // scratch: [ctr 64 B | miss_list | rowidx | leaders | followers | fol_leader | slot_of] u32[n_total] each
  char* ws = (char*)mt->ws_miss.get(64 + 6 * sizeof(uint32_t) * (size_t)n_total, s);
  uint32_t* ctr = reinterpret_cast<uint32_t*>(ws);  // [0] misses [1] leaders [2] followers
  uint32_t* miss_list = reinterpret_cast<uint32_t*>(ws + 64);
  uint32_t* rowidx = miss_list + n_total;
  uint32_t* leaders = rowidx + n_total;
  uint32_t* followers = leaders + n_total;
  uint32_t* fol_leader = followers + n_total;
  uint32_t* slot_of = fol_leader + n_total;
  FirstOcc* set = (FirstOcc*)mt->ws_a.get(sizeof(FirstOcc) * (size_t)cap, s);
  MONO_CUDA(cudaMemsetAsync(ctr, 0, 64, s));
  MONO_CUDA(cudaMemsetAsync(set, 0xFF, sizeof(FirstOcc) * (size_t)cap, s));

  UpsertArgs a = upsert_args(mt, cb, nsegs, ids_dev, n_total, vals_dev, (uint32_t)update_time, ctr, miss_list, rowidx);
  a.filter_mode = call.any_filter ? 1 : 0;
  resolve_hit_kernel<false><<<resident_grid(resolve_hit_kernel<false>, n_total, kThreads), kThreads, 0, s>>>(a);
  MONO_CHECK_LAUNCH();
  // misses are few in steady state: small grids, counts stay on the device
  const int gm = (int)std::min<int64_t>(device_sms() * 2, (n_total + kThreads - 1) / kThreads);
  dup_claim_kernel<<<gm, kThreads, 0, s>>>(cb.segs, nsegs, ids_dev, miss_list, 0, set, cap - 1, slot_of, ctr);
  MONO_CHECK_LAUNCH();
  miss_split_kernel<<<gm, kThreads, 0, s>>>(miss_list, ctr, set, slot_of, leaders, followers, fol_leader, ctr);
  MONO_CHECK_LAUNCH();
  UpsertArgs am = a;
  am.miss_list = leaders;
  am.miss_ctr = ctr + 1;
  resolve_miss_kernel<false><<<gm, kThreads, 0, s>>>(am);
  MONO_CHECK_LAUNCH();
  miss_follow_kernel<<<gm, kThreads, 0, s>>>(followers, fol_leader, ctr + 2, rowidx);
  MONO_CHECK_LAUNCH();
  launch_upsert_finalize(mt, cb, ctr, (uint32_t)update_time, s);
  for (int g = 0; g < ngroups; ++g) {
    const int64_t b = group_begin[g], e = group_begin[g + 1];
    if (e <= b) continue;
    UpsertArgs ag = a;
    ag.pos0 = b;
    ag.n = e - b;
    ag.rowidx = rowidx + b;
    launch_optimize_apply(call.G, ag, ag.n, s);
  }
  call.issued(mt, update_time, s);
}

// Apply pass over one requester's segment of the owner-side window (device-driven sharded step): items are
// positions pos0 .. pos0 + *n_dev of ids_base / grads_base (rows of dim floats), rows already resolved in rowidx.
void launch_apply_window(mono_mtable* mt, int k, const CallBlob& cb, const int64_t* ids_base, const float* grads_base,
                         int64_t pos0, const uint32_t* n_dev, int64_t n_upper, uint32_t* rowidx, uint32_t update_ts,
                         const uint64_t* wait_flag, uint64_t wait_seq, cudaStream_t s) {
  mt->note_insert(s);
  UpsertArgs a = upsert_args(mt, cb, 1, ids_base, n_upper, grads_base, update_ts, nullptr, nullptr, rowidx + pos0);
  a.n_dev = n_dev;
  a.pos0 = pos0;
  a.wait_flag = wait_flag;
  a.wait_seq = wait_seq;
  launch_optimize_apply(pick_group(mt->tables[k].dim), a, n_upper, s);
}

void launch_upsert_finalize(mono_mtable* mt, const CallBlob& cb, uint32_t* miss_ctr, uint32_t update_ts, cudaStream_t s) {
  upsert_finalize_kernel<<<(cb.ntab + 63) / 64, 64, 0, s>>>(mt->d_tables, cb.table_ids, cb.ntab, miss_ctr, update_ts);
  MONO_CHECK_LAUNCH();
}

}  // namespace mono
