// xstep.cu — the device-driven sharded sparse step: FID-hash sharded table across the GPUs of one NVSwitch box with
// NOTHING returning to the host inside a step (replaces the reference's distributed_ps / distributed_ps_sync
// orchestration — ref: NT/distributed_ps.py:1501-2001, NT/distributed_ps_sync.py:95-512 — and round 1's
// host-driven ShardedStep, whose per-step count exchange through the host and three all-rank barriers cost more than
// its kernels at 8 GPUs).
//
// Every rank owns a window (peer.cu) with FIXED regions sized for the worst case, one sub-region per SOURCE rank:
//     ids_in  [2 (step parity)] [N sources] [C]      int64   FID buckets sent to this owner
//     rows_in [C] [D]                                float   rows of this rank's own bucketed unique list
//     grads_in[N sources] [C] [D]                    float   summed gradient rows sent to this owner
// so a sender never needs to know what the other senders send: all offsets are local knowledge.  A requester tells
// each owner two numbers with its FIDs — how many, and where the owner shall put the rows (the bucket's offset in
// the requester's rows_in) — in a header word next to the arrival flag.  Synchronisation is DIRECTIONAL: a
// producer raises a per-(phase, source) flag in the consumer's flag page when its data has landed
// (st.release.sys after the producing kernels); a consumer waits only for the data it is about to read
// (ld.acquire.sys), source by source where the work is separable (owner lookup, owner apply).  No all-rank barrier,
// no host round trip, no collective launch: the host enqueues a whole step — or several — without ever
// synchronising, and the device-side counts size every loop.
//
//   requester                                        owner
//   grouping_build (claim, sort, runs; counts stay on the device)
//   xput_ids: bucket o -> o.ids_in[par][me]  + header, flag IDS[me] ------>
//                                                    xlookup_push: for every source r (whichever has arrived):
//                                                      probe + gather, row i of r's bucket stored into
//   <----------------------------------------------  r.rows_in[dst_off_r + i]; then flag ROWS[me] at every r
//   wait ROWS[*]; gather_pool(rows_in) -> pooled rows
//   ... dense tower ...
//   reduce (seg_reduce STORE): summed row of unique u -> owner.grads_in[me][u - bucket start]; flag GRADS[me] ---->
//                                                    xowner_resolve (all received FIDs: probe / insert, ts bump;
//                                                      may run before the gradients arrive)
//                                                    apply source 0, 1, ... in rank order (the reference's order),
//                                                      each launch waiting for GRADS[r] only
// Reuse of the regions without barriers (why a flag per phase suffices): a rank issues step e+1's traffic to owner o
// only after its own step e finished, which needed o's rows of step e, which o produced after ITS step e-1; ids_in is
// double-buffered by step parity because an owner still applies step e from ids_in while a fast requester already
// pushes step e+1's FIDs (derivation as in round 1's distributed_ps.py).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "rowops.cuh"

namespace mono {

constexpr int kPhaseIds = 0, kPhaseRows = 1, kPhaseGrads = 2;
constexpr int kFlagSlot0 = 16;    // flag page: [0,16) barrier flags; 16 + 16 * phase + source: directional flags
constexpr int kHdrSlot0 = 80;     // 80 + source: header word of the IDS phase = count << 32 | row offset

__device__ __forceinline__ void st_release_sys_u64(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys_u64(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t now_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// spin until the flag reaches seq; a peer that never arrives trips the timeout (loud failure, no hang)
__device__ __forceinline__ void wait_flag(const uint64_t* f, uint64_t seq, uint64_t timeout_ns, int what, int src) {
  const uint64_t t0 = now_ns();
  while (ld_acquire_sys_u64(f) < seq) {
    if (timeout_ns != 0 && now_ns() - t0 > timeout_ns) {
      printf("mono xstep: timed out waiting for phase %d of rank %d (seq %llu)\n", what, src, (unsigned long long)seq);
      __trap();
    }
  }
}

// 1 requester: FID bucket o of the bucketed unique list -> owner o's ids_in[par][me]
__global__ void __launch_bounds__(kThreads)
xput_ids_kernel(const int64_t* __restrict__ uniq, const uint32_t* __restrict__ owner_cnt, XWin w, int par) {
  __shared__ int64_t s_start[kMaxPeers + 1];
  if (threadIdx.x == 0) {
    int64_t run = 0;
    for (int r = 0; r <= kMaxPeers; ++r) {
      s_start[r] = run;
      if (r < w.N) run += owner_cnt[r];
    }
  }
  __syncthreads();
  const int64_t total = s_start[w.N];
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int o = peer_part(s_start, w.N, i);
    w.ids_in(o, par, w.me)[i - s_start[o]] = uniq[i];
  }
}

// one warp: lane r tells rank r that this rank's data of `phase` has landed (everything the earlier kernels of the
// stream stored).  IDS phase: the header word (count, row offset of the bucket) goes first.
__global__ void __launch_bounds__(32)
xsignal_kernel(XWin w, int phase, uint64_t seq, const uint32_t* __restrict__ owner_cnt /* IDS phase only */) {
  const int r = threadIdx.x;
  uint32_t cnt = 0;
  if (owner_cnt && r < w.N) cnt = owner_cnt[r];
  uint32_t incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
    if (r >= o) incl += y;
  }
  if (r >= w.N) return;
  __threadfence_system();
  uint64_t* f = w.flags(r);
  if (owner_cnt) f[kHdrSlot0 + w.me] = ((uint64_t)cnt << 32) | (uint64_t)(incl - cnt);
  __threadfence_system();
  st_release_sys_u64(f + kFlagSlot0 + 16 * phase + w.me, seq);
}

// one warp: wait until every rank's flag of `phase` has reached seq
__global__ void __launch_bounds__(32) xwait_kernel(XWin w, int phase, uint64_t seq, uint64_t timeout_ns) {
  const int r = threadIdx.x;
  if (r >= w.N) return;
  wait_flag(w.flags(w.me) + kFlagSlot0 + 16 * phase + r, seq, timeout_ns, phase, r);
}

// 2 owner: lookup fused with the row exchange, source by source as the FID buckets arrive.  Every block visits all
// sources (starting at a block-dependent one, taking whichever has arrived first) and grid-strides over the
// source's warp tiles; rows go straight into the requester's rows_in (one 128-bit NVLink store per lane).
template <int G, bool CONFIRM>
__global__ void __launch_bounds__(kThreads, 6)
xlookup_push_kernel(const TableDev* __restrict__ t0, XWin w, int par, uint64_t seq, uint64_t timeout_ns) {
  constexpr int RPI = 32 / G;
  constexpr int ITERS = G;
  constexpr int UNR = 4;
  __shared__ uint32_t s_src;
  __shared__ uint64_t s_hdr;
  const int lane = threadIdx.x & 31, gl = Group<G>::gl(), grp = lane / G;
  const int c = gl * 4;
  const int D0 = t0->dim;
  const float* __restrict__ emb0 = t0->emb;
  const uint32_t stride0 = t0->emb_stride;
  const uint64_t* myf = w.flags(w.me);
  uint32_t done = 0;  // block-uniform: sources already served
  for (int served = 0; served < w.N; ++served) {
    if (threadIdx.x == 0) {  // pick a source whose FIDs have arrived (block-dependent start: spread the waiting)
      const uint64_t t_begin = now_ns();
      int pick = -1;
      while (pick < 0) {
        for (int q = 0; q < w.N; ++q) {
          const int r = (int)((blockIdx.x + w.me + q) % (unsigned)w.N);
          if (!((done >> r) & 1u) && ld_acquire_sys_u64(myf + kFlagSlot0 + 16 * kPhaseIds + r) >= seq) {
            pick = r;
            break;
          }
        }
        if (pick < 0 && timeout_ns != 0 && now_ns() - t_begin > timeout_ns) {
          printf("mono xstep: rank %d timed out waiting for FID buckets (seq %llu)\n", w.me, (unsigned long long)seq);
          __trap();
        }
      }
      s_src = (uint32_t)pick;
      s_hdr = myf[kHdrSlot0 + pick];
    }
    __syncthreads();
    const int src = (int)s_src;
    const int64_t n_src = (int64_t)(s_hdr >> 32);
    const int64_t dst_off = (int64_t)(s_hdr & 0xFFFFFFFFull);
    __syncthreads();
    done |= 1u << src;
    const int64_t* __restrict__ ids = w.ids_in(w.me, par, src);
    float* __restrict__ dst_rows = w.rows_in(src) + dst_off * D0;
    const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * 32;
    const int64_t wfirst = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * 32;
    int64_t key_next = wfirst + lane < n_src ? ids[wfirst + lane] : 0;  // next tile's FIDs one iteration ahead
    for (int64_t wbase = wfirst; wbase < n_src; wbase += wstride) {
      const int64_t i = wbase + lane;
      const int64_t key = key_next;
      if (i + wstride < n_src) key_next = ids[i + wstride];
      uint32_t row = kEmptyRow;
      if (i < n_src) {
        row = probe_lane(t0, key);
        if (CONFIRM && row == kEmptyRow) row = probe_lane_confirm_miss(t0, key);  // inserts on another stream (rowops.cuh)
      }
#pragma unroll
      for (int it0 = 0; it0 < ITERS; it0 += UNR) {
        float4 x[UNR];
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          const uint32_t r = __shfl_sync(0xffffffffu, row, (it0 + u) * RPI + grp);
          x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (r != kEmptyRow && c < D0) x[u] = __ldg(reinterpret_cast<const float4*>(emb0 + (size_t)r * stride0 + c));
        }
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          const int src_lane = (it0 + u) * RPI + grp;
          const int64_t ir = wbase + src_lane;
          const uint32_t r_st = __shfl_sync(0xffffffffu, row, src_lane);
          if (ir >= n_src) continue;
          float* dst = dst_rows + ir * D0;
          if (c < D0) *reinterpret_cast<float4*>(dst + c) = x[u];
          for (int cc = c + 4 * G; cc < D0; cc += 4 * G) {  // wide rows (dim > 128)
            float4 y = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r_st != kEmptyRow) y = __ldg(reinterpret_cast<const float4*>(emb0 + (size_t)r_st * stride0 + cc));
            *reinterpret_cast<float4*>(dst + cc) = y;
          }
        }
      }
    }
  }
}

// 7a owner: resolve every received FID (all sources; needs only the FIDs, not the gradients): hit -> row index +
// expiry-timestamp bump; miss -> queued.  Position of item i of source r = r * C + i.
__global__ void __launch_bounds__(kThreads)
xowner_resolve_kernel(const TableDev* __restrict__ t, XWin w, int par, uint32_t update_ts, uint32_t* __restrict__ rowidx,
                      uint32_t* __restrict__ miss_ctr, uint32_t* __restrict__ miss_list) {
  const int lane = threadIdx.x & 31;
  const uint64_t* myf = w.flags(w.me);
  for (int src = 0; src < w.N; ++src) {
    const int64_t n_src = (int64_t)(myf[kHdrSlot0 + src] >> 32);
    const int64_t* __restrict__ ids = w.ids_in(w.me, par, src);
    const int64_t wstride = (int64_t)gridDim.x * (kThreads / 32) * 32;
    for (int64_t wbase = ((int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)) * 32; wbase < n_src; wbase += wstride) {
      const int64_t i = wbase + lane;
      bool miss = false;
      if (i < n_src) {
        Entry* slot = nullptr;
        const uint32_t row = probe_lane_slot(t, ids[i], &slot);
        if (row == kEmptyRow) {
          miss = true;
        } else {
          slot->ts = update_ts;
          rowidx[src * w.C + i] = row;
        }
      }
      const uint32_t mbal = __ballot_sync(0xffffffffu, miss);
      if (mbal) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(miss_ctr, (uint32_t)__popc(mbal));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (miss) miss_list[base + __popc(mbal & ((1u << lane) - 1u))] = (uint32_t)(src * w.C + i);
      }
    }
  }
}

// 7b absent FIDs: the same new FID may come from several sources.  Every miss claims the scratch-set slot of its FID
// (epoch-versioned set, never cleared) and the LOWEST position per slot is recorded with one 64-bit atomicMax
// (epoch << 32 | ~position: a newer epoch always wins, inside an epoch the lowest position does).
__global__ void __launch_bounds__(kThreads)
xmiss_claim_kernel(XWin w, int par, const uint32_t* __restrict__ miss_ctr, const uint32_t* __restrict__ miss_list, Entry* set,
                   uint32_t cap, uint32_t epoch, unsigned long long* __restrict__ first, uint32_t* __restrict__ slot_of) {
  const int64_t n = (int64_t)*miss_ctr;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t pos = miss_list[q];
    const int src = (int)(pos / (uint64_t)w.C);
    const int64_t key = w.ids_in(w.me, par, src)[pos - (uint64_t)src * w.C];
    uint32_t idx = __umulhi((uint32_t)(mix64((uint64_t)key) >> 24), cap);
    while (true) {
      Entry* p = set + idx;
      Entry e = ld_entry_cg(p);
      while (e.ts != epoch) {
        Entry ne;
        ne.key = key;
        ne.row = kEmptyRow;
        ne.ts = epoch;
        const Entry old = cas_entry_old(p, e, ne);
        if (old.key == e.key && old.row == e.row && old.ts == e.ts) e = ne; else e = old;
      }
      if (e.key == key) break;
      idx = idx + 1 == cap ? 0 : idx + 1;
    }
    slot_of[q] = idx;
    atomicMax(first + idx, ((unsigned long long)epoch << 32) | (unsigned long long)(~pos));
  }
}

// leaders (lowest position of a new FID = the first requester in rank order) insert: admission filter, row from the
// free list / bump allocator, lock-free cuckoo insert; the row is parked in the set entry for the followers
__global__ void __launch_bounds__(kThreads)
xmiss_insert_kernel(const TableDev* __restrict__ t, XWin w, int par, const uint32_t* __restrict__ miss_ctr,
                    const uint32_t* __restrict__ miss_list, Entry* set, const unsigned long long* __restrict__ first,
                    const uint32_t* __restrict__ slot_of, uint32_t update_ts, uint32_t* __restrict__ rowidx) {
  const int64_t n = (int64_t)*miss_ctr;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t pos = miss_list[q];
    const uint32_t sl = slot_of[q];
    if ((uint32_t)(~first[sl]) != pos) continue;  // a follower
    const int src = (int)(pos / (uint64_t)w.C);
    const int64_t key = w.ids_in(w.me, par, src)[pos - (uint64_t)src * w.C];
    uint32_t row = kEmptyRow;
    if (!should_be_filtered(t, key, 1u)) {
      const uint32_t ticket = atomicAdd(t->ctrs + kCtrMiss, 1u);
      const uint32_t fc = t->ctrs[kCtrFree];
      row = ticket < fc ? t->free_list[fc - 1 - ticket] : t->ctrs[kCtrBump] + (ticket - fc);
      if (row >= t->row_cap) {
        atomicOr(t->ctrs + kCtrError, 2u);
        row = kEmptyRow;
      } else {
        Entry e;
        e.key = key;
        e.row = row;
        e.ts = update_ts;
        cuckoo_insert(t, e);
      }
    }
    set[sl].row = row;
    rowidx[pos] = row == kEmptyRow ? row : (row | kFreshBit);
  }
}

__global__ void __launch_bounds__(kThreads)
xmiss_follow_kernel(const uint32_t* __restrict__ miss_ctr, const uint32_t* __restrict__ miss_list, const Entry* __restrict__ set,
                    const unsigned long long* __restrict__ first, const uint32_t* __restrict__ slot_of,
                    uint32_t* __restrict__ rowidx) {
  const int64_t n = (int64_t)*miss_ctr;
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < n; q += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t pos = miss_list[q];
    const uint32_t sl = slot_of[q];
    if ((uint32_t)(~first[sl]) == pos) continue;  // the leader
    rowidx[pos] = set[sl].row;                     // not fresh: the leader's requester initialises the row
  }
}

}  // namespace mono

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
namespace mono {

static int64_t al256(int64_t x) { return (x + 255) & ~(int64_t)255; }

int64_t xstep_window_bytes(int N, int64_t C, int D) {
  return 2 * al256((int64_t)N * C * 8) + al256(C * D * 4) + al256((int64_t)N * C * D * 4);
}

mono_xstep* xstep_create(mono_mtable* mt, int k, mono_peer* win, int64_t cap_pair) {
  if (!win->attached) throw ArgError("xstep: the peer window is not attached");
  if (win->device != mt->device) throw ArgError("xstep: window and table on different devices");
  const int D = mt->tables[k].dim;
  if ((D & 3) || D > 128) throw ArgError("xstep needs dim % 4 == 0 and dim <= 128");
  if (cap_pair <= 0 || cap_pair >= ((int64_t)1 << 29)) throw ArgError("xstep: bad capacity");
  if ((uint64_t)cap_pair * (uint64_t)win->world >= ((uint64_t)1 << 31)) throw ArgError("xstep: capacity x ranks exceeds 2^31");
  if ((size_t)xstep_window_bytes(win->world, cap_pair, D) > win->bytes) throw ArgError("xstep: the window is too small");
  auto x = new mono_xstep();
  x->mt = mt;
  x->k = k;
  x->win = win;
  x->C = cap_pair;
  x->N = win->world;
  x->me = win->rank;
  x->D = D;
  for (int q = 0; q < 2; ++q) {
    x->grouping[q] = grouping_create(mt->device);
    MONO_CUDA(cudaEventCreateWithFlags(&x->ev_prep[q], cudaEventDisableTiming));
    MONO_CUDA(cudaEventCreateWithFlags(&x->ev_bwd[q], cudaEventDisableTiming));
  }
  XWin& w = x->w;
  std::memset(&w, 0, sizeof(w));
  for (int r = 0; r < x->N; ++r) w.base[r] = win->base[r];
  w.N = x->N;
  w.me = x->me;
  w.D = D;
  w.C = cap_pair;
  w.off_ids[0] = 0;
  w.off_ids[1] = al256((int64_t)x->N * cap_pair * 8);
  w.off_rows = 2 * al256((int64_t)x->N * cap_pair * 8);
  w.off_grads = w.off_rows + al256(cap_pair * D * 4);
  const char* e = std::getenv("MONO_PEER_TIMEOUT_S");
  const double sec = e ? std::atof(e) : 600.0;
  x->timeout_ns = sec <= 0 ? 0ull : (uint64_t)(sec * 1e9);
  return x;
}

void xstep_destroy(mono_xstep* x) {
  if (!x) return;
  cudaSetDevice(x->mt->device);
  cudaDeviceSynchronize();
  x->ws.release();
  x->miss_set.release();
  for (int q = 0; q < 2; ++q) {
    x->uniq[q].release();
    x->offs[q].release();
    if (x->ev_prep[q]) cudaEventDestroy(x->ev_prep[q]);
    if (x->ev_bwd[q]) cudaEventDestroy(x->ev_bwd[q]);
    grouping_destroy(x->grouping[q]);
  }
  delete x;
}

// forward of one step: group, send FID buckets, serve the other ranks' buckets, pool.  Nothing returns to the host.
void xstep_forward(mono_xstep* x, const int64_t* fids_dev, int64_t M, const int32_t* row_offsets, int64_t n_rows,
                   int pooling, float* out, int64_t out_stride, int out_col, cudaStream_t s) {
  MONO_CUDA(cudaSetDevice(x->mt->device));
  if (M <= 0 || M > x->C) throw ArgError("xstep: batch larger than the window capacity (or empty)");
  mono_mtable* mt = x->mt;
  upload_tables(mt, s);
  const XWin& w = x->w;
  const uint64_t seq = ++x->step;
  const int par = (int)(seq & 1);
  mono_grouping* g = x->grouping[par];
  int64_t* uniq;
  int32_t* offs;
  if (x->prep_seq == seq && x->prep_fids == fids_dev && x->prep_m == M) {
    // the grouping of this batch was built ahead of time on another stream (xstep_prepare): just order after it
    MONO_CUDA(cudaStreamWaitEvent(s, x->ev_prep[par], 0));
    uniq = (int64_t*)x->uniq[par].p;
    offs = (int32_t*)x->offs[par].p;
  } else {
    uniq = (int64_t*)x->uniq[par].get(8 * (size_t)M, s);
    offs = (int32_t*)x->offs[par].get(4 * (size_t)M, s);
    grouping_build(g, fids_dev, M, x->N, x->D, uniq, offs, nullptr, nullptr, s);
  }
  x->prep_seq = 0;
  const uint32_t* owner_cnt = g->plan.ctr + kCtrOwners;
  xput_ids_kernel<<<resident_grid(xput_ids_kernel, M, kThreads), kThreads, 0, s>>>(uniq, owner_cnt, w, par);
  MONO_CHECK_LAUNCH();
  xsignal_kernel<<<1, 32, 0, s>>>(w, kPhaseIds, seq, owner_cnt);
  MONO_CHECK_LAUNCH();
  const TableDev* t = mt->d_tables + x->k;
  // the grid is sized for the capacity bound; the kernel loops over what actually arrived
  const bool confirm = mt->lookup_must_confirm(s);  // inserts may be running on another stream
#define XLP(GG)                                                                                                        \
  if (confirm)                                                                                                         \
    xlookup_push_kernel<GG, true><<<resident_grid(xlookup_push_kernel<GG, true>, M, kThreads), kThreads, 0, s>>>(     \
        t, w, par, seq, x->timeout_ns);                                                                                \
  else                                                                                                                 \
    xlookup_push_kernel<GG, false><<<resident_grid(xlookup_push_kernel<GG, false>, M, kThreads), kThreads, 0, s>>>(   \
        t, w, par, seq, x->timeout_ns)
  switch (pick_group(x->D)) {
    case 4: XLP(4); break;
    case 8: XLP(8); break;
    case 16: XLP(16); break;
    default: XLP(32); break;
  }
#undef XLP
  MONO_CHECK_LAUNCH();
  xsignal_kernel<<<1, 32, 0, s>>>(w, kPhaseRows, seq, nullptr);
  MONO_CHECK_LAUNCH();
  xwait_kernel<<<1, 32, 0, s>>>(w, kPhaseRows, seq, x->timeout_ns);
  MONO_CHECK_LAUNCH();
  const float* rows_in = reinterpret_cast<const float*>(x->win->local + kPeerFlagBytes + w.off_rows);
  launch_gather_pool(rows_in, offs, row_offsets, row_offsets ? n_rows : M, x->D, pooling, out, out_stride, out_col, s);
  x->last_m = M;
  x->last_rows = row_offsets ? n_rows : M;
  x->fwd_done = true;
}

// backward of the step started by the last forward: per-FID gradient sums pushed to the owners, then this rank, as
// an owner, resolves what it received and applies the sources in rank order.
void xstep_backward(mono_xstep* x, const float* pooled_grad, int64_t grad_stride, int grad_col,
                    const int32_t* row_offsets, int pooling, const float* lr_host, int64_t update_time, cudaStream_t s) {
  MONO_CUDA(cudaSetDevice(x->mt->device));
  if (!x->fwd_done) throw ArgError("xstep_backward without a forward");
  x->fwd_done = false;
  mono_mtable* mt = x->mt;
  mt->note_insert(s);
  HostTable& ht = mt->tables[x->k];
  const XWin& w = x->w;
  const uint64_t seq = x->step;
  const int par = (int)(seq & 1);
  // requester: reduce + push
  PeerOut po;
  std::memset(&po, 0, sizeof(po));
  po.n = x->N;
  for (int r = 0; r < x->N; ++r)
    po.base[r] = x->win->base[r] + kPeerFlagBytes + w.off_grads + (int64_t)x->me * x->C * x->D * 4;
  mono_grouping* g = x->grouping[par];
  po.cnt_dev = g->plan.ctr + kCtrOwners;
  grouping_reduce_push(g, pooled_grad, grad_stride, grad_col, row_offsets, x->last_rows, pooling, po, s);
  xsignal_kernel<<<1, 32, 0, s>>>(w, kPhaseGrads, seq, nullptr);
  MONO_CHECK_LAUNCH();
  // owner: resolve (+ insert) everything received, then apply source by source
  const int64_t cap_total = (int64_t)x->N * x->C;
  // rows the received FIDs may need: with hash-balanced owners a rank receives about its own distinct count; twice
  // the batch is a generous bound.  (A pathological batch that exceeds it trips the table's row-slab overflow flag:
  // the next call fails loudly, nothing is silently dropped without notice.)
  ensure_capacity(mt, x->k, (uint64_t)std::min<int64_t>(cap_total, 2 * x->last_m), s);
  upload_tables(mt, s);
  CallSeg sg;
  sg.id_begin = 0;
  sg.id_end = cap_total;
  sg.val_off = 0;
  sg.table = x->k;
  sg.lr_off = 0;
  CallBlob cb = stage_call(mt, &sg, 1, lr_host, ht.slices, s);
  const uint32_t cap = claim_set_slots(cap_total);
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_ctr = take(256), o_ridx = take(4 * (size_t)cap_total), o_miss = take(4 * (size_t)cap_total);
  const size_t o_slot = take(4 * (size_t)cap_total);
  char* ws = (char*)x->ws.get(off, s);
  uint32_t* ctr = (uint32_t*)(ws + o_ctr);
  uint32_t* rowidx = (uint32_t*)(ws + o_ridx);
  uint32_t* miss_list = (uint32_t*)(ws + o_miss);
  uint32_t* slot_of = (uint32_t*)(ws + o_slot);
  MONO_CUDA(cudaMemsetAsync(ctr, 0, 256, s));
  // set entries (16 B) followed by the per-slot "lowest position" words (8 B)
  uint32_t epoch = 0;
  char* setmem = (char*)x->miss_set.get((sizeof(Entry) + 8) * (size_t)cap, s, &epoch);
  Entry* set = (Entry*)setmem;
  unsigned long long* first = (unsigned long long*)(setmem + sizeof(Entry) * (size_t)cap);
  const TableDev* t = mt->d_tables + x->k;
  const int64_t work = (int64_t)x->N * x->last_m;
  xowner_resolve_kernel<<<resident_grid(xowner_resolve_kernel, work, kThreads), kThreads, 0, s>>>(
      t, w, par, (uint32_t)update_time, rowidx, ctr, miss_list);
  MONO_CHECK_LAUNCH();
  const int gm = (int)std::min<int64_t>(device_sms() * 2, (work + kThreads - 1) / kThreads);  // misses are few in steady state
  xmiss_claim_kernel<<<gm, kThreads, 0, s>>>(w, par, ctr, miss_list, set, cap, epoch, first, slot_of);
  MONO_CHECK_LAUNCH();
  xmiss_insert_kernel<<<gm, kThreads, 0, s>>>(t, w, par, ctr, miss_list, set, first, slot_of, (uint32_t)update_time, rowidx);
  MONO_CHECK_LAUNCH();
  xmiss_follow_kernel<<<gm, kThreads, 0, s>>>(ctr, miss_list, set, first, slot_of, rowidx);
  MONO_CHECK_LAUNCH();
  launch_upsert_finalize(mt, cb, ctr, (uint32_t)update_time, s);
  const int64_t* ids_base = reinterpret_cast<const int64_t*>(x->win->local + kPeerFlagBytes + w.off_ids[par]);
  const float* grads_base = reinterpret_cast<const float*>(x->win->local + kPeerFlagBytes + w.off_grads);
  const uint64_t* myf = reinterpret_cast<const uint64_t*>(x->win->local);
  for (int src = 0; src < x->N; ++src) {
    // count of source src = high half of its header word (little endian)
    const uint32_t* n_dev = reinterpret_cast<const uint32_t*>(myf + kHdrSlot0 + src) + 1;
    launch_apply_window(mt, x->k, cb, ids_base, grads_base, (int64_t)src * x->C, n_dev, x->last_m, rowidx,
                        (uint32_t)update_time, myf + kFlagSlot0 + 16 * kPhaseGrads + src, seq, s);
  }
  ht.issued_total += (uint64_t)x->last_m;
  ht.max_update_ts = std::max<int64_t>(ht.max_update_ts, update_time);
  request_snapshot(mt, x->k, s);
  MONO_CUDA(cudaEventRecord(x->ev_bwd[par], s));  // grouping [par] is free again once this point is reached
  x->bwd_recorded[par] = true;
}

// Build the grouping of the NEXT batch on stream s2 while the current step runs on its own stream: the grouping
// (claim, sort, run list, bucketed unique list) depends on the batch only, not on the table, so it may overlap the
// NVLink-bound and flag-waiting phases of the step in flight (the reference pipelines the same way: the next batch's
// id shuffling runs under the current batch's dense compute, NT/distributed_ps_sync.py:199-204,270-275).  The next
// mono_xstep_forward must be called with the same fids pointer and count to use it.
void xstep_prepare(mono_xstep* x, const int64_t* fids_next_dev, int64_t M, cudaStream_t s2) {
  MONO_CUDA(cudaSetDevice(x->mt->device));
  if (M <= 0 || M > x->C) throw ArgError("xstep_prepare: batch larger than the window capacity (or empty)");
  const uint64_t seq = x->step + 1;
  const int par = (int)(seq & 1);
  if (x->bwd_recorded[par]) MONO_CUDA(cudaStreamWaitEvent(s2, x->ev_bwd[par], 0));  // last user of grouping [par]
  int64_t* uniq = (int64_t*)x->uniq[par].get(8 * (size_t)M, s2);
  int32_t* offs = (int32_t*)x->offs[par].get(4 * (size_t)M, s2);
  grouping_build(x->grouping[par], fids_next_dev, M, x->N, x->D, uniq, offs, nullptr, nullptr, s2);
  MONO_CUDA(cudaEventRecord(x->ev_prep[par], s2));
  x->prep_seq = seq;
  x->prep_fids = fids_next_dev;
  x->prep_m = M;
}

}  // namespace mono
