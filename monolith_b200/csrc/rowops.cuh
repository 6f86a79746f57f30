// rowops.cuh — device code shared by ops.cu (lookup / upsert family) and bwd.cu (fused backward): the sparse
// optimizer steps restated op by op, apply_row, and the lane-per-key probes.
#pragma once

#include <cuda_bf16.h>

#include "engine.h"
#include "rowelem.cuh"

namespace mono {

// ------------------------------------------------------------------------------------------
// optimizer math (bit-exact with oracle/oracle.cc; every step is an explicit IEEE op so that
// nvcc never contracts a*b+c on its own)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ int state_floats_dev(const SegDev& s) {
  switch (s.opt_type) {
    case MONO_OPT_ADAGRAD: return s.dim;
    case MONO_OPT_FTRL: return 2 * s.dim;
    case MONO_OPT_ADAM: return 2 * s.dim + 2;
    case MONO_OPT_MOMENTUM: case MONO_OPT_RMSPROP: case MONO_OPT_RMSPROPV2: return s.dim;
    case MONO_OPT_ADADELTA: return 2 * s.dim;
    case MONO_OPT_AMSGRAD: return 3 * s.dim + 2;
    case MONO_OPT_GROUP_ADAGRAD: return 1;
    default: return 0;
  }
}

__device__ __forceinline__ float init_emb_value(const TableDev* t, const SegDev& s, int64_t key,
                                                int col) {
  switch (s.init_type) {
    case MONO_INIT_ONES: return 1.0f;
    case MONO_INIT_CONSTANT: return s.init_a;
    case MONO_INIT_UNIFORM: return uniform_init(t->seed, key, col, s.init_a, s.init_b);
    default: return 0.0f;
  }
}

// initial value of state float `lj` (local index inside the segment's state block)
// ref: adagrad_optimizer.cc:47-52, ftrl_optimizer.cc:45-52, adam_optimizer.cc:44-55
__device__ __forceinline__ float init_state_value(const SegDev& s, int lj) {
  switch (s.opt_type) {
    case MONO_OPT_ADAGRAD: return s.p[0];
    case MONO_OPT_FTRL: return lj < s.dim ? s.p[0] : 0.0f;
    case MONO_OPT_ADAM: return lj < 2 * s.dim ? 0.0f : (lj == 2 * s.dim ? s.p[0] : s.p[1]);
    case MONO_OPT_AMSGRAD: return lj < 3 * s.dim ? 0.0f : (lj == 3 * s.dim ? s.p[0] : s.p[1]);  // amsgrad_optimizer.cc:44-56
    case MONO_OPT_GROUP_ADAGRAD: return s.p[0];  // group_adagrad_optimizer.cc:45-48
    default: return 0.0f;  // momentum / rmsprop / adadelta start from zero state
  }
}

// One element of one optimizer step.  a/b are the element's state values
// (Adagrad: a = norm; FTRL: a = norm, b = zero; Adam: a = m, b = v).  `lr` is the slice learning rate
// (for Adam: the bias-corrected lr_t of the row).  `avx_form` selects the reference's AVX-path
// arithmetic for Adagrad (first floor(dim/8)*8 lanes, ref: avx_utils.h:96-119) vs the baseline form.
template <int OPT>
__device__ __forceinline__ void opt_elem_t(const float* __restrict__ p, bool avx_form, float lr, float g,
                                           float& w, float& a, float& b) {
  if (OPT == MONO_OPT_SGD) {  // sgd_optimizer.cc:46-48
    w = __fsub_rn(w, __fmul_rn(lr, g));
  } else if (OPT == MONO_OPT_ADAGRAD) {
    const float wd = p[1];
    if (avx_form) {  // avx_utils.h:106-113
      float ug = __fmaf_rn(wd, w, g);
      float nn = __fmaf_rn(ug, ug, a);
      a = nn;
      float eff = __fdiv_rn(lr, __fsqrt_rn(nn));
      w = __fmaf_rn(-eff, g, w);
    } else {  // avx_utils.h:31-37
      float gg = __fadd_rn(g, __fmul_rn(wd, w));
      a = __fadd_rn(a, __fmul_rn(gg, gg));
      float eff = __fdiv_rn(lr, __fsqrt_rn(a));
      w = __fsub_rn(w, __fmul_rn(eff, gg));
    }
  } else if (OPT == MONO_OPT_FTRL) {  // ftrl_optimizer.cc:62-75
    const float beta = p[1], l1 = p[2], l2 = p[3];
    float norm_new = __fadd_rn(a, __fmul_rn(g, g));
    float sigma = __fdiv_rn(__fsub_rn(__fsqrt_rn(norm_new), __fsqrt_rn(a)), lr);
    b = __fadd_rn(b, __fsub_rn(g, __fmul_rn(sigma, w)));
    a = norm_new;
    if (fabsf(b) > l1) {
      float sb = signbit(b) ? 1.0f : 0.0f;
      float num = __fmul_rn(lr, __fsub_rn(__fmul_rn(sb, l1), b));
      float den = __fadd_rn(__fadd_rn(__fsqrt_rn(a), beta), __fmul_rn(l2, lr));
      w = __fdiv_rn(num, den);
    } else {
      w = 0.0f;
    }
  } else if (OPT == MONO_OPT_ADAM) {  // adam_optimizer.cc:65-80
    const float beta1 = p[0], beta2 = p[1], eps = p[2], wd = p[3];
    const bool nesterov = p[4] != 0.0f;
    float cur = __fadd_rn(g, __fmul_rn(wd, w));
    float new_m = __fadd_rn(a, __fmul_rn(__fsub_rn(cur, a), __fsub_rn(1.0f, beta1)));
    float new_v = __fadd_rn(b, __fmul_rn(__fsub_rn(__fmul_rn(cur, cur), b), __fsub_rn(1.0f, beta2)));
    float den = __fadd_rn(__fsqrt_rn(new_v), eps);
    if (nesterov) {
      float t1 = __fadd_rn(__fmul_rn(cur, __fsub_rn(1.0f, beta1)), __fmul_rn(beta1, new_m));
      w = __fsub_rn(w, __fdiv_rn(__fmul_rn(t1, lr), den));
    } else {
      w = __fsub_rn(w, __fdiv_rn(__fmul_rn(new_m, lr), den));
    }
    a = new_m;
    b = new_v;
  }
}

__device__ __forceinline__ void opt_elem(const SegDev& s, bool avx_form, float lr, float g, float& w,
                                         float& a, float& b) {
  switch (s.opt_type) {
    case MONO_OPT_SGD: opt_elem_t<MONO_OPT_SGD>(s.p, avx_form, lr, g, w, a, b); break;
    case MONO_OPT_ADAGRAD: opt_elem_t<MONO_OPT_ADAGRAD>(s.p, avx_form, lr, g, w, a, b); break;
    case MONO_OPT_FTRL: opt_elem_t<MONO_OPT_FTRL>(s.p, avx_form, lr, g, w, a, b); break;
    case MONO_OPT_ADAM: opt_elem_t<MONO_OPT_ADAM>(s.p, avx_form, lr, g, w, a, b); break;
  }
}

// One element of the further optimizers (generic path only).  sp = the segment's state block, lc = local column.
// Every step is an explicit IEEE operation in the reference's order (rmsprop computes in double, like the reference).
__device__ __forceinline__ void opt_elem_more(const SegDev& s, int lc, float lr, float g, float& w, float* __restrict__ sp,
                                              bool init_all, float lr_amsgrad) {
  const int D = s.dim;
  if (s.opt_type == MONO_OPT_MOMENTUM) {  // momentum_optimizer.cc:52-72
    const float mom = s.p[0], wd = s.p[1];
    const float n0 = init_all ? 0.0f : sp[lc];
    const float dx = __fmul_rn(lr, __fadd_rn(g, __fmul_rn(wd, w)));
    const float n1 = __fsub_rn(__fmul_rn(mom, n0), dx);
    if (s.p[2] != 0.0f) w = __fadd_rn(w, __fadd_rn(__fmul_rn(-mom, n0), __fmul_rn(__fadd_rn(1.0f, mom), n1)));
    else w = __fadd_rn(w, n1);
    sp[lc] = n1;
  } else if (s.opt_type == MONO_OPT_RMSPROP || s.opt_type == MONO_OPT_RMSPROPV2) {  // rmsprop_optimizer.cc:49-68,121-141
    const double mom = (double)s.p[0], wd = (double)s.p[1];
    const float n0 = init_all ? 0.0f : sp[lc];
    const double dx = __dadd_rn((double)g, __dmul_rn(wd, (double)w));
    float n1;
    double eta;
    if (s.opt_type == MONO_OPT_RMSPROP) {
      n1 = (float)__dadd_rn(__dmul_rn(mom, (double)n0), __dmul_rn(__dmul_rn(__dsub_rn(1.0, mom), dx), dx));
      eta = __ddiv_rn((double)s.p[2], (double)__fadd_rn(__fsqrt_rn(n1), 1.0f));   // the CONFIG's learning rate; sqrt(n) + 1 is a FLOAT sum in the reference
    } else {
      n1 = (float)__dadd_rn(__dmul_rn(mom, (double)n0), __dmul_rn(dx, dx));
      eta = __ddiv_rn((double)lr, (double)__fadd_rn(__fsqrt_rn(n1), 1.0f));
    }
    w = (float)__dsub_rn((double)w, __dmul_rn(eta, dx));
    sp[lc] = n1;
  } else if (s.opt_type == MONO_OPT_ADADELTA) {  // adadelta_optimizer.cc:51-72
    const float rho = s.p[0], eps = s.p[1], wd = s.p[2];
    const float a0 = init_all ? 0.0f : sp[lc], u0 = init_all ? 0.0f : sp[D + lc];
    const float cg = __fadd_rn(g, __fmul_rn(wd, w));
    const float a1 = __fadd_rn(__fmul_rn(a0, rho), __fmul_rn(__fmul_rn(cg, cg), __fsub_rn(1.0f, rho)));
    const float upd = __fmul_rn(__fdiv_rn(__fsqrt_rn(__fadd_rn(u0, eps)), __fsqrt_rn(__fadd_rn(a1, eps))), cg);
    w = __fsub_rn(w, __fmul_rn(upd, lr));
    sp[lc] = a1;
    sp[D + lc] = __fadd_rn(__fmul_rn(u0, rho), __fmul_rn(__fmul_rn(upd, upd), __fsub_rn(1.0f, rho)));
  } else if (s.opt_type == MONO_OPT_AMSGRAD) {  // amsgrad_optimizer.cc:58-88 (lr_amsgrad: bias-corrected, per row)
    const float beta1 = s.p[0], beta2 = s.p[1], eps = s.p[2], wd = s.p[3];
    const float m0 = init_all ? 0.0f : sp[lc], v0 = init_all ? 0.0f : sp[D + lc], h0 = init_all ? 0.0f : sp[2 * D + lc];
    const float cg = __fadd_rn(g, __fmul_rn(wd, w));
    const float m1 = __fadd_rn(m0, __fmul_rn(__fsub_rn(cg, m0), __fsub_rn(1.0f, beta1)));
    const float v1 = __fadd_rn(v0, __fmul_rn(__fsub_rn(__fmul_rn(cg, cg), v0), __fsub_rn(1.0f, beta2)));
    const float h1 = fmaxf(h0, v1);
    const float den = __fadd_rn(__fsqrt_rn(h1), eps);
    if (s.p[4] != 0.0f) {
      const float t1 = __fadd_rn(__fmul_rn(cg, __fsub_rn(1.0f, beta1)), __fmul_rn(beta1, m1));
      w = __fsub_rn(w, __fdiv_rn(__fmul_rn(t1, lr_amsgrad), den));
    } else {
      w = __fsub_rn(w, __fdiv_rn(__fmul_rn(m1, lr_amsgrad), den));
    }
    sp[lc] = m1;
    sp[D + lc] = v1;
    sp[2 * D + lc] = h1;
  } else if (s.opt_type == MONO_OPT_MOVING_AVERAGE) {  // moving_average_optimizer.cc:44-52 (no learning rate, no state)
    const float mom = s.p[0];
    w = __fadd_rn(__fmul_rn(mom, w), __fmul_rn(__fsub_rn(1.0f, mom), g));
  }
}

// GroupAdaGrad (group_adagrad_optimizer.cc:50-89): the segment is ONE group — the accumulator grows by the largest
// squared (decayed) gradient of the group, and the new weights are the group-shrunk z.  The two reductions (max, and
// the sum of squares in column order) make it a whole-segment step: one lane walks the segment, in the reference's
// order, so the result is bit-exact with the oracle.  w = the segment's dim weights (in place), sp = its 1-float state.
__device__ __forceinline__ void group_adagrad_segment(const SegDev& s, float lr, const float* __restrict__ g,
                                                      float* __restrict__ w, float* __restrict__ sp, bool init_all,
                                                      const TableDev* t, int64_t key) {
  const float wd = s.p[1], beta = s.p[2], l2 = s.p[3];
  const int D = s.dim;
  float maxsq = 0.0f;
  for (int i = 0; i < D; ++i) {
    const float wi = init_all ? init_emb_value(t, s, key, s.col_begin + i) : w[i];
    const float gd = __fadd_rn(g[i], __fmul_rn(wd, wi));
    const float sq = __fmul_rn(gd, gd);
    if (sq > maxsq) maxsq = sq;
  }
  const float acc = __fadd_rn(init_all ? s.p[0] : sp[0], maxsq);
  sp[0] = acc;
  const float eff = __fdiv_rn(lr, __fadd_rn(beta, __fsqrt_rn(acc)));
  float zn = 0.0f;
  for (int i = 0; i < D; ++i) {
    const float wi = init_all ? init_emb_value(t, s, key, s.col_begin + i) : w[i];
    const float gd = __fadd_rn(g[i], __fmul_rn(wd, wi));
    const float z = __fsub_rn(gd, __fdiv_rn(wi, eff));
    w[i] = z;
    zn = __fadd_rn(zn, __fmul_rn(z, z));
  }
  zn = __fsqrt_rn(zn);
  if (zn < l2) {
    for (int i = 0; i < D; ++i) w[i] = 0.0f;
  } else {
    const float coef = __fdiv_rn(__fmul_rn(-eff, __fsub_rn(zn, l2)), zn);
    for (int i = 0; i < D; ++i) w[i] = __fmul_rn(coef, w[i]);
  }
}

__device__ __forceinline__ float adam_lr(float lr0, float b1p, float b2p) {  // adam_optimizer.cc:63
  return __fdiv_rn(__fmul_rn(lr0, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));
}

__device__ __forceinline__ int seg_of_col(const TableDev* t, int c) {
  int s = 0;
  for (int i = 1; i < t->num_segs; ++i)
    if (c >= t->segs[i].col_begin) s = i;
  return s;
}
__device__ __forceinline__ int seg_of_state(const TableDev* t, int j) {
  int s = 0;
  for (int i = 1; i < t->num_segs; ++i)
    if (j >= t->segs[i].state_off) s = i;
  return s;
}

// Apply operation OP to row `row` of table t with G lanes.  `fresh` == row was just allocated for a
// key that was absent (ref: UpsertEntry init_fn: Init then fn, cuckoo_embedding_hash_table.cc:346-353).
// vals points at this id's dim floats (grad / value); for kOpRestore at dim+state+2 floats.
template <int G, int OP>
__device__ __forceinline__ void apply_row(const TableDev* __restrict__ t, uint32_t row, int64_t key,
                                          const float* __restrict__ vals,
                                          const float* __restrict__ lr, bool fresh) {
  const int gl = Group<G>::gl();
  const int D = t->dim;
  float* __restrict__ w_row = t->emb + (size_t)row * t->emb_stride;
  float* __restrict__ s_row = t->state + (size_t)row * t->state_stride;
  const bool init_all = fresh || OP == kOpReinit;

  if (OP == kOpOptimize) {
    // ---- fast path: one segment, dim % 4 == 0: 128-bit accesses on w, state and grad ----
    const SegDev& s0 = t->segs[0];
    if (t->num_segs == 1 && s0.opt_type <= MONO_OPT_ADAM && (D & 3) == 0 &&
        ((reinterpret_cast<uintptr_t>(vals) & 15) == 0)) {
      const float lr0 = lr[0];
      float lrt = lr0;
      float b1p = 0.f, b2p = 0.f;
      if (s0.opt_type == MONO_OPT_ADAM) {
        b1p = init_all ? s0.p[0] : s_row[2 * D];
        b2p = init_all ? s0.p[1] : s_row[2 * D + 1];
        lrt = adam_lr(lr0, b1p, b2p);
      }
      const int d8 = D & ~7;
      for (int c = gl * 4; c < D; c += G * 4) {
        float4 g4 = __ldg(reinterpret_cast<const float4*>(vals + c));
        float4 w4, a4 = make_float4(0, 0, 0, 0), b4 = make_float4(0, 0, 0, 0);
        if (init_all) {
          w4.x = init_emb_value(t, s0, key, c);
          w4.y = init_emb_value(t, s0, key, c + 1);
          w4.z = init_emb_value(t, s0, key, c + 2);
          w4.w = init_emb_value(t, s0, key, c + 3);
          a4.x = a4.y = a4.z = a4.w = init_state_value(s0, 0);
          b4.x = b4.y = b4.z = b4.w = init_state_value(s0, D);
        } else {
          w4 = *reinterpret_cast<const float4*>(w_row + c);
          if (s0.opt_type != MONO_OPT_SGD) a4 = *reinterpret_cast<const float4*>(s_row + c);
          if (s0.opt_type == MONO_OPT_FTRL || s0.opt_type == MONO_OPT_ADAM)
            b4 = *reinterpret_cast<const float4*>(s_row + D + c);
        }
        const bool avx = c < d8;  // c is a multiple of 4 and d8 of 8: the 4 lanes agree
        opt_elem(s0, avx, lrt, g4.x, w4.x, a4.x, b4.x);
        opt_elem(s0, avx, lrt, g4.y, w4.y, a4.y, b4.y);
        opt_elem(s0, avx, lrt, g4.z, w4.z, a4.z, b4.z);
        opt_elem(s0, avx, lrt, g4.w, w4.w, a4.w, b4.w);
        *reinterpret_cast<float4*>(w_row + c) = w4;
        if (s0.opt_type != MONO_OPT_SGD) *reinterpret_cast<float4*>(s_row + c) = a4;
        if (s0.opt_type == MONO_OPT_FTRL || s0.opt_type == MONO_OPT_ADAM)
          *reinterpret_cast<float4*>(s_row + D + c) = b4;
      }
      if (s0.opt_type == MONO_OPT_ADAM) {  // adam_optimizer.cc:82-83
        __syncwarp(Group<G>::mask());  // every lane has read the old powers
        if (gl == 0) {
          s_row[2 * D] = __fmul_rn(b1p, s0.p[0]);
          s_row[2 * D + 1] = __fmul_rn(b2p, s0.p[1]);
        }
      }
      return;
    }
  }

  // ---- generic path: any segment mix, any dim; one float per lane per step ----
  if (OP == kOpRestore) {
    for (int c = gl; c < D; c += G) w_row[c] = vals[c];
    for (int j = gl; j < t->state_dim; j += G) s_row[j] = vals[D + j];
    return;
  }
  if (OP == kOpOptimize) {  // whole-segment optimizers: one lane per segment, ahead of the per-column loop
    for (int si = gl; si < t->num_segs; si += G) {
      const SegDev& s = t->segs[si];
      if (s.opt_type == MONO_OPT_GROUP_ADAGRAD)
        group_adagrad_segment(s, lr[si], vals + s.col_begin, w_row + s.col_begin, s_row + s.state_off, init_all, t, key);
    }
  }
  for (int c = gl; c < D; c += G) {
    const int si = seg_of_col(t, c);
    const SegDev& s = t->segs[si];
    const int lc = c - s.col_begin;
    if (OP == kOpOptimize && s.opt_type == MONO_OPT_GROUP_ADAGRAD) continue;  // done above
    float w = init_all ? init_emb_value(t, s, key, c) : w_row[c];
    if (OP == kOpAssign) {
      w = vals[c];
    } else if (OP == kOpAssignAdd) {
      w = __fadd_rn(w, vals[c]);
    } else if (OP == kOpOptimize) {
      float a = 0.f, b = 0.f, lrt = lr[si];
      float* sp = s_row + s.state_off;
      if (s.opt_type > MONO_OPT_ADAM) {
        float lra = lrt;
        if (s.opt_type == MONO_OPT_AMSGRAD)
          lra = adam_lr(lrt, init_all ? s.p[0] : sp[3 * s.dim], init_all ? s.p[1] : sp[3 * s.dim + 1]);
        opt_elem_more(s, lc, lrt, vals[c], w, sp, init_all, lra);
        w_row[c] = w;
        continue;
      }
      if (s.opt_type == MONO_OPT_ADAGRAD) {
        a = init_all ? s.p[0] : sp[lc];
      } else if (s.opt_type == MONO_OPT_FTRL) {
        a = init_all ? s.p[0] : sp[lc];
        b = init_all ? 0.0f : sp[s.dim + lc];
      } else if (s.opt_type == MONO_OPT_ADAM) {
        a = init_all ? 0.0f : sp[lc];
        b = init_all ? 0.0f : sp[s.dim + lc];
        float b1p = init_all ? s.p[0] : sp[2 * s.dim];
        float b2p = init_all ? s.p[1] : sp[2 * s.dim + 1];
        lrt = adam_lr(lrt, b1p, b2p);
      }
      opt_elem(s, lc < (s.dim & ~7), lrt, vals[c], w, a, b);
      if (s.opt_type == MONO_OPT_ADAGRAD) {
        sp[lc] = a;
      } else if (s.opt_type == MONO_OPT_FTRL || s.opt_type == MONO_OPT_ADAM) {
        sp[lc] = a;
        sp[s.dim + lc] = b;
      }
    }
    w_row[c] = w;
  }
  if (OP == kOpOptimize) {
    // per-row beta powers advance once per step (after every lane has read the old values)
    __syncwarp(Group<G>::mask());
    if (gl == 0) {
      for (int si = 0; si < t->num_segs; ++si) {
        const SegDev& s = t->segs[si];
        if (s.opt_type != MONO_OPT_ADAM && s.opt_type != MONO_OPT_AMSGRAD) continue;
        float* sp = s_row + s.state_off;
        const int po = (s.opt_type == MONO_OPT_ADAM ? 2 : 3) * s.dim;  // where the beta powers live
        float b1p = init_all ? s.p[0] : sp[po];
        float b2p = init_all ? s.p[1] : sp[po + 1];
        sp[po] = __fmul_rn(b1p, s.p[0]);
        sp[po + 1] = __fmul_rn(b2p, s.p[1]);
      }
    }
  } else if (init_all) {
    // assign / assign_add / reinitialize on a fresh (or re-initialised) row: optimizer Init
    for (int j = gl; j < t->state_dim; j += G) {
      const SegDev& s = t->segs[seg_of_state(t, j)];
      s_row[j] = init_state_value(s, j - s.state_off);
    }
  }
}

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// lane-per-key probe of the bucketised table: the whole 64-byte bucket with 4 x LDG.128 per lane
// DUAL: both candidate buckets are requested together (8 x LDG.128).  A warp-tile of 32 probes almost always holds a
// key that lives in its second bucket, so the sequential form costs the WARP two dependent round trips; DUAL trades
// 64 extra bytes per key for one round trip (knobs lookup_dual / claim_dual).
// LD = 0: read-only (non-coherent, L1) loads; LD = 1: loads coherent at L2 (the confirm-a-miss path below)
template <bool DUAL = false, int LD = 0>
__device__ __forceinline__ uint32_t probe_lane(const TableDev* __restrict__ t, int64_t key) {
  const Entry* __restrict__ buckets = t->buckets;
  uint32_t b1, b2;
  bucket_pair(key, t->num_buckets, b1, b2);
  uint32_t row = kEmptyRow;
  if (DUAL) {
    const Entry* p = buckets + (size_t)b1 * kBucketSlots;
    const Entry* q = buckets + (size_t)b2 * kBucketSlots;
    Entry e0 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p), e1 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 1), e2 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 2), e3 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 3);
    Entry f0 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(q), f1 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(q + 1), f2 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(q + 2), f3 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(q + 3);
    if (f0.key == key && f0.row < kTombRow) row = f0.row & kRowMask;
    if (f1.key == key && f1.row < kTombRow) row = f1.row & kRowMask;
    if (f2.key == key && f2.row < kTombRow) row = f2.row & kRowMask;
    if (f3.key == key && f3.row < kTombRow) row = f3.row & kRowMask;
    if (e0.key == key && e0.row < kTombRow) row = e0.row & kRowMask;
    if (e1.key == key && e1.row < kTombRow) row = e1.row & kRowMask;
    if (e2.key == key && e2.row < kTombRow) row = e2.row & kRowMask;
    if (e3.key == key && e3.row < kTombRow) row = e3.row & kRowMask;
    if (row == kEmptyRow && (LD == 0 ? t->ctrs[kCtrStash] : ld_acquire_u32(t->ctrs + kCtrStash)) != 0) {
      const uint32_t mask = t->stash_cap - 1;
      const uint32_t s = (uint32_t)(mix64((uint64_t)key) >> 17) & mask;
      for (uint32_t i = 0; i <= mask; ++i) {
        Entry e = ld_entry_cg(t->stash + ((s + i) & mask));
        if (e.row == kEmptyRow) break;
        if (e.key == key && e.row < kTombRow) { row = e.row & kRowMask; break; }
      }
    }
    return row;
  }
  {
    const Entry* p = buckets + (size_t)b1 * kBucketSlots;
    Entry e0 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p), e1 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 1), e2 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 2), e3 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 3);
    if (e0.key == key && e0.row < kTombRow) row = e0.row & kRowMask;
    if (e1.key == key && e1.row < kTombRow) row = e1.row & kRowMask;
    if (e2.key == key && e2.row < kTombRow) row = e2.row & kRowMask;
    if (e3.key == key && e3.row < kTombRow) row = e3.row & kRowMask;
  }
  if (row == kEmptyRow) {
    const Entry* p = buckets + (size_t)b2 * kBucketSlots;
    Entry e0 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p), e1 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 1), e2 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 2), e3 = (LD == 0 ? ld_entry_nc : ld_entry_cg)(p + 3);
    if (e0.key == key && e0.row < kTombRow) row = e0.row & kRowMask;
    if (e1.key == key && e1.row < kTombRow) row = e1.row & kRowMask;
    if (e2.key == key && e2.row < kTombRow) row = e2.row & kRowMask;
    if (e3.key == key && e3.row < kTombRow) row = e3.row & kRowMask;
    if (row == kEmptyRow && (LD == 0 ? t->ctrs[kCtrStash] : ld_acquire_u32(t->ctrs + kCtrStash)) != 0) {
      const uint32_t mask = t->stash_cap - 1;
      const uint32_t s = (uint32_t)(mix64((uint64_t)key) >> 17) & mask;
      for (uint32_t i = 0; i <= mask; ++i) {
        Entry e = ld_entry_cg(t->stash + ((s + i) & mask));
        if (e.row == kEmptyRow) break;
        if (e.key == key && e.row < kTombRow) { row = e.row & kRowMask; break; }
      }
    }
  }
  return row;
}


// A lookup that missed while ANOTHER STREAM may be inserting.  cuckoo_insert moves a resident entry between its two
// buckets copy-first and bumps ctrs[kCtrMoves] between the copy and the overwrite of the old slot, so a reader can
// only miss a resident key if the counter changes between its two bucket reads.  The fast probe cannot be trusted for
// that (its non-coherent loads may be served by an L1 line that is older than the move), so every miss is confirmed:
// probe again with loads that are coherent at L2, bracketed by counter reads, until one probe runs with no move in
// between — and with no entry in flight: the rare exchange fallback of cuckoo_insert carries a resident entry in a
// register, ctrs[kCtrInflight] counts those.  Cost: three L2-hit loads and one extra probe per MISS (absent FIDs only;
// resident FIDs never come here).
static __device__ __noinline__ uint32_t probe_lane_confirm_miss(const TableDev* __restrict__ t, int64_t key) {
  const uint32_t* mv = t->ctrs + kCtrMoves;
  const uint32_t* fl = t->ctrs + kCtrInflight;
  uint32_t ma = ld_acquire_u32(mv);
  for (int tries = 0; tries < 64; ++tries) {
    const uint32_t row = probe_lane<false, 1>(t, key);
    if (row != kEmptyRow) return row;
    __threadfence();
    // the in-flight count is read BEFORE the move counter: an insert that re-places a carried entry bumps the counter
    // and only then leaves the in-flight count, so "nothing in flight" + "counter unchanged" cannot both be observed
    // around a probe that ran while the entry was in a register (tests/test_cuckoo_protocol_model.py found the other order)
    const uint32_t in_flight = ld_acquire_u32(fl);
    const uint32_t mb = ld_acquire_u32(mv);
    if (mb == ma && in_flight == 0) return kEmptyRow;   // absent for sure
    ma = mb;
  }
  return kEmptyRow;
}

constexpr uint32_t kFreshBit = 0x80000000u;

// probe that also returns the matching entry's address (for the timestamp bump)
template <bool DUAL = false>
__device__ __forceinline__ uint32_t probe_lane_slot(const TableDev* __restrict__ t, int64_t key,
                                                    Entry** slot) {
  Entry* buckets = t->buckets;
  uint32_t b1, b2;
  bucket_pair(key, t->num_buckets, b1, b2);
  uint32_t row = kEmptyRow;
  if (DUAL) {
    Entry* p = buckets + (size_t)b1 * kBucketSlots;
    Entry* q = buckets + (size_t)b2 * kBucketSlots;
    Entry e0 = ld_entry(p), e1 = ld_entry(p + 1), e2 = ld_entry(p + 2), e3 = ld_entry(p + 3);
    Entry f0 = ld_entry(q), f1 = ld_entry(q + 1), f2 = ld_entry(q + 2), f3 = ld_entry(q + 3);
    if (f0.key == key && f0.row < kTombRow) { row = f0.row & kRowMask; *slot = q; }
    if (f1.key == key && f1.row < kTombRow) { row = f1.row & kRowMask; *slot = q + 1; }
    if (f2.key == key && f2.row < kTombRow) { row = f2.row & kRowMask; *slot = q + 2; }
    if (f3.key == key && f3.row < kTombRow) { row = f3.row & kRowMask; *slot = q + 3; }
    if (e0.key == key && e0.row < kTombRow) { row = e0.row & kRowMask; *slot = p; }
    if (e1.key == key && e1.row < kTombRow) { row = e1.row & kRowMask; *slot = p + 1; }
    if (e2.key == key && e2.row < kTombRow) { row = e2.row & kRowMask; *slot = p + 2; }
    if (e3.key == key && e3.row < kTombRow) { row = e3.row & kRowMask; *slot = p + 3; }
    if (row != kEmptyRow) return row;
  } else {
#pragma unroll
    for (int round = 0; round < 2; ++round) {
      Entry* p = buckets + (size_t)(round == 0 ? b1 : b2) * kBucketSlots;
      Entry e0 = ld_entry(p), e1 = ld_entry(p + 1), e2 = ld_entry(p + 2), e3 = ld_entry(p + 3);
      if (e0.key == key && e0.row < kTombRow) { row = e0.row & kRowMask; *slot = p; }
      if (e1.key == key && e1.row < kTombRow) { row = e1.row & kRowMask; *slot = p + 1; }
      if (e2.key == key && e2.row < kTombRow) { row = e2.row & kRowMask; *slot = p + 2; }
      if (e3.key == key && e3.row < kTombRow) { row = e3.row & kRowMask; *slot = p + 3; }
      if (row != kEmptyRow) return row;
    }
  }
  if (t->ctrs[kCtrStash] != 0) {
    const uint32_t mask = t->stash_cap - 1;
    const uint32_t s = (uint32_t)(mix64((uint64_t)key) >> 17) & mask;
    for (uint32_t i = 0; i <= mask; ++i) {
      Entry* p = t->stash + ((s + i) & mask);
      Entry e = ld_entry_cg(p);
      if (e.row == kEmptyRow) break;
      if (e.key == key && e.row < kTombRow) { *slot = p; return e.row & kRowMask; }
    }
  }
  return kEmptyRow;
}


__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

// ---- cp.async staging: rows requested kStage at a time into per-thread shared-memory slots (zero register cost) ----
constexpr int kStage = 16;
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}

// cp.async of a lane's 4 elements into its 16-byte stage slot (a bf16 row fills the slot's first 8 bytes)
__device__ __forceinline__ void cp_async_row4(void* smem_dst, const float* gsrc) { cp_async16(smem_dst, gsrc); }
__device__ __forceinline__ void cp_async_row4(void* smem_dst, const __nv_bfloat16* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(gsrc) : "memory");
}
// ---- host helpers implemented in ops.cu ----
struct CallBlob {  // device pointers into the staged per-call descriptor block
  const CallSeg* segs;
  const float* lr;
  const int32_t* table_ids;
  int ntab;
};
CallBlob stage_call(mono_mtable* mt, const CallSeg* h_segs, int nsegs, const float* lr_host, int n_lr, cudaStream_t s);
int pick_group(int max_dim);
void launch_apply_window(mono_mtable* mt, int k, const CallBlob& cb, const int64_t* ids_base, const float* grads_base,
                         int64_t pos0, const uint32_t* n_dev, int64_t n_upper, uint32_t* rowidx, uint32_t update_ts,
                         const uint64_t* wait_flag, uint64_t wait_seq, cudaStream_t s);
// folds the call's per-table miss tickets into the allocator counters (upsert_finalize_kernel)
void launch_upsert_finalize(mono_mtable* mt, const CallBlob& cb, uint32_t* miss_ctr, uint32_t update_ts, cudaStream_t s);

}  // namespace mono
