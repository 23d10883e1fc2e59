// nnk_mlpg.cu -- batched MLPG (maximum likelihood parameter generation) on sm_90a.
//
// Replaces, for a whole batch of utterances and every static dimension at once:
//   paramgen.mlpg       paramgen/_mlpg.py:92-199  (build_poe :53-89 -> _bandmat/tensor.pyx:20-64,
//                       82-174; bla.solveh -> _bandmat/linalg.pyx:36-104, 106-176, 290-304)
//   paramgen.mlpg_grad  paramgen/_mlpg.py:202-281 (closed form  tau_w * (W_w P^-1 o), O(T))
// and, additive, the gradient in the means and the variances together (MODE_VJP, nnk_mlpg_vjp).
//
// Mapping: one "chain" = one static dimension of one stream of one utterance = one symmetric
// banded T x T system  P y = b,  P = sum_w W_w^T diag(tau_w) W_w,  b = sum_w W_w^T (tau_w * mu_w).
// One warp owns 32 chains of one utterance (lane = feature dimension, so every global access is a
// coalesced row segment of the (T, D) frame matrix) and walks time:
//   forward sweep : assemble row t of P and b in registers from a sliding window of frames,
//                   eliminate (L D L^T, band depth S = L+U), forward-substitute; the S+1 numbers a
//                   frame needs later (z/d, l_1..l_S) go to a float64 scratch laid out
//                   [t][j][lane] so each access is one 256 B line per warp;
//   backward sweep: y[t] = zs[t] - sum_j l_j[t] y[t+j], written to the output in the input dtype.
// All arithmetic is float64 (the reference's bandmat is float64-only); P is never materialised in
// HBM.  L D L^T instead of the reference's L L^T: same pivots d[t] (so the same not-positive-
// definite test, linalg.pyx:79), no sqrt on the loop-carried dependency chain, results agree to
// rounding (1e-15 relative).
//
// Two kernels: mlpg_kernel below (one warp per work item, register-prefetched loads, every mode) and the
// warp-specialised, TMA-staged mlpg_fwd_as_kernel of nnk_mlpg_as.cuh.  launch_mlpg takes the staged kernel
// for forward solves and float32-grad_output gradients whose window set fills its template instance
// (nw == NW), with NT <= 5 and rows narrow enough for as_geometry; everything else runs mlpg_kernel.
#include <type_traits>

#include "nnk_mlpg.cuh"
#include "nnk_mlpg_as.cuh"

namespace nnk {

// staged kernel configuration, settled by the A/B measurements of DESIGN.md §3.1: 4-frame tiles, three
// assembler warps per chain group with one TMA stage each (two per assembler pair when a CTA serves two chain
// groups), a band-row ring of 6 tiles (>= the paired producers' tile stride 2 NA - 1, see nnk_mlpg_as.cuh), and
// 8-frame backward tiles, 8 in flight (4 when the variance rows ride along in the gradient)
constexpr int AS_TT = 4, AS_NA = 3, AS_NSA1 = 1, AS_NSA2 = 2, AS_ND = 6, AS_TTB = 8;

__device__ __forceinline__ double load_go(const void* go, int is_f64, int64_t idx) {
  return is_f64 ? ld_stream(reinterpret_cast<const double*>(go) + idx)
                : (double)ld_stream(reinterpret_cast<const float*>(go) + idx);
}

// ---- global-variance refinement (MODE_GV, nnk_mlpg_gv) --------------------------------------------------
// One chain (one lane).  The sweeps below have left per frame t, in the lane's scratch column col (stride 32):
//   0: zs_t = (L^-1 b)_t / d_t,   1..S: l_j[t] = L[t+j][t],   NT: d_t,   NT+1: c_m,t = (P^-1 b)_t
// of P = L D L^T.  gv_refine maximises
//   F(c) = omega (b^T c - c^T P c / 2) - prec (v(c) - mu)^2 / 2,   v(c) = (1/T) sum_t (c_t - mean(c))^2
// (Toda, Black & Tokuda 2007, Eq. 44 with a diagonal GV covariance) from c0 = mean + sqrt(mu / v(c_m)) (c_m - mean)
// by n_iter trials of the P-preconditioned step  delta = (c_m - c) + P^-1 g / omega,  g_t = -(2/T) prec (v - mu)
// (c_t - mean):  c + alpha delta replaces c when F does not decrease, otherwise alpha halves.  F comes from the
// factors: with e = L^T c,  b^T c = sum_t d_t zs_t e_t  and  c^T P c = sum_t d_t e_t^2.  The current and the trial
// trajectory live in columns NT+2 / NT+3 and swap roles on acceptance.  Every sum runs over t in a fixed order, so
// results do not depend on the batch around the chain.
template <int S, int NTS, typename Tout>
__device__ __forceinline__ void gv_refine(double* ws, int T, double mu, double prec, double omega,
                                          int n_iter, double step, Tout* out, int64_t out_ld) {
  constexpr int NT = S + 1, C_D = NT, C_CM = NT + 1, SP = S > 0 ? S : 1;
  auto at = [&](int t, int col) -> double& { return ws[(size_t)t * (NTS * 32) + col * 32]; };
  const double invT = 1.0 / (double)T;
  auto variance = [&](int col, double mean) {
    double v = 0.0;
    for (int t = 0; t < T; ++t) {
      const double dv = at(t, col) - mean;
      v = fma(dv, dv, v);
    }
    return v * invT;
  };
  // x_t goes to column dst; returns sum_t d_t e_t (zs_t - e_t / 2) with e = L^T x, and sum_t x_t in sx.  With
  // SOLVE, dst holds (L^-1 g)_t / d_t on entry and x_t = c_t + alpha ((c_m,t - c_t) + z_t / omega), z = P^-1 g;
  // otherwise x_t = c0_t = mean + scale (c_m,t - mean).
  auto back_pass = [&](auto solve_tag, int src, int dst, double a, double b, double& sx) {
    constexpr bool SOLVE = decltype(solve_tag)::value;
    double xw[S + 1], zw[S + 1];
#pragma unroll
    for (int j = 0; j <= S; ++j) { xw[j] = 0.0; zw[j] = 0.0; }
    double q = 0.0;
    sx = 0.0;
    for (int t = T - 1; t >= 0; --t) {
      double l[S + 1];
#pragma unroll
      for (int j = 1; j <= S; ++j) l[j] = at(t, j);
#pragma unroll
      for (int j = S; j > 0; --j) { xw[j] = xw[j - 1]; zw[j] = zw[j - 1]; }
      const double cm = at(t, C_CM);
      double x;
      if constexpr (SOLVE) {
        double z = at(t, dst);
#pragma unroll
        for (int j = 1; j <= S; ++j) z = fma(-l[j], zw[j], z);
        zw[0] = z;
        const double c = at(t, src);
        x = c + a * ((cm - c) + z / b);
      } else {
        x = a + b * (cm - a);
      }
      xw[0] = x;
      at(t, dst) = x;
      double e = x;
#pragma unroll
      for (int j = 1; j <= S; ++j) e = fma(l[j], xw[j], e);
      q = fma(at(t, C_D) * e, at(t, 0) - 0.5 * e, q);
      sx += x;
    }
    return q;
  };

  // start point.  The mean of c_m is taken about its last frame, so that a c_m with one value at every frame has
  // v(c_m) == 0 exactly: (sum_t c_m,t) * (1 / T) can miss that value by an ulp, which sqrt(mu / v) would scale
  // up to the target variance.
  const double c_last = at(T - 1, C_CM);
  double dsum = 0.0;
  for (int t = T - 1; t >= 0; --t) dsum += at(t, C_CM) - c_last;
  const double mean_m = c_last + dsum * invT;
  const double vm = variance(C_CM, mean_m);
  int cur = NT + 2, nxt = NT + 3;
  double sx;
  double q = back_pass(std::false_type{}, C_CM, cur, mean_m, vm > 0.0 ? sqrt(mu / vm) : 1.0, sx);
  double mean = sx * invT, v = variance(cur, mean);
  double f = omega * q - 0.5 * prec * (v - mu) * (v - mu);

  double alpha = step;
  for (int it = 0; it < n_iter; ++it) {
    // forward substitution of g: column nxt = (L^-1 g) / d
    const double gs = -2.0 * invT * prec * (v - mu);
    double pend[SP];  // pend[k]: sum of the eliminated terms of frame t + k
#pragma unroll
    for (int k = 0; k < SP; ++k) pend[k] = 0.0;
    for (int t = 0; t < T; ++t) {
      const double w = gs * (at(t, cur) - mean) - pend[0];
      if constexpr (S > 0) {
#pragma unroll
        for (int k = 0; k + 1 < S; ++k) pend[k] = fma(at(t, k + 1), w, pend[k + 1]);
        pend[S - 1] = at(t, S) * w;
      }
      at(t, nxt) = w / at(t, C_D);
    }
    double sx2;
    const double q2 = back_pass(std::true_type{}, cur, nxt, alpha, omega, sx2);
    const double mean2 = sx2 * invT, v2 = variance(nxt, mean2);
    const double f2 = omega * q2 - 0.5 * prec * (v2 - mu) * (v2 - mu);
    if (f2 >= f) {
      const int tmp = cur; cur = nxt; nxt = tmp;
      f = f2; mean = mean2; v = v2;
    } else {
      alpha *= 0.5;
    }
  }
  for (int t = 0; t < T; ++t) st_stream(out + (int64_t)t * out_ld, (Tout)at(t, cur));
}

// ---- trajectory-model log-likelihood (MODE_TLL, MODE_TLL_GRAD; nnk_mlpg_traj_ll) ------------------------------
// The forward sweep is MODE_FWD's; it also sums log d_t and, with the gradient, stores 1 / d_t in scratch column NT.
// The backward sweep recomputes cbar = P^-1 b as MODE_FWD does, keeps windows of cbar and of the targets x, and at
// step t handles row r = t + L (the row MODE_GRAD emits at the same step): u = W_w x and ubar = W_w cbar over frames
// t .. t + S give the tau (u - ubar)^2 term of l and dl/dmu = tau (u - ubar).  With the gradient it also carries
// the (S+1) x (S+1) block Sigma[t + a][t + b] of Sigma = P^-1, by the backward recurrence for the band of an
// inverse (Takahashi et al. 1973; l_k[t] = L[t+k][t]):
//   Sigma[t][t+j] = -sum_k l_k[t] Sigma[t+k][t+j]  (j = 1..S),   Sigma[t][t] = 1/d_t - sum_k l_k[t] Sigma[t][t+k],
// which gives w_r^T Sigma w_r and dl/dvar, and emits dl/dx at frame t + S from a window of the dl/dmu rows.
// The block is upper-triangular in registers (a <= b).
template <int S>
__device__ __forceinline__ double sym_at(const double (&sg)[S + 1][S + 1], int a, int b) {
  return a <= b ? sg[a][b] : sg[b][a];
}

// ---- sampling from the trajectory model (MODE_SAMPLE, nnk_mlpg_traj_sample) --------------------------------------
// The comment of nnk_mlpg_traj_sample in include/nnk_b200.h is the normative definition of the noise; these two
// functions restate it.
// Philox4x32-10 (Salmon et al. 2011); the key bump after the last round is not used.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

// the Box-Muller pair of counter c: zc for the even frame 2 (t >> 1), zs for the odd one
__device__ __forceinline__ void normal_pair(uint4 c, unsigned long long seed, double& zc, double& zs) {
  const uint4 r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  const unsigned long long nu = ((unsigned long long)(r.x >> 6) << 26) | (r.y >> 6);
  const unsigned long long nv = ((unsigned long long)(r.z >> 6) << 26) | (r.w >> 6);
  const double u = ((double)nu + 0.5) * 0x1p-52;  // exact: nu < 2^52
  const double v = (double)nv * 0x1p-52;
  const double rad = sqrt(-2.0 * log(u));
  double sn, cs;
  sincospi(2.0 * v, &sn, &cs);
  zc = rad * cs;
  zs = rad * sn;
}

// One chain (one lane).  The forward sweep has left per frame t, in the lane's scratch column col (stride 32):
//   0: zs_t = (L^-1 b)_t / d_t,   1..S: l_j[t] = L[t+j][t],   NT: 1 / sqrt(d_t), computed as sqrt(1 / d_t)
// Each sample is one backward sweep over those factors, MODE_FWD's term for term but for its start value:
//   y_t = fma(scale * z_{s,t}, 1 / sqrt(d_t), zs_t) - sum_j l_j[t] y_{t+j}   (j = 1 .. S in that order, as fmas)
// so scale = 0 gives MODE_FWD's trajectory.  Sample s goes to out + s * sample_stride.  The frames of a PF block
// get their noise first, off the serial chain; one Philox call serves the pair (t, t - 1) for odd t, and an even
// last frame T - 1 takes the cosine of its own call.  A sample's bits depend on s, never on n_samples.
template <int S, int NTS, int PF, typename Tout>
__device__ __forceinline__ void sample_sweeps(const double* ws, int T, int n_samples, int64_t sample_stride,
                                              uint32_t out_col, uint32_t key, unsigned long long seed, double scale,
                                              Tout* out, int64_t out_ld) {
  constexpr int NT = S + 1;
  auto load = [&](int t, double& z, double(&l)[S + 1], double& isd) {
    z = 0.0; isd = 0.0;
#pragma unroll
    for (int j = 0; j <= S; ++j) l[j] = 0.0;
    if (t >= 0) {
      const double* wsp = ws + (size_t)t * (NTS * 32);
      z = wsp[0];
#pragma unroll
      for (int j = 1; j <= S; ++j) l[j] = wsp[j * 32];
      isd = wsp[NT * 32];
    }
  };
  for (int s = 0; s < n_samples; ++s) {
    Tout* o = out + (int64_t)s * sample_stride;
    double yw[S + 1];
#pragma unroll
    for (int j = 0; j <= S; ++j) yw[j] = 0.0;
    double rz[PF], rl[PF][S + 1], ri[PF];
#pragma unroll
    for (int j = 0; j < PF; ++j) load(T - 1 - j, rz[j], rl[j], ri[j]);
    double zc = 0.0;  // the cosine normal of the pair of the last odd frame
    for (int t0 = T - 1; t0 >= 0; t0 -= PF) {
      double y0[PF];
#pragma unroll
      for (int jj = 0; jj < PF; ++jj) {
        const int t = t0 - jj;
        double z = zc;
        if (t >= 0 && ((t & 1) || t == T - 1)) {
          double zs;
          normal_pair(make_uint4((uint32_t)t >> 1, out_col, (uint32_t)s, key), seed, zc, zs);
          z = (t & 1) ? zs : zc;
        }
        y0[jj] = fma(scale * z, ri[jj], rz[jj]);
      }
#pragma unroll
      for (int jj = 0; jj < PF; ++jj) {
        const int t = t0 - jj;
        if (t >= 0) {
#pragma unroll
          for (int j = S; j > 0; --j) yw[j] = yw[j - 1];
          double y = y0[jj];
#pragma unroll
          for (int j = 1; j <= S; ++j) y = fma(-rl[jj][j], yw[j], y);
          yw[0] = y;
          load(t - PF, rz[jj], rl[jj], ri[jj]);
          st_stream(o + (int64_t)t * out_ld, (Tout)y);
        }
      }
    }
  }
}

// ---- gradient in means and variances (MODE_VJP, nnk_mlpg_vjp) ---------------------------------------------------
// The forward sweep eliminates two right-hand sides with the same factors: b from the means (MODE_FWD's) and o, the
// gradient with respect to the trajectory, read at the output's rows and columns (MODE_GRAD's, which reads it by
// chain); (L^-1 o)_t / d_t goes to scratch column NT.  The backward sweep back-substitutes both, cbar = P^-1 b and
// g = P^-1 o, keeps windows of them over frames t .. t + S, and at step t emits row r = t + L (as MODE_GRAD does),
// reloading that row's means and variances:
//   dL/dmu_{r,w} = tau_{r,w} (W_w g)_r,   dL/dvar_{r,w} = -tau_{r,w}^2 (W_w g)_r (mu_{r,w} - (W_w cbar)_r).
// Global variances sum dL/dvar over the rows in that order in the lane (TLL_GRAD's partials).
template <typename Tin, int NW, int L, int U, int MODE, int PF>
__global__ void __launch_bounds__(32) mlpg_kernel(const __grid_constant__ typename KernelParams<Tin, NW, L, U, MODE>::type p) {
  constexpr int S = L + U;
  constexpr int NT = S + 1;
  constexpr int NTS = WsCols<MODE, NT>::value;
  constexpr bool TLL = (MODE == MODE_TLL || MODE == MODE_TLL_GRAD);
  constexpr bool TGRAD = (MODE == MODE_TLL_GRAD);
  constexpr bool VJP = (MODE == MODE_VJP);
  // means in (trajectories out, but TLL and VJP)
  constexpr bool FWDLIKE = (MODE == MODE_FWD || MODE == MODE_GV || TLL || MODE == MODE_SAMPLE || VJP);
  const int lane = threadIdx.x;
  const int item = blockIdx.x;
  const int urank = p.urank0 + item / p.n_groups;
  const int grp = item % p.n_groups;
  const int utt = p.order ? p.order[urank] : urank;
  const int64_t row0 = p.utt_off[utt];
  const int T = p.utt_len ? p.utt_len[utt] : (int)(p.utt_off[utt + 1] - row0);
  if (T <= 0) return;
  const int64_t orow0 = p.out_off ? p.out_off[utt] : row0;
  const int chain = grp * 32 + lane;
  const bool active = chain < p.n_chain;
  nnk_chain_t ch;
  ch.in_col = 0; ch.win_stride = 0; ch.out_col = 0; ch.flags = 1;
  if (active) ch = p.chains[chain];
  const bool solve = active && !(ch.flags & 1);
  const int nw = p.win.nw;
  const int m_edge = p.win.m_edge;
  const bool var_global = (p.var_ld == 0);

  const Tin* mptr = p.means + row0 * p.in_ld + ch.in_col;
  const Tin* vptr = p.vars + (var_global ? 0 : row0 * p.var_ld) + ch.in_col;
  double* ws = p.ws + (size_t)item * ((size_t)p.max_T * NTS * 32) + lane;

  // ---- pass-through chains (flags & 1): plain copy (fwd) / gradient of a copy (grad) -----------
  if (active && (ch.flags & 1)) {
    if constexpr (TLL) {
      p.ll[(int64_t)utt * p.n_chain + chain] = 0.0;
    } else if constexpr (MODE == MODE_SAMPLE) {
      for (int s = 0; s < p.n_samples; ++s) {
        Tin* o = reinterpret_cast<Tin*>(p.out) + s * p.sample_stride + orow0 * p.out_ld + ch.out_col;
        for (int t = 0; t < T; ++t) o[(int64_t)t * p.out_ld] = mptr[(int64_t)t * p.in_ld];
      }
    } else if constexpr (VJP) {
      const Tin* go = reinterpret_cast<const Tin*>(p.go) + orow0 * p.go_ld + ch.out_col;
      Tin* o = p.grad_means + row0 * p.gm_ld + ch.in_col;
      for (int t = 0; t < T; ++t) o[(int64_t)t * p.gm_ld] = go[(int64_t)t * p.go_ld];
    } else if (FWDLIKE) {
      Tin* o = reinterpret_cast<Tin*>(p.out) + orow0 * p.out_ld + ch.out_col;
      for (int t = 0; t < T; ++t) o[(int64_t)t * p.out_ld] = mptr[(int64_t)t * p.in_ld];
    } else if (MODE == MODE_GRAD) {
      float* o = reinterpret_cast<float*>(p.out) + orow0 * p.out_ld + ch.in_col;
      for (int t = 0; t < T; ++t) o[(int64_t)t * p.out_ld] = (float)load_go(p.go, p.go_f64, (row0 + t) * p.go_ld + chain);
    }
  }

  Tin gv[NW];
#pragma unroll
  for (int w = 0; w < NW; ++w) gv[w] = (solve && var_global && w < nw) ? vptr[w * ch.win_stride] : Tin(1);

  // VJP: o of the chain's frame 0, at the output's row and column
  const Tin* gop = VJP ? reinterpret_cast<const Tin*>(p.go) + orow0 * p.go_ld + ch.out_col : nullptr;
  // raw (un-converted) frame loads; t outside [0, T) or idle lanes give zeros
  auto load_raw = [&](int t, Tin(&m)[NW], Tin(&v)[NW], double& g) {
#pragma unroll
    for (int w = 0; w < NW; ++w) { m[w] = Tin(0); v[w] = Tin(1); }
    g = 0.0;
    if (t >= 0 && t < T && solve) {
#pragma unroll
      for (int w = 0; w < NW; ++w) {
        if (w < nw) {
          if (FWDLIKE) m[w] = ld_stream(mptr + (int64_t)t * p.in_ld + w * ch.win_stride);
          v[w] = var_global ? gv[w] : ld_stream(vptr + (int64_t)t * p.var_ld + w * ch.win_stride);
        }
      }
      if constexpr (VJP) g = (double)ld_stream(gop + (int64_t)t * p.go_ld);
      else if (!FWDLIKE) g = load_go(p.go, p.go_f64, (row0 + t) * p.go_ld + chain);
    }
  };
  // tau_w[t] with the reference's edge rule; tm = tau * mu (paramgen/_mlpg.py:188-195)
  auto to_frame = [&](int t, const Tin(&m)[NW], const Tin(&v)[NW], double(&tau)[NW], double(&tm)[NW]) {
    const bool in = (t >= 0 && t < T);
    const bool edge = (m_edge == 0) || (t < m_edge) || (t >= T - m_edge);
#pragma unroll
    for (int w = 0; w < NW; ++w) {
      const bool on = in && (w < nw) && !(w > 0 && edge);
      const double tw = on ? recip_in_dtype<Tin>::f(v[w]) : 0.0;
      tau[w] = tw;
      tm[w] = tw * (double)m[w];
    }
  };

  // ---- forward sweep -----------------------------------------------------------------------------
  double wt[NT][NW], wm[NT][NW];  // wt[i] = tau of frame (t + L - i)
  double wg[NT];                  // grad/solve mode, VJP: right-hand side (o) of frame (t + L - i)
#pragma unroll
  for (int i = 0; i < NT; ++i) {
    wg[i] = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) { wt[i][w] = 0.0; wm[i][w] = 0.0; }
  }
  // window before step 0 (after the shift at step 0, wt[i] = frame L - i): preload frames 0..L-1
#pragma unroll
  for (int i = 0; i < L; ++i) {  // frame f = L-1-i goes to slot i (it will be shifted to i+1)
    Tin m[NW], v[NW]; double g;
    load_raw(L - 1 - i, m, v, g);
    to_frame(L - 1 - i, m, v, wt[i], wm[i]);
    wg[i] = g;
  }
  Tin rm[PF][NW], rv[PF][NW];
  double rg[PF];
#pragma unroll
  for (int j = 0; j < PF; ++j) load_raw(L + j, rm[j], rv[j], rg[j]);

  double vcol[S + 1][S + 1], lcol[S + 1][S + 1], zz[S + 1];
  double zo[S + 1];  // VJP: zz of the second right-hand side, o
#pragma unroll
  for (int k = 0; k <= S; ++k) {
    zz[k] = 0.0;
    zo[k] = 0.0;
#pragma unroll
    for (int j = 0; j <= S; ++j) { vcol[k][j] = 0.0; lcol[k][j] = 0.0; }
  }
  double iv1 = 0.0;
  bool reported = false;
  double sld = 0.0;  // TLL: sum_t log d_t

  for (int t0 = 0; t0 < T; t0 += PF) {
#pragma unroll
    for (int jj = 0; jj < PF; ++jj) {
      const int t = t0 + jj;
      if (t < T) {
        // slide the frame window and take frame t+L from the prefetch ring; refill the ring
#pragma unroll
        for (int i = NT - 1; i > 0; --i) {
          wg[i] = wg[i - 1];
#pragma unroll
          for (int w = 0; w < NW; ++w) { wt[i][w] = wt[i - 1][w]; wm[i][w] = wm[i - 1][w]; }
        }
        to_frame(t + L, rm[jj], rv[jj], wt[0], wm[0]);
        wg[0] = rg[jj];
        load_raw(t + L + PF, rm[jj], rv[jj], rg[jj]);

        // row t of P (acc[m] = P[t][t+m]) and of b
        double acc[S + 1];
#pragma unroll
        for (int m = 0; m <= S; ++m) {
          double a = 0.0;
#pragma unroll
          for (int w = 0; w < NW; ++w)
#pragma unroll
            for (int i = 0; i + m < NT; ++i) a = fma(p.win.q[w][m][i], wt[i][w], a);
          acc[m] = a;
        }
        double bb;
        if (FWDLIKE) {
          bb = 0.0;
#pragma unroll
          for (int w = 0; w < NW; ++w)
#pragma unroll
            for (int i = 0; i < NT; ++i) bb = fma(p.win.c[w][i], wm[i][w], bb);
        } else {
          bb = wg[L];
        }
        double bo = 0.0;
        if constexpr (VJP) bo = wg[L];
        // eliminate: older columns first (their normalised entries are ready) ...
#pragma unroll
        for (int k = 2; k <= S; ++k) {
#pragma unroll
          for (int m = 0; m + k <= S; ++m) acc[m] = fma(-vcol[k][k + m], lcol[k][k], acc[m]);
          bb = fma(-lcol[k][k], zz[k], bb);
          if constexpr (VJP) bo = fma(-lcol[k][k], zo[k], bo);
        }
        // ... the newest column last: only this part waits on the previous pivot's reciprocal
        if (S >= 1) {
#pragma unroll
          for (int m = 0; m + 1 <= S; ++m) acc[m] = fma(-(vcol[1][1 + m] * vcol[1][1]), iv1, acc[m]);
          bb = fma(-(vcol[1][1] * zz[1]), iv1, bb);
          if constexpr (VJP) bo = fma(-(vcol[1][1] * zo[1]), iv1, bo);
        }
        const double d = acc[0];
        if (!(d > 0.0) && solve && !reported) {  // linalg.pyx:79-82
          reported = true;
          report_not_pd(p.status, utt, chain, t + 1);
        }
        const double ivd = __drcp_rn(d);
        double* wsp = ws + (size_t)t * (NTS * 32);
        wsp[0] = bb * ivd;
        if (MODE == MODE_GV) wsp[NT * 32] = d;
        if constexpr (TGRAD) wsp[NT * 32] = ivd;
        if constexpr (TLL) sld += log(d);
        if constexpr (MODE == MODE_SAMPLE) wsp[NT * 32] = sqrt(ivd);
        if constexpr (VJP) wsp[NT * 32] = bo * ivd;
#pragma unroll
        for (int k = S; k >= 2; --k) {
          zz[k] = zz[k - 1];
          if constexpr (VJP) zo[k] = zo[k - 1];
#pragma unroll
          for (int j = 0; j <= S; ++j) { vcol[k][j] = vcol[k - 1][j]; lcol[k][j] = lcol[k - 1][j]; }
        }
        if (S >= 1) {
          zz[1] = bb;
          if constexpr (VJP) zo[1] = bo;
#pragma unroll
          for (int j = 1; j <= S; ++j) {
            vcol[1][j] = acc[j];
            const double lj = acc[j] * ivd;
            lcol[1][j] = lj;
            wsp[j * 32] = lj;
          }
          iv1 = ivd;
        }
      }
    }
  }

  // ---- backward sweep ----------------------------------------------------------------------------
  double yw[S + 1];  // yw[j] = y[t + j]
#pragma unroll
  for (int j = 0; j <= S; ++j) yw[j] = 0.0;
  double rz[PF], rl[PF][S + 1];
  auto load_ws = [&](int t, double& z, double(&l)[S + 1]) {
    z = 0.0;
#pragma unroll
    for (int j = 0; j <= S; ++j) l[j] = 0.0;
    if (t >= 0) {
      const double* wsp = ws + (size_t)t * (NTS * 32);
      z = wsp[0];
#pragma unroll
      for (int j = 1; j <= S; ++j) l[j] = wsp[j * 32];
    }
  };
#pragma unroll
  for (int j = 0; j < PF; ++j) load_ws(T - 1 - j, rz[j], rl[j]);

  // TLL state: windows of the targets (xw[j] = x[t + j]) and of dl/dmu (gw[i][w] = row t + L + i), the Sigma
  // block, the prefetch rings of x and 1 / d, the quadratic term of l and the global-variance gradient sums
  double xw[S + 1], gw[S + 1][NW], sg[S + 1][S + 1], rx[PF], rdi[PF], qll = 0.0, vsum[NW];
  auto load_tll = [&](int t, double& x, double& di) {
    x = 0.0; di = 0.0;
    if constexpr (TLL) {
      if (t >= 0 && solve) {
        x = (double)ld_stream(p.targets + (orow0 + t) * p.tgt_ld + ch.out_col);
        if constexpr (TGRAD) di = ws[(size_t)t * (NTS * 32) + NT * 32];
      }
    }
  };
  if constexpr (TLL) {
#pragma unroll
    for (int j = 0; j <= S; ++j) {
      xw[j] = 0.0;
#pragma unroll
      for (int w = 0; w < NW; ++w) gw[j][w] = 0.0;
#pragma unroll
      for (int k = 0; k <= S; ++k) sg[j][k] = 0.0;
    }
#pragma unroll
    for (int w = 0; w < NW; ++w) vsum[w] = 0.0;
#pragma unroll
    for (int j = 0; j < PF; ++j) load_tll(T - 1 - j, rx[j], rdi[j]);
  }
  // VJP state: the window of g = P^-1 o (gq[j] = g[t + j]) and the prefetch ring of (L^-1 o)_t / d_t
  double gq[S + 1], rgo[PF];
  if constexpr (VJP) {
#pragma unroll
    for (int j = 0; j <= S; ++j) gq[j] = 0.0;
#pragma unroll
    for (int w = 0; w < NW; ++w) vsum[w] = 0.0;
#pragma unroll
    for (int j = 0; j < PF; ++j) rgo[j] = T - 1 - j >= 0 ? ws[(size_t)(T - 1 - j) * (NTS * 32) + NT * 32] : 0.0;
  }

  // MODE_SAMPLE runs its own sweeps (sample_sweeps, below) instead of this one
  const int t_end = (MODE == MODE_GRAD || MODE == MODE_TLL || VJP) ? -L : (MODE == MODE_TLL_GRAD) ? -S
                    : (MODE == MODE_SAMPLE) ? T : 0;
  for (int t0 = T - 1; t0 >= t_end; t0 -= PF) {
#pragma unroll
    for (int jj = 0; jj < PF; ++jj) {
      const int t = t0 - jj;
      if (t >= t_end) {
#pragma unroll
        for (int j = S; j > 0; --j) yw[j] = yw[j - 1];
        double y = rz[jj];
#pragma unroll
        for (int j = 1; j <= S; ++j) y = fma(-rl[jj][j], yw[j], y);
        if (t < 0) y = 0.0;
        yw[0] = y;
        if constexpr (VJP) {  // the same back substitution for g, before the ring slot is refilled
#pragma unroll
          for (int j = S; j > 0; --j) gq[j] = gq[j - 1];
          double g = rgo[jj];
#pragma unroll
          for (int j = 1; j <= S; ++j) g = fma(-rl[jj][j], gq[j], g);
          gq[0] = t < 0 ? 0.0 : g;
          rgo[jj] = t - PF >= 0 ? ws[(size_t)(t - PF) * (NTS * 32) + NT * 32] : 0.0;
        }
        double lt[S + 1];  // TLL_GRAD: l_k[t], before the ring slot is refilled
        if constexpr (TGRAD) {
#pragma unroll
          for (int k = 1; k <= S; ++k) lt[k] = rl[jj][k];
        }
        load_ws(t - PF, rz[jj], rl[jj]);
        if constexpr (TLL) {
#pragma unroll
          for (int j = S; j > 0; --j) xw[j] = xw[j - 1];
          xw[0] = rx[jj];
          double di = rdi[jj];
          load_tll(t - PF, rx[jj], rdi[jj]);
          if constexpr (TGRAD) {
            // Sigma block of rows t .. t + S from that of rows t + 1 .. t + S + 1 (zero past T, and for t < 0,
            // where l and 1 / d load as zero)
#pragma unroll
            for (int a = S; a > 0; --a)
#pragma unroll
              for (int b = S; b >= a; --b) sg[a][b] = sg[a - 1][b - 1];
#pragma unroll
            for (int j = 1; j <= S; ++j) {
              double s = 0.0;
#pragma unroll
              for (int k = 1; k <= S; ++k) s = fma(-lt[k], sym_at<S>(sg, k, j), s);
              sg[0][j] = s;
            }
#pragma unroll
            for (int k = 1; k <= S; ++k) di = fma(-lt[k], sg[0][k], di);
            sg[0][0] = di;
          }
          // row r = t + L
          const int r = t + L;
          double gr[NW];
#pragma unroll
          for (int w = 0; w < NW; ++w) gr[w] = 0.0;
          if (r >= 0 && r < T && solve) {
            Tin m[NW], v[NW];
            double tau[NW], tm[NW];
#pragma unroll
            for (int w = 0; w < NW; ++w) { m[w] = Tin(0); v[w] = Tin(1); }
#pragma unroll
            for (int w = 0; w < NW; ++w)
              if (w < nw) {
                if constexpr (TGRAD) m[w] = mptr[(int64_t)r * p.in_ld + w * ch.win_stride];
                v[w] = var_global ? gv[w] : vptr[(int64_t)r * p.var_ld + w * ch.win_stride];
              }
            to_frame(r, m, v, tau, tm);
#pragma unroll
            for (int w = 0; w < NW; ++w) {
              if (w < nw) {
                double ux = 0.0, uc = 0.0;
#pragma unroll
                for (int i = 0; i < NT; ++i) {  // c[w][L+k], k = i-L: frames r + k = t + i
                  ux = fma(p.win.c[w][i], xw[i], ux);
                  uc = fma(p.win.c[w][i], yw[i], uc);
                }
                const double e = ux - uc;
                const double g = tau[w] * e;
                qll = fma(g, e, qll);
                if constexpr (TGRAD) {
                  gr[w] = g;
                  double wsw = 0.0;  // w_r^T Sigma w_r = sum_m (2 - [m == 0]) sum_i q[w][m][i] Sigma[t+i][t+i+m]
#pragma unroll
                  for (int mm = S; mm >= 1; --mm) {
#pragma unroll
                    for (int i = 0; i + mm < NT; ++i) wsw = fma(p.win.q[w][mm][i], sg[i][i + mm], wsw);
                  }
                  wsw *= 2.0;
#pragma unroll
                  for (int i = 0; i < NT; ++i) wsw = fma(p.win.q[w][0][i], sg[i][i], wsw);
                  const double mu = (double)m[w];
                  const double dx = ux - mu, dc = uc - mu;
                  const double gvr = -0.5 * tau[w] * tau[w] * (wsw - dx * dx + dc * dc);
                  const int64_t col = ch.in_col + w * ch.win_stride;
                  p.grad_means[(row0 + r) * p.gm_ld + col] = (Tin)g;
                  if (var_global) vsum[w] += gvr;
                  else reinterpret_cast<Tin*>(p.grad_vars)[(row0 + r) * p.gv_ld + col] = (Tin)gvr;
                }
              }
            }
          }
          if constexpr (TGRAD) {
            // dl/dx at frame s = t + S: -sum_w sum_i c[w][S - i] dl/dmu[row t + L + i][w]
#pragma unroll
            for (int i = S; i > 0; --i)
#pragma unroll
              for (int w = 0; w < NW; ++w) gw[i][w] = gw[i - 1][w];
#pragma unroll
            for (int w = 0; w < NW; ++w) gw[0][w] = gr[w];
            const int s = t + S;
            if (s >= 0 && s < T && solve) {
              double gx = 0.0;
#pragma unroll
              for (int w = 0; w < NW; ++w)
#pragma unroll
                for (int i = 0; i <= S; ++i) gx = fma(p.win.c[w][S - i], gw[i][w], gx);
              p.grad_targets[(orow0 + s) * p.gx_ld + ch.out_col] = (Tin)(-gx);
            }
          }
        } else if constexpr (VJP) {
          const int r = t + L;  // >= 0
          if (r < T && solve) {
            Tin m[NW], v[NW];
            double tau[NW], tm[NW];
#pragma unroll
            for (int w = 0; w < NW; ++w) { m[w] = Tin(0); v[w] = Tin(1); }
#pragma unroll
            for (int w = 0; w < NW; ++w)
              if (w < nw) {
                m[w] = mptr[(int64_t)r * p.in_ld + w * ch.win_stride];
                v[w] = var_global ? gv[w] : vptr[(int64_t)r * p.var_ld + w * ch.win_stride];
              }
            to_frame(r, m, v, tau, tm);
#pragma unroll
            for (int w = 0; w < NW; ++w) {
              if (w < nw) {
                double ug = 0.0, uc = 0.0;
#pragma unroll
                for (int i = 0; i < NT; ++i) {  // c[w][L+k], k = i-L: frames r + k = t + i
                  ug = fma(p.win.c[w][i], gq[i], ug);
                  uc = fma(p.win.c[w][i], yw[i], uc);
                }
                const double gm = tau[w] * ug;
                const double gvr = -tau[w] * gm * ((double)m[w] - uc);
                const int64_t col = ch.in_col + w * ch.win_stride;
                p.grad_means[(row0 + r) * p.gm_ld + col] = (Tin)gm;
                if (var_global) vsum[w] += gvr;
                else reinterpret_cast<Tin*>(p.grad_vars)[(row0 + r) * p.gv_ld + col] = (Tin)gvr;
              }
            }
          }
        } else if (MODE == MODE_GV) {
          ws[(size_t)t * (NTS * 32) + (NT + 1) * 32] = y;  // c_m, refined below
        } else if (MODE != MODE_GRAD) {
          if (solve) st_stream(reinterpret_cast<Tin*>(p.out) + (orow0 + t) * p.out_ld + ch.out_col, (Tin)y);
        } else {
          // row r = t + L of the gradient: tau_w[r] * sum_k c[w][L+k] x[r+k],  x[r+k] = yw[L+k]
          const int r = t + L;
          if (r < T && solve) {
            Tin m[NW], v[NW];
            double tau[NW], tm[NW];
#pragma unroll
            for (int w = 0; w < NW; ++w) { m[w] = Tin(0); v[w] = Tin(1); }
#pragma unroll
            for (int w = 0; w < NW; ++w)
              if (w < nw) v[w] = var_global ? gv[w] : vptr[(int64_t)r * p.var_ld + w * ch.win_stride];
            to_frame(r, m, v, tau, tm);
#pragma unroll
            for (int w = 0; w < NW; ++w) {
              if (w < nw) {
                double s = 0.0;
#pragma unroll
                for (int i = 0; i < NT; ++i) s = fma(p.win.c[w][i], yw[i], s);  // c[w][L+k], k = i-L
                reinterpret_cast<float*>(p.out)[(orow0 + r) * p.out_ld + ch.in_col + w * ch.win_stride] =
                    (float)(tau[w] * s);
              }
            }
          }
        }
      }
    }
  }

  if constexpr (TLL) {
    if (solve) {
      constexpr double LOG_2PI = 1.8378770664093454836;
      p.ll[(int64_t)utt * p.n_chain + chain] = 0.5 * (sld - qll) - 0.5 * LOG_2PI * (double)T;
      if constexpr (TGRAD) {
        if (var_global) {
          double* gp = reinterpret_cast<double*>(p.grad_vars) + (int64_t)utt * p.gv_ld + ch.in_col;
#pragma unroll
          for (int w = 0; w < NW; ++w)
            if (w < nw) gp[w * ch.win_stride] = vsum[w];
        }
      }
    }
  }

  if constexpr (VJP) {
    if (solve && var_global) {
      double* gp = reinterpret_cast<double*>(p.grad_vars) + (int64_t)utt * p.gv_ld + ch.in_col;
#pragma unroll
      for (int w = 0; w < NW; ++w)
        if (w < nw) gp[w * ch.win_stride] = vsum[w];
    }
  }

  if constexpr (MODE == MODE_SAMPLE) {
    if (solve)
      sample_sweeps<S, NTS, PF>(ws, T, p.n_samples, p.sample_stride, (uint32_t)ch.out_col,
                                p.keys ? p.keys[utt] : (uint32_t)utt, p.seed, p.scale,
                                reinterpret_cast<Tin*>(p.out) + orow0 * p.out_ld + ch.out_col, p.out_ld);
  }

  if constexpr (MODE == MODE_GV) {
    if (solve) {
      Tin* o = reinterpret_cast<Tin*>(p.out) + orow0 * p.out_ld + ch.out_col;
      gv_refine<S, NTS>(ws, T, p.gv_mean[ch.out_col], 1.0 / p.gv_var[ch.out_col],
                        p.gv_weight > 0.0 ? p.gv_weight : 1.0 / ((double)nw * (double)T), p.gv_n_iter, p.gv_step,
                        o, p.out_ld);
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------------
template <int NW, int L, int U>
static bool fill_wintab(const nnk_windows_t& w, WinTab<NW, L, U>& tab) {
  constexpr int NT = L + U + 1, S = L + U;
  if (w.nw < 1 || w.nw > NW) return false;
  int m_edge = 0;
  for (int i = 0; i < NW; ++i)
    for (int j = 0; j < NT; ++j) tab.c[i][j] = 0.0;
  for (int i = 0; i < w.nw; ++i) {
    if (w.l[i] < 0 || w.u[i] < 0 || w.l[i] > L || w.u[i] > U) return false;
    for (int k = -w.l[i]; k <= w.u[i]; ++k) tab.c[i][L + k] = w.coef[i][w.l[i] + k];
    m_edge = w.l[i] > m_edge ? w.l[i] : m_edge;
    m_edge = w.u[i] > m_edge ? w.u[i] : m_edge;
  }
  for (int i = 0; i < NW; ++i)
    for (int m = 0; m <= S; ++m)
      for (int j = 0; j < NT; ++j) tab.q[i][m][j] = (j + m < NT) ? tab.c[i][j] * tab.c[i][j + m] : 0.0;
  tab.nw = w.nw;
  tab.m_edge = m_edge;
  return true;
}

static void win_extent(const nnk_windows_t& w, int& L, int& U) {
  L = 0; U = 0;
  for (int i = 0; i < w.nw && i < NNK_MAX_WIN; ++i) {
    L = w.l[i] > L ? w.l[i] : L;
    U = w.u[i] > U ? w.u[i] : U;
  }
}

// which template instance serves a window set: returns S (band depth of the instance) or -1
static int pick_instance(const nnk_windows_t& w, int& inst) {
  if (w.nw < 1 || w.nw > NNK_MAX_WIN) return -1;
  int L, U;
  win_extent(w, L, U);
  if (L > NNK_MAX_HALF || U > NNK_MAX_HALF) return -1;
  if (w.nw == 1 && L == 0 && U == 0) { inst = 0; return 0; }
  if (w.nw <= 3 && L <= 1 && U <= 1) { inst = 1; return 2; }
  if (w.nw <= 3 && L <= 2 && U <= 2) { inst = 2; return 4; }
  inst = 3;
  return 2 * NNK_MAX_HALF;
}

static bool is_std_windows(const nnk_windows_t& w) {
  if (w.nw != 3 || w.l[0] != 0 || w.u[0] != 0 || w.l[1] != 1 || w.u[1] != 1 || w.l[2] != 1 || w.u[2] != 1) return false;
  return w.coef[0][0] == 1.0 && w.coef[1][0] == -0.5 && w.coef[1][1] == 0.0 && w.coef[1][2] == 0.5 &&
         w.coef[2][0] == 1.0 && w.coef[2][1] == -2.0 && w.coef[2][2] == 1.0;
}

// one launch of the staged kernel with G chain groups per CTA; the standard window set (STD: closed-form band
// rows) and global (D,) variances (VARG) are template parameters
template <typename Tin, int NW, int L, int U, int MODE, int NSA, int G>
static int launch_as(const MlpgParams<Tin, NW, L, U>& p, const AsGeom& g, size_t smem, int grid, bool stdw, bool varg,
                     cudaStream_t st) {
  constexpr bool CAN_STD = (NW == 3 && L == 1 && U == 1);
  constexpr int NSB = (MODE == MODE_GRAD) ? 4 : 8;
#define NNK_LAUNCH_AS(STDV, VARGV)                                                                                \
  do {                                                                                                           \
    auto kern = mlpg_fwd_as_kernel<Tin, NW, L, U, STDV, VARGV, MODE, AS_TT, AS_NA, NSA, AS_ND, AS_TTB, NSB, G>; \
    NNK_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));        \
    kern<<<grid, 32 * G * (AS_NA + 1), smem, st>>>(p, g);                                                       \
  } while (0)
  if (stdw && !varg) NNK_LAUNCH_AS(CAN_STD, false);
  else if (stdw && varg) NNK_LAUNCH_AS(CAN_STD, true);
  else if (!varg) NNK_LAUNCH_AS(false, false);
  else NNK_LAUNCH_AS(false, true);
#undef NNK_LAUNCH_AS
  return NNK_OK;
}

template <typename Tin, int NW, int L, int U, int MODE>
static int launch_mlpg(const nnk_mlpg_args_t& a, const nnk_mlpg_gv_t* gv, cudaStream_t st,
                       const nnk_traj_ll_t* tl = nullptr, const nnk_traj_sample_t* ts = nullptr,
                       const nnk_mlpg_vjp_t* vj = nullptr) {
  constexpr int NT = L + U + 1;
  constexpr int NTS = WsCols<MODE, NT>::value;
  constexpr int PF = (L + U <= 2) ? 4 : 2;
  constexpr int ES = (int)sizeof(Tin);
  constexpr bool GRAD = (MODE == MODE_GRAD);
  typename KernelParams<Tin, NW, L, U, MODE>::type p;
  if constexpr (MODE == MODE_TLL || MODE == MODE_TLL_GRAD) {
    p.targets = (const Tin*)tl->targets; p.tgt_ld = tl->tgt_ld; p.ll = tl->ll;
    p.grad_means = (Tin*)tl->grad_means; p.gm_ld = tl->gm_ld;
    p.grad_vars = tl->grad_vars; p.gv_ld = tl->gv_ld;
    p.grad_targets = (Tin*)tl->grad_targets; p.gx_ld = tl->gx_ld;
  }
  if constexpr (MODE == MODE_SAMPLE) {
    p.sample_stride = ts->sample_stride; p.n_samples = ts->n_samples; p.seed = ts->seed; p.keys = ts->keys;
    p.scale = ts->scale;
  }
  if (!fill_wintab<NW, L, U>(a.win, p.win)) { set_error("window set does not fit kernel instance"); return NNK_ERR_UNSUPPORTED; }
  p.means = (const Tin*)a.means; p.vars = (const Tin*)a.vars; p.go = a.grad_out; p.go_f64 = a.go_f64; p.out = a.out;
  p.in_ld = a.in_ld; p.var_ld = a.var_ld; p.go_ld = a.go_ld; p.out_ld = a.out_ld;
  p.utt_off = a.utt_off; p.out_off = a.out_off; p.utt_len = a.utt_len; p.order = a.order; p.chains = a.chains;
  p.n_utt = a.n_utt; p.n_chain = a.n_chain; p.n_groups = (a.n_chain + 31) / 32; p.max_T = a.max_T;
  p.ws = (double*)a.workspace; p.status = (unsigned long long*)a.status_word;
  p.gv_mean = gv ? gv->gv_mean : nullptr; p.gv_var = gv ? gv->gv_var : nullptr;
  p.gv_step = gv ? gv->step : 0.0; p.gv_weight = gv ? gv->weight : 0.0; p.gv_n_iter = gv ? gv->n_iter : 0;
  if constexpr (MODE == MODE_VJP) {  // grad_out is of Tin and read at the output's rows and columns
    p.go = vj->grad_out; p.go_ld = vj->go_ld; p.go_f64 = 0;
    p.grad_means = (Tin*)vj->grad_means; p.gm_ld = vj->gm_ld; p.grad_vars = vj->grad_vars; p.gv_ld = vj->gv_ld;
  }
  const size_t per_item = (size_t)a.max_T * NTS * 32 * sizeof(double);
  size_t items_cap = per_item ? a.workspace_bytes / per_item : 0;
  int utt_per_launch = (int)(items_cap / (size_t)p.n_groups);
  if (utt_per_launch < 1) { set_error("workspace too small: need >= %zu bytes", per_item * p.n_groups); return NNK_ERR_WORKSPACE; }
  // The staged kernel serves forward solves and gradients with a float32 grad_out (what autograd hands over)
  // when the window set fills the instance (nw == NW) and the rows fit as_geometry's rings.  It is compiled only
  // for NT <= 5 and never for nnk_mlpg_solve or nnk_mlpg_gv; everything else runs mlpg_kernel.
  constexpr bool CAN_AS = (MODE == MODE_FWD || MODE == MODE_GRAD) && (NT <= 5);
  // float32 forward solves with two or more chain groups: one CTA per pair of groups (an odd last group runs
  // with an empty second half), when that geometry fits two CTAs per SM.  Float64 rows and the gradient keep
  // one group per CTA, and so do band depths S > 2: at the 128 registers of two 256-thread CTAs per SM the
  // S = 4 assembler spills.
  constexpr bool CAN_G2 = CAN_AS && (MODE == MODE_FWD) && (ES == 4) && (NT <= 3);
  constexpr int NSB = GRAD ? 4 : 8;
  AsGeom geom, geom2;
  size_t smem = 0, smem2 = 0;
  bool staged = false, grouped = false;
  if constexpr (CAN_AS) {
    staged = (a.win.nw == NW) && !(GRAD && a.go_f64) &&
             as_geometry<AS_TT, AS_NA, AS_NSA1, AS_ND, AS_TTB, NSB>(GRAD ? a.go_ld * 4 : a.in_ld * ES, a.var_ld * ES, GRAD,
                                                                    L, NT, ES, geom, smem);
    if constexpr (CAN_G2)
      grouped = staged && p.n_groups >= 2 &&
                as_geometry<AS_TT, AS_NA, AS_NSA2, AS_ND, AS_TTB, NSB, 2>(a.in_ld * ES, a.var_ld * ES, false, L, NT, ES,
                                                                          geom2, smem2);
  }
  const bool stdw = (NW == 3 && L == 1 && U == 1) && is_std_windows(a.win);
  const bool varg = (a.var_ld == 0);
  for (int u0 = 0; u0 < a.n_utt; u0 += utt_per_launch) {
    const int nu = (a.n_utt - u0 < utt_per_launch) ? a.n_utt - u0 : utt_per_launch;
    p.urank0 = u0;
    if (!staged) {
      mlpg_kernel<Tin, NW, L, U, MODE, PF><<<nu * p.n_groups, 32, 0, st>>>(p);
    } else if constexpr (CAN_AS) {
      int r;
      if constexpr (CAN_G2)
        r = grouped ? launch_as<Tin, NW, L, U, MODE, AS_NSA2, 2>(p, geom2, smem2, nu * ((p.n_groups + 1) / 2), stdw, varg, st)
                    : launch_as<Tin, NW, L, U, MODE, AS_NSA1, 1>(p, geom, smem, nu * p.n_groups, stdw, varg, st);
      else
        r = launch_as<Tin, NW, L, U, MODE, AS_NSA1, 1>(p, geom, smem, nu * p.n_groups, stdw, varg, st);
      if (r != NNK_OK) return r;
    }
    count_launch();
    NNK_CUDA_CHECK(cudaGetLastError());
  }
  return NNK_OK;
}

template <typename Tin, int MODE>
static int dispatch_inst(const nnk_mlpg_args_t& a, cudaStream_t st, const nnk_mlpg_gv_t* gv = nullptr,
                         const nnk_traj_ll_t* tl = nullptr, const nnk_traj_sample_t* ts = nullptr,
                         const nnk_mlpg_vjp_t* vj = nullptr) {
  int inst = -1;
  if (pick_instance(a.win, inst) < 0) {
    set_error("unsupported window set: nw=%d (max %d) or half-width > %d", a.win.nw, NNK_MAX_WIN, NNK_MAX_HALF);
    return NNK_ERR_UNSUPPORTED;
  }
  switch (inst) {
    case 0: return launch_mlpg<Tin, 1, 0, 0, MODE>(a, gv, st, tl, ts, vj);
    case 1: return launch_mlpg<Tin, 3, 1, 1, MODE>(a, gv, st, tl, ts, vj);
    case 2: return launch_mlpg<Tin, 3, 2, 2, MODE>(a, gv, st, tl, ts, vj);
    default: return launch_mlpg<Tin, NNK_MAX_WIN, NNK_MAX_HALF, NNK_MAX_HALF, MODE>(a, gv, st, tl, ts, vj);
  }
}

static int check_args(const nnk_mlpg_args_t* a, bool grad) {
  NNK_REQUIRE(a != nullptr, NNK_ERR_ARG, "args is NULL");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(a->n_utt >= 0 && a->n_chain >= 0 && a->max_T >= 0, NNK_ERR_ARG, "negative size");
  NNK_REQUIRE(a->n_chain < (1 << 21) && a->max_T < (1 << 21) - 1 && a->n_utt < (1 << 22), NNK_ERR_ARG, "size exceeds status key range");
  if (a->n_utt == 0 || a->n_chain == 0 || a->max_T == 0) return 1;  // nothing to do
  NNK_REQUIRE(a->vars && a->out && a->utt_off && a->chains && a->status_word, NNK_ERR_ARG, "NULL device pointer");
  NNK_REQUIRE(grad ? a->grad_out != nullptr : a->means != nullptr, NNK_ERR_ARG, "NULL input pointer");
  NNK_REQUIRE(a->workspace != nullptr, NNK_ERR_WORKSPACE, "NULL workspace");
  return 0;
}

}  // namespace nnk

using namespace nnk;

static size_t workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win, int extra_cols) {
  int inst = -1;
  if (!win) return 0;
  const int S = pick_instance(*win, inst);
  if (S < 0) return 0;
  const size_t groups = (size_t)((n_chain + 31) / 32);
  return (size_t)n_utt * groups * (size_t)max_T * (size_t)(S + 1 + extra_cols) * 32 * sizeof(double);
}

extern "C" size_t nnk_mlpg_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win) {
  return workspace_bytes(n_utt, n_chain, max_T, win, 0);
}

extern "C" size_t nnk_mlpg_gv_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win) {
  return workspace_bytes(n_utt, n_chain, max_T, win, WsCols<MODE_GV, 0>::value);
}

extern "C" size_t nnk_mlpg_traj_ll_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T,
                                                   const nnk_windows_t* win) {
  return workspace_bytes(n_utt, n_chain, max_T, win, WsCols<MODE_TLL, 0>::value);
}

extern "C" size_t nnk_mlpg_traj_sample_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T,
                                                       const nnk_windows_t* win) {
  return workspace_bytes(n_utt, n_chain, max_T, win, WsCols<MODE_SAMPLE, 0>::value);
}

extern "C" size_t nnk_mlpg_vjp_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win) {
  return workspace_bytes(n_utt, n_chain, max_T, win, WsCols<MODE_VJP, 0>::value);
}

#ifdef NNK_AS_PROF
// debug builds only: read and clear the NNK_AS_PROF_SLOTS phase counters of mlpg_fwd_as_kernel (synchronises)
extern "C" int nnk_as_prof_read(unsigned long long* out) {
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out, nnk::g_as_prof, sizeof(unsigned long long) * NNK_AS_PROF_SLOTS);
  unsigned long long z[NNK_AS_PROF_SLOTS] = {0};
  cudaMemcpyToSymbol(nnk::g_as_prof, z, sizeof(z));
  return 0;
}
#endif

extern "C" int nnk_mlpg_fwd(const nnk_mlpg_args_t* a, void* stream) {
  int r = check_args(a, false);
  if (r < 0) return r;
  if (r > 0) return NNK_OK;
  DeviceGuard guard(a->out);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_FWD>(*a, st) : dispatch_inst<double, MODE_FWD>(*a, st);
}

extern "C" int nnk_mlpg_solve(const nnk_mlpg_args_t* a, void* stream) {
  int r = check_args(a, true);
  if (r < 0) return r;
  if (r > 0) return NNK_OK;
  DeviceGuard guard(a->out);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_SOLVE>(*a, st) : dispatch_inst<double, MODE_SOLVE>(*a, st);
}

extern "C" int nnk_mlpg_grad(const nnk_mlpg_args_t* a, void* stream) {
  int r = check_args(a, true);
  if (r < 0) return r;
  if (r > 0) return NNK_OK;
  DeviceGuard guard(a->out);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_GRAD>(*a, st) : dispatch_inst<double, MODE_GRAD>(*a, st);
}

extern "C" int nnk_mlpg_gv(const nnk_mlpg_args_t* a, const nnk_mlpg_gv_t* gv, void* stream) {
  int r = check_args(a, false);
  if (r < 0) return r;
  NNK_REQUIRE(gv != nullptr, NNK_ERR_ARG, "gv is NULL");
  NNK_REQUIRE(gv->n_iter >= 0, NNK_ERR_ARG, "n_iter must be >= 0");
  NNK_REQUIRE(gv->step > 0.0, NNK_ERR_ARG, "step must be > 0");
  NNK_REQUIRE(!(gv->weight < 0.0) && gv->weight == gv->weight, NNK_ERR_ARG, "weight must be > 0 (or 0 for 1 / (nw T))");
  if (r > 0) return NNK_OK;
  NNK_REQUIRE(gv->gv_mean && gv->gv_var, NNK_ERR_ARG, "NULL gv_mean / gv_var");
  DeviceGuard guard(a->out);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_GV>(*a, st, gv) : dispatch_inst<double, MODE_GV>(*a, st, gv);
}

extern "C" int nnk_mlpg_traj_ll(const nnk_mlpg_args_t* a, const nnk_traj_ll_t* tl, void* stream) {
  NNK_REQUIRE(a != nullptr && tl != nullptr, NNK_ERR_ARG, "args or tl is NULL");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(a->n_utt >= 0 && a->n_chain >= 0 && a->max_T >= 0, NNK_ERR_ARG, "negative size");
  NNK_REQUIRE(a->n_chain < (1 << 21) && a->max_T < (1 << 21) - 1 && a->n_utt < (1 << 22), NNK_ERR_ARG, "size exceeds status key range");
  NNK_REQUIRE(tl->grad == 0 || tl->grad == 1, NNK_ERR_ARG, "grad must be 0 or 1");
  if (a->n_utt == 0 || a->n_chain == 0 || a->max_T == 0) return NNK_OK;
  NNK_REQUIRE(a->means && a->vars && a->utt_off && a->chains && a->status_word, NNK_ERR_ARG, "NULL device pointer");
  NNK_REQUIRE(tl->targets && tl->ll, NNK_ERR_ARG, "NULL targets or ll");
  NNK_REQUIRE(!tl->grad || (tl->grad_means && tl->grad_vars && tl->grad_targets), NNK_ERR_ARG, "NULL gradient output");
  NNK_REQUIRE(a->workspace != nullptr, NNK_ERR_WORKSPACE, "NULL workspace");
  DeviceGuard guard(tl->ll);
  cudaStream_t st = (cudaStream_t)stream;
  if (tl->grad)
    return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_TLL_GRAD>(*a, st, nullptr, tl)
                               : dispatch_inst<double, MODE_TLL_GRAD>(*a, st, nullptr, tl);
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_TLL>(*a, st, nullptr, tl)
                             : dispatch_inst<double, MODE_TLL>(*a, st, nullptr, tl);
}

extern "C" int nnk_mlpg_traj_sample(const nnk_mlpg_args_t* a, const nnk_traj_sample_t* ts, void* stream) {
  NNK_REQUIRE(ts != nullptr, NNK_ERR_ARG, "ts is NULL");
  int r = check_args(a, false);
  if (r < 0) return r;
  NNK_REQUIRE(ts->n_samples >= 1, NNK_ERR_ARG, "n_samples must be >= 1");
  NNK_REQUIRE(ts->sample_stride >= 0, NNK_ERR_ARG, "sample_stride must be >= 0");
  NNK_REQUIRE(ts->scale >= 0.0 && ts->scale <= 1.7976931348623157e308, NNK_ERR_ARG, "scale must be finite and >= 0");
  if (r > 0) return NNK_OK;
  DeviceGuard guard(a->out);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_SAMPLE>(*a, st, nullptr, nullptr, ts)
                             : dispatch_inst<double, MODE_SAMPLE>(*a, st, nullptr, nullptr, ts);
}

extern "C" int nnk_mlpg_vjp(const nnk_mlpg_args_t* a, const nnk_mlpg_vjp_t* vj, void* stream) {
  NNK_REQUIRE(a != nullptr && vj != nullptr, NNK_ERR_ARG, "args or vj is NULL");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F32 or NNK_F64");
  NNK_REQUIRE(a->n_utt >= 0 && a->n_chain >= 0 && a->max_T >= 0, NNK_ERR_ARG, "negative size");
  NNK_REQUIRE(a->n_chain < (1 << 21) && a->max_T < (1 << 21) - 1 && a->n_utt < (1 << 22), NNK_ERR_ARG, "size exceeds status key range");
  NNK_REQUIRE(vj->go_ld >= 0 && vj->gm_ld >= 0 && vj->gv_ld >= 0, NNK_ERR_ARG, "negative row stride");
  if (a->n_utt == 0 || a->n_chain == 0 || a->max_T == 0) return NNK_OK;
  NNK_REQUIRE(a->means && a->vars && a->utt_off && a->chains && a->status_word, NNK_ERR_ARG, "NULL device pointer");
  NNK_REQUIRE(vj->grad_out && vj->grad_means && vj->grad_vars, NNK_ERR_ARG, "NULL grad_out or gradient output");
  NNK_REQUIRE(a->workspace != nullptr, NNK_ERR_WORKSPACE, "NULL workspace");
  DeviceGuard guard(vj->grad_means);
  cudaStream_t st = (cudaStream_t)stream;
  return a->dtype == NNK_F32 ? dispatch_inst<float, MODE_VJP>(*a, st, nullptr, nullptr, nullptr, vj)
                             : dispatch_inst<double, MODE_VJP>(*a, st, nullptr, nullptr, nullptr, vj);
}
