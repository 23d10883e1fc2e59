// nnk_ms_gen.cu -- parameter generation considering the modulation spectrum (paramgen.mlpg_ms_batch; C ABI:
// nnk_mlpg_ms and, for the segment level, nnk_mlpg_ms_segment in include/nnk_b200.h; definition in DESIGN.md 3.18).
//
// nnk_mlpg_ms chains existing pieces: nnk_mlpg_fwd gives c_m, and every trial's h = P^-1 g is one nnk_mlpg_solve
// with a float64 right-hand side.  What is new is ms_gen_kernel<LOGN, TRIAL>, one CTA per (utterance, chain):
//   TRIAL: c' = c + alpha ((c_m - c) + h / omega) from the current c (the output column), c_m and h;
//   init:  c' = c_m, copied to the output column (pass-through chains are copied and stop there).
// It evaluates F(c') = omega Q(c') + MS(c'), Q = -1/2 sum_w sum_t tau_w,t ((W_w c')_t - mu_w,t)^2 (F up to a
// constant, from a window stencil over the chain's means and variances), MS from the packed real FFT of c' in
// shared memory (nnk_fft.cuh).  The trial is kept when F(c') >= F(c): F, alpha and the output column are updated.
// Then, unless it is the last trial, the gradient of the MS term at the current c,
//   g_t = sum_{k=1}^{n/2} 2 G_k Re(Y_k e^{2 pi i k t / n}),  G_k = -q_k (s_k - nu_k) / |Y_k|^2,
// i.e. n irfft(C) with C_k = G_k Y_k (C_{n/2} doubled, C_0 = 0), goes to the solve's right-hand side.  An accepted
// trial reuses the spectrum already in shared memory; a rejected one transforms c again.  Both sums (Q and the
// MS term) are per-thread partials over a fixed index set and a fixed tree: the bits do not depend on the batch.
#include "nnk_common.cuh"
#include "nnk_fft.cuh"

namespace nnk {

constexpr int MSG_LOGN_MIN = 8, MSG_LOGN_MAX = 12;  // n = 256 .. 4096

template <int LOGN> constexpr int ms_gen_threads() { return (1 << (LOGN - 2)) < 256 ? (1 << (LOGN - 2)) : 256; }

struct MsGenParams {
  const double* means;
  const double* vars;
  int64_t in_ld, var_ld, out_ld;
  const int64_t* utt_off;
  const int32_t* utt_len;
  const nnk_chain_t* chains;
  int n_chain, nw, m_edge;
  int l[NNK_MAX_WIN], u[NNK_MAX_WIN];
  double coef[NNK_MAX_WIN][NNK_MAX_TAPS];
  const double* cm;  // (n_rows, out_ld)
  const double* h;   // (n_rows, out_ld)
  double* c;         // the output (n_rows, out_ld): the current trajectory
  double* g;         // (n_rows, n_chain)
  double* F;         // (n_utt, n_chain)
  double* alpha;     // (n_utt, n_chain)
  const double* ms_mean;
  const double* ms_var;
  double step, weight;
  int want_grad;
};

template <int LOGN, bool TRIAL>
__global__ void __launch_bounds__(ms_gen_threads<LOGN>()) ms_gen_kernel(const __grid_constant__ MsGenParams p) {
  using V = double2;
  constexpr int N = 1 << LOGN, M = N / 2, LOGM = LOGN - 1, NT = ms_gen_threads<LOGN>();
  extern __shared__ __align__(16) unsigned char msg_smem[];
  V* z = reinterpret_cast<V*>(msg_smem);
  V* tw = z + M;
  V* red = tw + M;                                  // (Q, MS) partials, NT
  double* cs = reinterpret_cast<double*>(red + NT);  // TRIAL: the current c
  double* xs = cs + (TRIAL ? N : 0);                 // c'
  const int tid = threadIdx.x;
  const int chain = (int)(blockIdx.x % (unsigned)p.n_chain), utt = (int)(blockIdx.x / (unsigned)p.n_chain);
  const int64_t row0 = p.utt_off[utt];
  const int T = p.utt_len ? p.utt_len[utt] : (int)(p.utt_off[utt + 1] - row0);
  if (T <= 0 || T > N) return;
  const nnk_chain_t ch = p.chains[chain];
  const int64_t ld = p.out_ld;
  double* c = p.c + row0 * ld + ch.out_col;
  const double* cm = p.cm + row0 * ld + ch.out_col;
  if (ch.flags & 1) {  // pass-through: nnk_mlpg_fwd copied the column into c_m
    if (!TRIAL)
      for (int t = tid; t < T; t += NT) c[t * ld] = cm[t * ld];
    return;
  }
  const size_t si = (size_t)utt * p.n_chain + chain;
  const double omega = p.weight > 0.0 ? p.weight : 1.0 / ((double)p.nw * (double)T);
  for (int j = tid; j < M; j += NT) {  // W^j = e^{-2 pi i j / n}
    double s, co;
    sincospi(double(2 * j) / double(N), &s, &co);
    tw[j] = cx<V>(co, -s);
  }
  const double alpha = TRIAL ? p.alpha[si] : p.step;
  if (TRIAL) {
    const double* h = p.h + row0 * ld + ch.out_col;
    for (int t = tid; t < T; t += NT) {
      const double ct = c[t * ld];
      cs[t] = ct;
      xs[t] = ct + alpha * ((cm[t * ld] - ct) + h[t * ld] / omega);
    }
  } else {
    for (int t = tid; t < T; t += NT) xs[t] = cm[t * ld];
  }
  auto load_fft = [&](const double* x) {  // x (T frames, zeros up to n) -> Z in natural order
    for (int t = tid; t < M; t += NT) {
      const double x0 = 2 * t < T ? x[2 * t] : 0.0, x1 = 2 * t + 1 < T ? x[2 * t + 1] : 0.0;
      z[__brev(t) >> (32 - LOGM)] = cx<V>(x0, x1);
    }
    __syncthreads();
    block_fft_dit<LOGN, NT>(z, tw, tid);
  };
  __syncthreads();
  // Q(c'): tau with nnk_mlpg_fwd's edge rule (dynamic windows have no precision on the first and last m_edge
  // frames, and on every frame when m_edge == 0)
  double q = 0.0;
  const double* mrow = p.means + row0 * p.in_ld + ch.in_col;
  const double* vrow = p.vars + (p.var_ld ? row0 * p.var_ld : 0) + ch.in_col;
  for (int t = tid; t < T; t += NT) {
    const bool edge = p.m_edge == 0 || t < p.m_edge || t >= T - p.m_edge;
    for (int w = 0; w < p.nw; ++w) {
      if (w > 0 && edge) continue;
      const int64_t col = (int64_t)w * ch.win_stride;
      const double tau = 1.0 / vrow[p.var_ld ? t * p.var_ld + col : col];
      double e = -mrow[t * p.in_ld + col];
      for (int k = -p.l[w]; k <= p.u[w]; ++k)
        if (t + k >= 0 && t + k < T) e = fma(p.coef[w][p.l[w] + k], xs[t + k], e);
      q = fma(tau * e, e, q);
    }
  }
  // the MS term of c'
  load_fft(xs);
  const double* nu = p.ms_mean + ch.out_col;
  const double* vv = p.ms_var + ch.out_col;
  auto bin_term = [&](V y, int k) {
    const double qk = 1.0 / vv[k * ld];
    if (qk == 0.0) return 0.0;
    const double d = log_power(y.x * y.x + y.y * y.y) - nu[k * ld];
    return qk * d * d;
  };
  double ms = 0.0;
  for (int k = tid; k <= M / 2; k += NT) {
    V Yk, Yj;
    rfft_bin_pair(z, tw, k, M, Yk, Yj);
    if (k > 0) ms += bin_term(Yk, k);
    if (M - k != k) ms += bin_term(Yj, M - k);
  }
  red[tid] = cx<V>(q, ms);
  __syncthreads();
#pragma unroll
  for (int s = NT / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] = cadd(red[tid], red[tid + s]);
    __syncthreads();
  }
  const double f2 = omega * (-0.5 * red[0].x) - 0.5 * red[0].y;
  const bool accept = !TRIAL || f2 >= p.F[si];
  __syncthreads();  // every thread has read F before thread 0 rewrites it
  if (tid == 0) {
    if (accept) p.F[si] = f2;
    p.alpha[si] = accept ? alpha : 0.5 * alpha;
  }
  if (accept)
    for (int t = tid; t < T; t += NT) c[t * ld] = xs[t];
  if (!p.want_grad) return;
  if (!accept) {
    __syncthreads();  // z is rewritten
    load_fft(cs);
  }
  // C_k = G_k Y_k, in place: each thread owns its pairs (k, M - k)
  auto grad_bin = [&](V y, int k) {
    const double qk = 1.0 / vv[k * ld], pw = y.x * y.x + y.y * y.y;
    if (qk == 0.0 || !(pw > DBL_MIN)) return cx<V>(0, 0);
    return scale(y, -qk * (log(pw) - nu[k * ld]) / pw * (k == M ? 2.0 : 1.0));
  };
  for (int k = tid; k <= M / 2; k += NT) {
    V Yk, Yj;
    rfft_bin_pair(z, tw, k, M, Yk, Yj);
    rfft_pack_pair(z, tw, k, M, k == 0 ? cx<V>(0, 0) : grad_bin(Yk, k), grad_bin(Yj, M - k));
  }
  __syncthreads();
  block_ifft_dif<LOGN, NT>(z, tw, tid);
  double* g = p.g + row0 * p.n_chain + chain;
  for (int t = tid; t < T; t += NT) {
    const V v = z[__brev(t >> 1) >> (32 - LOGM)];
    g[(int64_t)t * p.n_chain] = (t & 1) ? v.y : v.x;
  }
}

template <int LOGN, bool TRIAL> static size_t ms_gen_smem() {
  return (size_t)(2 * (1 << (LOGN - 1)) + ms_gen_threads<LOGN>()) * sizeof(double2) +
         (size_t)(TRIAL ? 2 : 1) * (1 << LOGN) * sizeof(double);
}

template <int LOGN, bool TRIAL>
static int launch_ms_gen(const MsGenParams& p, unsigned n_blocks, cudaStream_t st) {
  const size_t smem = ms_gen_smem<LOGN, TRIAL>();
  if (smem > 48 * 1024)  // per device: cheap enough to set on every launch
    NNK_CUDA_CHECK(cudaFuncSetAttribute(ms_gen_kernel<LOGN, TRIAL>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)smem));
  ms_gen_kernel<LOGN, TRIAL><<<n_blocks, ms_gen_threads<LOGN>(), smem, st>>>(p);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <bool TRIAL>
static int dispatch_ms_gen(int logn, const MsGenParams& p, unsigned n_blocks, cudaStream_t st) {
  switch (logn) {
    case 8: return launch_ms_gen<8, TRIAL>(p, n_blocks, st);
    case 9: return launch_ms_gen<9, TRIAL>(p, n_blocks, st);
    case 10: return launch_ms_gen<10, TRIAL>(p, n_blocks, st);
    case 11: return launch_ms_gen<11, TRIAL>(p, n_blocks, st);
    default: return launch_ms_gen<12, TRIAL>(p, n_blocks, st);
  }
}

// ---- the segment-level MS term (nnk_mlpg_ms_segment) --------------------------------------------------------------
// ms_gen_segment_kernel<LOGN, TRIAL> does ms_gen_kernel's job for the segment-level term, one CTA of 256 threads
// per (utterance, chain), for chains of any length.  It walks the chain in tiles of P hop blocks (H = L / 2
// frames each, the tiling of nnk_ms_segment.cu): the tile of blocks [p, p + P) stages frames
// [(p - 1) H - E, (p + P + 1) H + E) of the trajectory in shared memory (E = NNK_MAX_HALF: the stencil's reach),
// takes the Q term of its frames [p H, (p + P) H) and the MS term of segments p .. p + P - 1, one segment per
// warp at a time (window, n / 2-point FFT in the warp's own shared memory, bin pairs).  The per-thread partials
// of both sums run over the tiles in a fixed order and meet in a fixed tree.  c' is formed on the fly from c,
// c_m, h and alpha, and recomputed with the same expression when an accepted trial is committed.  The gradient
// pass stages c again and runs segments p .. p + P of every tile (forward FFT, C_j, inverse FFT, times w), even
// ones first, then odd ones adding into the tile's result in shared memory, as ms_segment_kernel overlaps.
// ms_gen_kernel keeps its own inline copy of the Q stencil and of the accept rule: moving them into these
// helpers changes its SASS (DESIGN.md 3.18).
constexpr int MSS_THREADS = 256, MSS_WARPS = MSS_THREADS / 32;
constexpr int MSS_LOGN_MIN = 5, MSS_LOGN_MAX = 9;  // n = 32 .. 512
constexpr int MSS_TILE_FRAMES = 256;               // frames of a tile, rounded to an even number of hop blocks
constexpr int MSS_EXT = NNK_MAX_HALF;              // frames staged beyond the segments for the Q stencil

struct MsSegGenParams {
  MsGenParams g;
  int L, P;  // segment length, hop blocks per tile (even)
};

static inline int mss_tile_blocks(int H) {
  const int q = (MSS_TILE_FRAMES / H) & ~1;
  return q > 2 ? q : 2;
}

// tau-weighted squared residual of frame t of the trajectory x (x[i] = frame i, read for i in [t - l, t + u]
// within [0, T)) added to q: tau with nnk_mlpg_fwd's edge rule (dynamic windows have no precision on the first
// and last m_edge frames, and on every frame when m_edge == 0).  Summed over t, -q / 2 is Q up to a constant.
__device__ __forceinline__ double ms_q_frame(const MsGenParams& p, const nnk_chain_t& ch, const double* mrow,
                                             const double* vrow, int t, int T, const double* x, double q) {
  const bool edge = p.m_edge == 0 || t < p.m_edge || t >= T - p.m_edge;
  for (int w = 0; w < p.nw; ++w) {
    if (w > 0 && edge) continue;
    const int64_t col = (int64_t)w * ch.win_stride;
    const double tau = 1.0 / vrow[p.var_ld ? t * p.var_ld + col : col];
    double e = -mrow[t * p.in_ld + col];
    for (int k = -p.l[w]; k <= p.u[w]; ++k)
      if (t + k >= 0 && t + k < T) e = fma(p.coef[w][p.l[w] + k], x[t + k], e);
    q = fma(tau * e, e, q);
  }
  return q;
}

// the accept rule, called by every thread of the CTA with the same F(c'): c' is kept when F(c') >= F(c) (always
// at the start point, !trial); thread 0 then updates F and alpha (halved on a rejection)
__device__ __forceinline__ bool ms_accept(const MsGenParams& p, size_t si, double f2, double alpha, bool trial,
                                          int tid) {
  const bool accept = !trial || f2 >= p.F[si];
  __syncthreads();  // every thread has read F before thread 0 rewrites it
  if (tid == 0) {
    if (accept) p.F[si] = f2;
    p.alpha[si] = accept ? alpha : 0.5 * alpha;
  }
  return accept;
}

template <int LOGN, bool TRIAL>
__global__ void __launch_bounds__(MSS_THREADS, 1) ms_gen_segment_kernel(const __grid_constant__ MsSegGenParams sp) {
  using V = double2;
  constexpr int N = 1 << LOGN, M = N / 2, LOGM = LOGN - 1, NT = MSS_THREADS;
  const MsGenParams& p = sp.g;
  const int L = sp.L, H = L / 2, P = sp.P, NX = (P + 2) * H + 2 * MSS_EXT;
  extern __shared__ __align__(16) unsigned char mss_smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  V* tw = reinterpret_cast<V*>(mss_smem);  // W^j = e^{-2 pi i j / n}, j < M
  V* red = tw + M;                          // (Q, MS) partials, NT
  V* z = red + NT + warp * M;               // this warp's FFT
  double* qs = reinterpret_cast<double*>(red + NT + MSS_WARPS * M);  // q_k, k <= M
  double* nus = qs + M + 1;                                          // nu_k
  double* win = nus + M + 1;                                         // periodic Hann window, L
  double* xs = win + L;   // frames (p - 1) H - E .. (p + P + 1) H + E - 1 of the trajectory, NX
  double* ys = xs + NX;   // gradient: frames p H .. (p + P) H - 1 of the tile's result
  const int chain = (int)(blockIdx.x % (unsigned)p.n_chain), utt = (int)(blockIdx.x / (unsigned)p.n_chain);
  const int64_t row0 = p.utt_off[utt];
  const int T = p.utt_len ? p.utt_len[utt] : (int)(p.utt_off[utt + 1] - row0);
  if (T <= 0) return;
  const nnk_chain_t ch = p.chains[chain];
  const int64_t ld = p.out_ld;
  double* c = p.c + row0 * ld + ch.out_col;
  const double* cm = p.cm + row0 * ld + ch.out_col;
  if (ch.flags & 1) {  // pass-through: nnk_mlpg_fwd copied the column into c_m
    if (!TRIAL)
      for (int t = tid; t < T; t += NT) c[t * ld] = cm[t * ld];
    return;
  }
  const size_t si = (size_t)utt * p.n_chain + chain;
  const double omega = p.weight > 0.0 ? p.weight : 1.0 / ((double)p.nw * (double)T);
  const int J = (T + H - 1) / H + 1, tiles = (J + P - 1) / P;
  for (int j = tid; j < M; j += NT) {
    double s, co;
    sincospi(double(2 * j) / double(N), &s, &co);
    tw[j] = cx<V>(co, -s);
  }
  for (int k = tid; k <= M; k += NT) {
    qs[k] = 1.0 / p.ms_var[k * ld + ch.out_col];
    nus[k] = p.ms_mean[k * ld + ch.out_col];
  }
  for (int m = tid; m < L; m += NT) {
    double s, co;
    sincospi(double(2 * m) / double(L), &s, &co);
    win[m] = 0.5 - 0.5 * co;
  }
  const double alpha = TRIAL ? p.alpha[si] : p.step;
  const double* h = p.h + row0 * ld + ch.out_col;
  // c' at frame t; the commit recomputes it with this expression, so the bits are those F(c') was taken at
  auto trial_point = [&](int t) {
    if (!TRIAL) return cm[t * ld];
    const double ct = c[t * ld];
    return fma(alpha, (cm[t * ld] - ct) + h[t * ld] / omega, ct);
  };
  // the trajectory of the tile of blocks [b0, b0 + P) into xs (zeros outside [0, T)); returns x, x[t] = frame t
  auto stage = [&](int b0, bool trial) {
    const int f0 = (b0 - 1) * H - MSS_EXT;
    __syncthreads();  // the previous tile's reads of xs are done
    for (int i = tid; i < NX; i += NT) {
      const int t = f0 + i;
      xs[i] = t >= 0 && t < T ? (trial ? trial_point(t) : c[t * ld]) : 0.0;
    }
    __syncthreads();
    return xs - f0;
  };
  // the windowed segment j of x, zero-padded to n, transformed in this warp's z (Z in natural order)
  auto segment_fft = [&](const double* x, int j) {
    const double* xc = x + (j - 1) * H;
    __syncwarp();  // the previous segment's reads of z are done
    for (int t = lane; t < M; t += 32) {
      const int m0 = 2 * t, m1 = 2 * t + 1;
      z[__brev(t) >> (32 - LOGM)] = cx<V>(m0 < L ? win[m0] * xc[m0] : 0.0, m1 < L ? win[m1] * xc[m1] : 0.0);
    }
    __syncwarp();
    warp_fft_dit<LOGN>(z, tw, lane);
  };
  __syncthreads();  // tw, qs, nus, win
  // F(c'): Q over each tile's frames, the MS term over each tile's segments
  const double* mrow = p.means + row0 * p.in_ld + ch.in_col;
  const double* vrow = p.vars + (p.var_ld ? row0 * p.var_ld : 0) + ch.in_col;
  auto bin_term = [&](V y, int k) {
    const double qk = qs[k];
    if (qk == 0.0) return 0.0;
    const double d = log_power(y.x * y.x + y.y * y.y) - nus[k];
    return qk * d * d;
  };
  double q = 0.0, ms = 0.0;
  for (int tile = 0; tile < tiles; ++tile) {
    const int b0 = tile * P;
    const double* x = stage(b0, true);
    const int t1 = min((b0 + P) * H, T);
    for (int t = b0 * H + tid; t < t1; t += NT) q = ms_q_frame(p, ch, mrow, vrow, t, T, x, q);
    const int j1 = min(b0 + P, J);
    for (int j = b0 + warp; j < j1; j += MSS_WARPS) {
      segment_fft(x, j);
      for (int k = lane; k <= M / 2; k += 32) {
        V Yk, Yj;
        rfft_bin_pair(z, tw, k, M, Yk, Yj);
        if (k > 0) ms += bin_term(Yk, k);
        if (M - k != k) ms += bin_term(Yj, M - k);
      }
    }
  }
  red[tid] = cx<V>(q, ms);
  __syncthreads();
#pragma unroll
  for (int s = NT / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] = cadd(red[tid], red[tid + s]);
    __syncthreads();
  }
  const double f2 = omega * (-0.5 * red[0].x) - 0.5 * red[0].y / (double)J;
  const bool accept = ms_accept(p, si, f2, alpha, TRIAL, tid);
  if (accept)
    for (int t = tid; t < T; t += NT) c[t * ld] = trial_point(t);
  if (!p.want_grad) return;
  // the gradient of the MS term at the current c: C_jk = G_jk Y_jk in place, each lane owning its pairs
  auto grad_bin = [&](V y, int k) {
    const double qk = qs[k], pw = y.x * y.x + y.y * y.y;
    if (qk == 0.0 || !(pw > DBL_MIN)) return cx<V>(0, 0);
    return scale(y, -qk * (log(pw) - nus[k]) / pw * (k == M ? 2.0 : 1.0));
  };
  double* g = p.g + row0 * p.n_chain + chain;
  for (int tile = 0; tile < tiles; ++tile) {
    const int b0 = tile * P;
    const double* x = stage(b0, false);  // its barriers also order the commit above before these reads
    for (int phase = 0; phase < 2; ++phase) {
      // segments b0 + qi, qi = phase, phase + 2, .. <= P: each phase covers the tile's P H frames once
      for (int qi = 2 * warp + phase; qi <= P; qi += 2 * MSS_WARPS) {
        const int j = b0 + qi;
        if (j >= J) {  // past the utterance: adds nothing
          __syncwarp();
          if (phase == 0)
            for (int m = lane; m < L; m += 32) {
              const int r = (qi - 1) * H + m;
              if (r >= 0 && r < P * H) ys[r] = 0.0;
            }
          continue;
        }
        segment_fft(x, j);
        for (int k = lane; k <= M / 2; k += 32) {
          V Yk, Yj;
          rfft_bin_pair(z, tw, k, M, Yk, Yj);
          rfft_pack_pair(z, tw, k, M, k == 0 ? cx<V>(0, 0) : grad_bin(Yk, k), grad_bin(Yj, M - k));
        }
        __syncwarp();
        warp_ifft_dif<LOGN>(z, tw, lane);
        for (int m = lane; m < L; m += 32) {  // frame m of n irfft(C_j), times w_m, into the tile's result
          const int r = (qi - 1) * H + m;
          if (r < 0 || r >= P * H) continue;
          const V v2 = z[__brev(m >> 1) >> (32 - LOGM)];
          const double v = win[m] * ((m & 1) ? v2.y : v2.x);
          if (phase == 0)
            ys[r] = v;
          else
            ys[r] += v;
        }
      }
      __syncthreads();
    }
    const int t1 = min((b0 + P) * H, T);
    for (int t = b0 * H + tid; t < t1; t += NT) g[(int64_t)t * p.n_chain] = ys[t - b0 * H] / (double)J;
  }
}

template <int LOGN> static size_t mss_smem(int L, int P) {
  constexpr int M = 1 << (LOGN - 1);
  const size_t H = L / 2;
  return (size_t)(M + MSS_THREADS + MSS_WARPS * M) * sizeof(double2) +
         (size_t)(2 * (M + 1) + L + (P + 2) * H + 2 * MSS_EXT + P * H) * sizeof(double);
}

template <int LOGN, bool TRIAL>
static int launch_ms_gen_segment(const MsSegGenParams& p, unsigned n_blocks, cudaStream_t st) {
  const size_t smem = mss_smem<LOGN>(p.L, p.P);
  if (smem > 48 * 1024)  // per device: cheap enough to set on every launch
    NNK_CUDA_CHECK(cudaFuncSetAttribute(ms_gen_segment_kernel<LOGN, TRIAL>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ms_gen_segment_kernel<LOGN, TRIAL><<<n_blocks, MSS_THREADS, smem, st>>>(p);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

template <bool TRIAL>
static int dispatch_ms_gen_segment(int logn, const MsSegGenParams& p, unsigned n_blocks, cudaStream_t st) {
  switch (logn) {
    case 5: return launch_ms_gen_segment<5, TRIAL>(p, n_blocks, st);
    case 6: return launch_ms_gen_segment<6, TRIAL>(p, n_blocks, st);
    case 7: return launch_ms_gen_segment<7, TRIAL>(p, n_blocks, st);
    case 8: return launch_ms_gen_segment<8, TRIAL>(p, n_blocks, st);
    default: return launch_ms_gen_segment<9, TRIAL>(p, n_blocks, st);
  }
}

// byte offsets of the workspace parts: the MLPG factor scratch, c_m, h, g, F, alpha (each 256-byte aligned)
struct MsGenWs {
  size_t cm, h, g, F, alpha, total;
};

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

static bool ms_gen_ws(int32_t n_utt, int32_t n_chain, int32_t max_T, int64_t n_rows, int64_t out_ld,
                      const nnk_windows_t* win, MsGenWs& w) {
  const size_t fac = nnk_mlpg_workspace_bytes(n_utt, n_chain, max_T, win);
  if (fac == 0 || n_rows < 0 || out_ld < 0) return false;
  w.cm = align256(fac);
  w.h = w.cm + align256((size_t)n_rows * out_ld * sizeof(double));
  w.g = w.h + align256((size_t)n_rows * out_ld * sizeof(double));
  w.F = w.g + align256((size_t)n_rows * n_chain * sizeof(double));
  w.alpha = w.F + align256((size_t)n_utt * n_chain * sizeof(double));
  w.total = w.alpha + align256((size_t)n_utt * n_chain * sizeof(double));
  return true;
}

// the launch sequence of both levels: validation common to both, nnk_mlpg_fwd (c_m), the first trial-kernel
// launch (copy c_m, first gradient), then per trial one nnk_mlpg_solve and one trial-kernel launch.
// launch(trial, params, n_blocks, stream) launches the level's trial kernel.
template <typename Launch>
static int mlpg_ms_sequence(const nnk_mlpg_args_t* a, const nnk_mlpg_ms_t* ms, void* stream, Launch launch) {
  NNK_REQUIRE(ms->n_iter >= 0, NNK_ERR_ARG, "n_iter must be >= 0");
  NNK_REQUIRE(ms->step > 0.0, NNK_ERR_ARG, "step must be > 0");
  NNK_REQUIRE(!(ms->weight < 0.0) && ms->weight == ms->weight, NNK_ERR_ARG, "weight must be > 0 (or 0 for 1 / (nw T))");
  if (a->n_utt == 0 || a->n_chain == 0 || a->max_T == 0) return NNK_OK;  // nothing to do
  NNK_REQUIRE(a->means && a->vars && a->out && a->utt_off && a->chains && a->status_word, NNK_ERR_ARG,
              "NULL device pointer");
  NNK_REQUIRE(ms->ms_mean && ms->ms_var, NNK_ERR_ARG, "NULL ms_mean / ms_var");
  NNK_REQUIRE(a->win.nw >= 1 && a->win.nw <= NNK_MAX_WIN, NNK_ERR_UNSUPPORTED, "unsupported window set");
  NNK_REQUIRE((int64_t)a->n_utt * a->n_chain <= 0x7fffffff, NNK_ERR_UNSUPPORTED, "batch too large for one launch");
  MsGenWs w;
  NNK_REQUIRE(ms_gen_ws(a->n_utt, a->n_chain, a->max_T, ms->n_rows, a->out_ld, &a->win, w), NNK_ERR_UNSUPPORTED,
              "window set not supported by the MLPG kernels");
  NNK_REQUIRE(a->workspace && a->workspace_bytes >= w.total, NNK_ERR_WORKSPACE,
              "workspace too small: need nnk_mlpg_ms_workspace_bytes()");
  DeviceGuard guard(a->out);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* ws = (unsigned char*)a->workspace;
  double* cm = (double*)(ws + w.cm);
  double* h = (double*)(ws + w.h);
  double* g = (double*)(ws + w.g);

  nnk_mlpg_args_t fa = *a;  // c_m = P^-1 b into the workspace
  fa.out = cm;
  fa.workspace_bytes = w.cm;
  int r = nnk_mlpg_fwd(&fa, stream);
  if (r != NNK_OK) return r;
  nnk_mlpg_args_t sa = fa;  // h = P^-1 g: chain c reads column c of g, writes column out_col of h
  sa.out = h;
  sa.grad_out = g;
  sa.go_ld = a->n_chain;
  sa.go_f64 = 1;

  MsGenParams p;
  p.means = (const double*)a->means; p.vars = (const double*)a->vars;
  p.in_ld = a->in_ld; p.var_ld = a->var_ld; p.out_ld = a->out_ld;
  p.utt_off = a->utt_off; p.utt_len = a->utt_len; p.chains = a->chains; p.n_chain = a->n_chain;
  p.nw = a->win.nw;
  p.m_edge = 0;
  for (int i = 0; i < NNK_MAX_WIN; ++i) {
    p.l[i] = i < a->win.nw ? a->win.l[i] : 0;
    p.u[i] = i < a->win.nw ? a->win.u[i] : 0;
    p.m_edge = p.l[i] > p.m_edge ? p.l[i] : p.m_edge;
    p.m_edge = p.u[i] > p.m_edge ? p.u[i] : p.m_edge;
    for (int k = 0; k < NNK_MAX_TAPS; ++k) p.coef[i][k] = a->win.coef[i][k];
  }
  p.cm = cm; p.h = h; p.c = (double*)a->out; p.g = g;
  p.F = (double*)(ws + w.F); p.alpha = (double*)(ws + w.alpha);
  p.ms_mean = ms->ms_mean; p.ms_var = ms->ms_var;
  p.step = ms->step; p.weight = ms->weight;
  const unsigned blocks = (unsigned)((int64_t)a->n_utt * a->n_chain);
  p.want_grad = ms->n_iter > 0;
  r = launch(false, p, blocks, st);
  for (int it = 0; r == NNK_OK && it < ms->n_iter; ++it) {
    r = nnk_mlpg_solve(&sa, stream);
    if (r != NNK_OK) return r;
    p.want_grad = it + 1 < ms->n_iter;
    r = launch(true, p, blocks, st);
  }
  return r;
}

// log2 of n when n is a power of two in [2^lo, 2^hi], else 0
static int ms_logn(int32_t n, int lo, int hi) {
  int logn = 0;
  while (logn < 31 && (1 << logn) < n) ++logn;
  return n > 0 && (1 << logn) == n && logn >= lo && logn <= hi ? logn : 0;
}

}  // namespace nnk

using namespace nnk;

extern "C" size_t nnk_mlpg_ms_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, int64_t n_rows,
                                              int64_t out_ld, const nnk_windows_t* win) {
  MsGenWs w;
  return ms_gen_ws(n_utt, n_chain, max_T, n_rows, out_ld, win, w) ? w.total : 0;
}

extern "C" int nnk_mlpg_ms(const nnk_mlpg_args_t* a, const nnk_mlpg_ms_t* ms, void* stream) {
  NNK_REQUIRE(a != nullptr && ms != nullptr, NNK_ERR_ARG, "args or ms is NULL");
  NNK_REQUIRE(a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F64 (widen float32 inputs first)");
  NNK_REQUIRE(a->out_off == nullptr, NNK_ERR_ARG, "out_off must be NULL");
  NNK_REQUIRE(a->n_utt >= 0 && a->n_chain >= 0 && a->max_T >= 0 && ms->n_rows >= 0, NNK_ERR_ARG, "negative size");
  const int logn = ms_logn(ms->n, MSG_LOGN_MIN, MSG_LOGN_MAX);
  NNK_REQUIRE(logn, NNK_ERR_ARG, "n must be 256, 512, 1024, 2048 or 4096");
  NNK_REQUIRE(a->max_T <= ms->n, NNK_ERR_ARG, "max_T exceeds n");
  return mlpg_ms_sequence(a, ms, stream, [logn](bool trial, const MsGenParams& p, unsigned blocks, cudaStream_t st) {
    return trial ? dispatch_ms_gen<true>(logn, p, blocks, st) : dispatch_ms_gen<false>(logn, p, blocks, st);
  });
}

extern "C" int nnk_mlpg_ms_segment(const nnk_mlpg_args_t* a, const nnk_mlpg_ms_t* ms, int32_t L, void* stream) {
  NNK_REQUIRE(a != nullptr && ms != nullptr, NNK_ERR_ARG, "args or ms is NULL");
  NNK_REQUIRE(a->dtype == NNK_F64, NNK_ERR_ARG, "dtype must be NNK_F64 (widen float32 inputs first)");
  NNK_REQUIRE(a->out_off == nullptr, NNK_ERR_ARG, "out_off must be NULL");
  NNK_REQUIRE(a->n_utt >= 0 && a->n_chain >= 0 && a->max_T >= 0 && ms->n_rows >= 0, NNK_ERR_ARG, "negative size");
  const int logn = ms_logn(ms->n, MSS_LOGN_MIN, MSS_LOGN_MAX);
  NNK_REQUIRE(logn, NNK_ERR_ARG, "n must be 32, 64, 128, 256 or 512");
  NNK_REQUIRE(L >= 4 && L <= ms->n && L % 2 == 0, NNK_ERR_ARG, "L must be even with 4 <= L <= n");
  return mlpg_ms_sequence(a, ms, stream, [logn, L](bool trial, const MsGenParams& p, unsigned blocks,
                                                   cudaStream_t st) {
    MsSegGenParams sp;
    sp.g = p;
    sp.L = L;
    sp.P = mss_tile_blocks(L / 2);
    return trial ? dispatch_ms_gen_segment<true>(logn, sp, blocks, st)
                 : dispatch_ms_gen_segment<false>(logn, sp, blocks, st);
  });
}
