// nnk_ms_gen.cu -- parameter generation considering the modulation spectrum (paramgen.mlpg_ms_batch; C ABI:
// include/nnk_ms_gen.h, definition in DESIGN.md 3.18).
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
#include "../../include/nnk_ms_gen.h"

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
  int logn = 0;
  while (logn < 31 && (1 << logn) < ms->n) ++logn;
  NNK_REQUIRE(ms->n > 0 && (1 << logn) == ms->n && logn >= MSG_LOGN_MIN && logn <= MSG_LOGN_MAX, NNK_ERR_ARG,
              "n must be 256, 512, 1024, 2048 or 4096");
  NNK_REQUIRE(a->max_T <= ms->n, NNK_ERR_ARG, "max_T exceeds n");
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
  r = dispatch_ms_gen<false>(logn, p, blocks, st);
  for (int it = 0; r == NNK_OK && it < ms->n_iter; ++it) {
    r = nnk_mlpg_solve(&sa, stream);
    if (r != NNK_OK) return r;
    p.want_grad = it + 1 < ms->n_iter;
    r = dispatch_ms_gen<true>(logn, p, blocks, st);
  }
  return r;
}
