/*
 * nnk_b200.h -- C ABI of libnnk_b200.so: the H100 (sm_90a) implementation of nnmnkwii's two
 * numeric hot paths, MLPG trajectory smoothing and DTW alignment.
 *
 * The reference (r9y9/nnmnkwii v0.1.3) has no FFI/plugin registry: its boundary is a set of Python
 * callables backed by Cython extensions.  Each entry point below names the reference interface
 * (file:line in r9y9/nnmnkwii v0.1.3) whose arithmetic it replaces; INTEGRATION.md shows the ctypes
 * stub a reference maintainer would add at each of those call sites.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types.
 *   - "device" pointers are CUDA device memory owned by the caller; "host" pointers are ordinary
 *     (ideally pinned) host memory.  All matrices are row-major.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 *   - Device entry points are asynchronous: they enqueue work on `stream` and return.  Numerical
 *     failures (non-positive pivot) are written to a caller-provided device status record that the
 *     host inspects after synchronising (nnk_status_t).  Host entry points synchronise internally.
 *   - Return value: NNK_OK or a negative NNK_ERR_* (argument / CUDA errors; nnk_last_error() has text).
 *   - There is no CPU fallback anywhere in this library.
 */
#ifndef NNK_B200_H
#define NNK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NNK_ABI_VERSION 2

#define NNK_OK 0
#define NNK_ERR_ARG -1          /* bad argument                                               */
#define NNK_ERR_UNSUPPORTED -2  /* window set larger than NNK_MAX_WIN / NNK_MAX_HALF           */
#define NNK_ERR_CUDA -3         /* CUDA runtime error                                          */
#define NNK_ERR_WORKSPACE -4    /* workspace too small (see *_workspace_bytes)                 */
#define NNK_ERR_NOT_PD -5       /* host entry points only: non-positive pivot (see status)     */

#define NNK_F32 0
#define NNK_F64 1
#define NNK_I32 2 /* integer element types: inputs of nnk_mulaw's inverse quantiser only       */
#define NNK_I64 3

#define NNK_MAX_WIN 4  /* windows per stream (static, delta, delta-delta, +1)                  */
#define NNK_MAX_HALF 4 /* max(l, u) of any window                                              */
#define NNK_MAX_TAPS (2 * NNK_MAX_HALF + 1)

/* Windows = the reference's list of (l, u, win_coeff) triples (paramgen/_mlpg.py:16-20).
 * coef[w][0 .. l[w]+u[w]] holds win_coeff of window w.                                        */
typedef struct nnk_windows {
  int32_t nw;
  int32_t l[NNK_MAX_WIN];
  int32_t u[NNK_MAX_WIN];
  double coef[NNK_MAX_WIN][NNK_MAX_TAPS];
} nnk_windows_t;

/* Failure record.  On the device it is ONE zero-initialised uint64 word (`status_word`) that the
 * kernels update atomically so that the lexicographically first failure (utterance, chain, frame)
 * wins -- the order in which the reference's Python loops would have raised.  The host decodes
 * it with nnk_status_decode().
 *   code 0 = ok, 1 = non-positive pivot (reference: scipy.linalg.LinAlgError
 *   "%d-th leading minor not positive definite", _bandmat/linalg.pyx:79-82)                    */
typedef struct nnk_status {
  int32_t code;
  int32_t utt;   /* utterance index                                                           */
  int32_t chain; /* chain index (static dimension within the layout)                          */
  int32_t frame; /* 1-based frame of the pivot, as in the reference's message                 */
} nnk_status_t;

/* One "chain" = one static dimension of one stream = one banded T x T solve.
 * A (T, D) frame matrix in Merlin layout holds several streams side by side (e.g. mgc 180 = 3 x 60,
 * lf0 3, vuv 1, bap 3); chain c reads window w of its stream at column in_col + w * win_stride and
 * writes its trajectory to column out_col.  flags & 1 = pass-through (copy in_col -> out_col, no
 * smoothing: the vuv column of the gallery notebooks).                                          */
typedef struct nnk_chain {
  int32_t in_col;
  int32_t win_stride;
  int32_t out_col;
  int32_t flags;
} nnk_chain_t;

/* Batched MLPG over a flat (n_rows, ld) frame matrix holding n_utt utterances back to back.    */
typedef struct nnk_mlpg_args {
  const void* means;          /* device (n_rows, in_ld)   dtype                                */
  const void* vars;           /* device (n_rows, var_ld) per-frame variances, or (>= D,) global
                                 variances when var_ld == 0 (paramgen/_mlpg.py:169-170)        */
  const void* grad_out;       /* device (n_rows, go_ld): nnk_mlpg_grad: backpropagated gradient;
                                 nnk_mlpg_solve: right-hand sides.  Chain c reads column c.
                                 float32, or float64 when go_f64 != 0                          */
  void* out;                  /* device: fwd (n_rows, out_ld) dtype ; grad (n_rows, out_ld) f32 */
  int32_t dtype;              /* NNK_F32 / NNK_F64 of means, vars (and out for fwd)            */
  int32_t n_utt;
  int64_t in_ld, var_ld, go_ld, out_ld; /* row strides in elements                            */
  const int64_t* utt_off;     /* device (n_utt + 1) row offsets                                */
  const int32_t* utt_len;     /* device (n_utt) frame counts, or NULL => utt_off[u+1]-utt_off[u];
                                 lets zero-padded (B, Tmax, D) batches be used in place        */
  const int32_t* order;       /* device (n_utt) processing order (e.g. longest first) or NULL  */
  const nnk_chain_t* chains;  /* device (n_chain)                                              */
  int32_t n_chain;
  int32_t max_T;              /* max utterance length (host knows it; sizes the workspace)     */
  int32_t go_f64;             /* grad_out / rhs element type: 0 = float32, 1 = float64         */
  nnk_windows_t win;
  void* workspace;            /* device scratch, >= nnk_mlpg_workspace_bytes()                 */
  size_t workspace_bytes;
  uint64_t* status_word;      /* device; must be zeroed by the caller before the first launch  */
  const int64_t* out_off;     /* device (n_utt) first OUTPUT row of every utterance, or NULL =>
                                 utt_off (same rows in and out).  Lets a rank write its slice of
                                 a sharded batch straight into its slot of the all-gather buffer */
} nnk_mlpg_args_t;

void nnk_status_decode(uint64_t status_word, nnk_status_t* out);

/* Replaces paramgen.mlpg (paramgen/_mlpg.py:92-199: build_poe :53-89, bla.solveh
 * _bandmat/linalg.pyx:290-304) for a whole batch: out[:, chain.out_col] = P^{-1} b per chain.   */
int nnk_mlpg_fwd(const nnk_mlpg_args_t* args, void* stream);

/* Replaces paramgen.mlpg_grad (paramgen/_mlpg.py:202-281) in closed form:
 * out[:, in_col + w*win_stride] = tau_w * (W_w P^{-1} grad_out[:, chain]); out is float32.      */
int nnk_mlpg_grad(const nnk_mlpg_args_t* args, void* stream);

/* General banded solve with the same P: out[:, chain.out_col] = P^{-1} rhs[:, chain] (dtype of
 * `out` = args->dtype).  Used to build unit_variance_mlpg_matrix (paramgen/_mlpg.py:297-373):
 * R = P^{-1} Wtilde^T with unit variances, one chain per column of Wtilde^T.                    */
int nnk_mlpg_solve(const nnk_mlpg_args_t* args, void* stream);

/* Scratch needed by the calls above for `n_utt` utterances of at most max_T frames.         */
size_t nnk_mlpg_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

/* Parameter generation considering global variance (Toda, Black & Tokuda 2007, Sec. IV; diagonal GV
 * covariance).  Per chain c (mu = gv_mean[c.out_col], p = 1 / gv_var[c.out_col], T frames) and with
 * c_m = P^-1 b the nnk_mlpg_fwd trajectory, maximises
 *   F(c) = omega (b^T c - c^T P c / 2) - p (v(c) - mu)^2 / 2,  v(c) = population variance of c over T
 * starting from c0 = mean(c_m) + sqrt(mu / v(c_m)) (c_m - mean(c_m)) (c0 = c_m when v(c_m) == 0), with
 * n_iter trials of c' = c + alpha ((c_m - c) + P^-1 g / omega), g = dv/dc * (-p (v - mu)): c' is kept
 * when F(c') >= F(c), otherwise alpha halves (alpha starts at `step`; a rejected trial still counts).
 * omega = weight, or 1 / (nw T) when weight == 0.  float64 arithmetic, output in args->dtype; pass-through
 * chains are copied.  Same arguments, status word and failure rule as nnk_mlpg_fwd; the workspace must hold
 * nnk_mlpg_gv_workspace_bytes() (the factors plus four columns per frame: d, c_m, c, trial c).        */
typedef struct nnk_mlpg_gv {
  const double* gv_mean;      /* device, indexed by chain out_col: target GV, >= 0                   */
  const double* gv_var;       /* device, indexed by chain out_col: variance of the GV, > 0             */
  int32_t n_iter;             /* >= 0 trials                                                           */
  double step;                /* > 0 initial step alpha                                                */
  double weight;              /* omega > 0, or 0 => 1 / (nw T) per utterance                           */
} nnk_mlpg_gv_t;
int nnk_mlpg_gv(const nnk_mlpg_args_t* args, const nnk_mlpg_gv_t* gv, void* stream);
size_t nnk_mlpg_gv_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

/* Per-segment moments of the columns of a row-major float32 / float64 matrix (row stride ld elements):
 * segment u is rows utt_off[u] .. utt_off[u] + len - 1, len = utt_len[u] (device int32, or NULL =>
 * utt_off[u+1] - utt_off[u]), every len >= 1.  mean (n_utt, D) (may be NULL) and var (n_utt, D) float64,
 * var = population variance, two passes (mean, then squared deviations), float64 accumulation in a fixed
 * order.  Serves paramgen.global_variance / gv_statistics.                                          */
int nnk_segment_moments(const void* X, int32_t dtype, int32_t D, int64_t ld, const int64_t* utt_off,
                        const int32_t* utt_len, int32_t n_utt, double* mean, double* var, void* stream);

/* Host-buffer convenience = what a cgo/ctypes binding of paramgen.mlpg would call: one utterance,
 * one stream, host pointers (means (T, D), variances (T, D) or (D,), out (T, D / nw)), copies
 * included, synchronous.  Returns NNK_ERR_NOT_PD with *bad_frame = 1-based frame on failure.    */
int nnk_mlpg_host(const void* means, const void* vars, int32_t var_is_1d, int32_t dtype, int64_t T,
                  int64_t D, const nnk_windows_t* win, void* out, int32_t* bad_frame);

/* Host-buffer batched MLPG: flat (n_rows, D) host matrices, chains/offsets on the host.  H2D and
 * D2H copies run chunked on two streams so they overlap the solve.  This is the end-to-end path
 * bench.py times as `e2e`.                                                                      */
int nnk_mlpg_batch_host(const void* means, const void* vars, int32_t var_is_1d, int32_t dtype,
                        int64_t n_rows, int64_t D, int64_t D_out, const int64_t* utt_off, int32_t n_utt,
                        const nnk_chain_t* chains, int32_t n_chain, const nnk_windows_t* win, void* out,
                        nnk_status_t* status);

/* ---- UnitVarianceMLPG (autograd/_impl/mlpg.py:70-172) ------------------------------------------
 * R (T, nw*T) row-major device matrix (float32, or float64 when dtype == NNK_F64) as produced by
 * unit_variance_mlpg_matrix (paramgen/_mlpg.py:297-373).
 * 1. nnk_uv_band_profile: profile[dist] = max |R[t, w*T+s]| over |t-s| == dist (T floats); the
 *    host picks the half-width K from it.
 * 2. nnk_uv_band_extract: Rb, RbT (T, nw, 2K+1) band tables (same dtype as R).
 * 3. nnk_uv_apply: backward == 0: y (B, T, sd) = R x   replacing torch.matmul(R, reshaped_means)
 *    (mlpg.py:138); backward != 0: y = R^T x replacing torch.matmul(R.transpose(0,1), grad_output)
 *    (mlpg.py:158).  The nw-window side is (B, T, nw*sd) when reshaped == 0 or (B, nw*T, sd)
 *    when reshaped != 0 (mlpg.py:124-136, :160-167); the other side is (B, T, sd).               */
int nnk_uv_band_profile(const void* R, int32_t dtype, int32_t T, int32_t nw, float* profile, void* stream);
int nnk_uv_band_extract(const void* R, int32_t dtype, int32_t T, int32_t nw, int32_t K, void* Rb, void* RbT, void* stream);
int nnk_uv_apply(const void* table, const void* x, void* y, int32_t dtype, int32_t B, int32_t T, int32_t sd,
                 int32_t nw, int32_t K, int32_t backward, int32_t reshaped, void* stream);
/* float32 variant exploiting that away from the two ends every row of a window block of R is the
 * same FIR filter: rows [t_lo, t_hi) use `taps` (HOST pointer, nw x (2K+1) floats, passed to the
 * kernel through the constant bank), the edge rows use `table` as above.                          */
int nnk_uv_apply_toeplitz(const void* table, const float* taps, const void* x, void* y, int32_t B, int32_t T,
                          int32_t sd, int32_t nw, int32_t K, int32_t t_lo, int32_t t_hi, int32_t backward,
                          int32_t reshaped, void* stream);

/* Factored float32 variant: in the shift-invariant rows every window block of R is one long filter h0
 * (a row of P^-1) convolved with a short window stencil, h_w = h0 * c_w; the host recovers c_w from R
 * (HOST pointers: h0 2K+1 floats, c nw x (2*KC+1) floats) and the sweep costs (2K+1) + ~7 multiply-adds
 * per output instead of nw*(2K+1) (replaces the same two torch.matmul calls, mlpg.py:138 / :158).
 * Packs two static dims per thread for any static_dim (odd ones, e.g. the reference's perf grid
 * static_dim = 59, perf/autograd_mlpg_perf.py:110-120, use predicated 4-byte accesses).              */
int nnk_uv_apply_factored(const void* table, const float* h0, const float* c, const void* x, void* y, int32_t B,
                          int32_t T, int32_t sd, int32_t nw, int32_t K, int32_t KC, int32_t t_lo, int32_t t_hi,
                          int32_t backward, int32_t reshaped, void* stream);

/* ---- DTW alignment (preprocessing/alignment.py:9-190) ------------------------------------------
 * Batched replacement of `dist, path = fastdtw(x, y, radius=self.radius, dist=self.dist)`
 * (alignment.py:50, :138; third-party slaypni/fastdtw, unpinned in setup.py:139 -- see DESIGN.md
 * "parity unpinned").  One CTA per pair; radius < 0 = exact DTW (full anti-diagonal wavefront),
 * radius >= 1 = FastDTW with that radius.  cost_kind 0 = default lambda x, y: norm(x - y)
 * (alignment.py:35), 1 = metrics.melcd (metrics/__init__.py:27-57).  Arithmetic is float64.     */
typedef struct nnk_dtw_args {
  const void* X;              /* device (n_pairs, .., D): pair p, frame t at X + p*x_pair_stride + t*x_ld */
  const void* Y;
  int32_t dtype;              /* NNK_F32 / NNK_F64 of X and Y                                   */
  int32_t n_pairs;
  int64_t x_pair_stride, y_pair_stride; /* elements                                           */
  int32_t x_ld, y_ld, D;
  const int32_t* len_x;       /* device (n_pairs): frames kept by trim_zeros_frames (alignment.py:49) */
  const int32_t* len_y;
  const int32_t* order;       /* device (n_pairs) processing order or NULL                      */
  int32_t cost_kind;
  int32_t radius;
  int32_t* path_i;            /* device (n_pairs, path_ld): pathx of alignment.py:52             */
  int32_t* path_j;            /* device (n_pairs, path_ld): pathy                                */
  int32_t path_ld;            /* >= max_tx + max_ty - 1                                         */
  int32_t* path_len;          /* device (n_pairs)                                               */
  double* dist;               /* device (n_pairs): accumulated cost D[Tx-1, Ty-1]               */
  int64_t* cells;             /* device (n_pairs) DP cells evaluated, or NULL                   */
  int32_t max_tx, max_ty;
  void* workspace;
  size_t workspace_bytes;     /* >= nnk_dtw_workspace_bytes()                                   */
} nnk_dtw_args_t;

int nnk_dtw_align(const nnk_dtw_args_t* args, void* stream);
size_t nnk_dtw_workspace_bytes(int32_t n_pairs, int32_t max_tx, int32_t max_ty, int32_t D, int32_t radius);

/* out[p, r, :] = X[p, path[p, r], :] for r < path_len[p], zero for r >= path_len[p]
 * (x = x[pathx]; X_aligned[idx][:len(x)] = x over a zero array: alignment.py:46-47, 52-54, 72-73)  */
int nnk_gather_rows(const void* X, int32_t dtype, int64_t x_pair_stride, int32_t x_ld, const int32_t* path,
                    int32_t path_ld, const int32_t* path_len, void* out, int64_t out_pair_stride, int32_t out_rows,
                    int32_t D, int32_t n_pairs, void* stream);

/* len[p] = len(trim_zeros_frames(X[p], eps, trim="b")) (preprocessing/generic.py:291-323)          */
int nnk_trim_lengths(const void* X, int32_t dtype, int64_t pair_stride, int32_t ld, int32_t T, int32_t D, double eps,
                     int32_t n_pairs, int32_t* len, void* stream);

/* ---- inverse from a Cholesky factor (util/linalg.py:7-36, util/_linalg.pyx:45-71), float64 ----------
 * B row-major (N, N) matrices back to back in, B full (N, N) results out; P must not alias the input
 * (it is the substitutions' scratch).  No workspace.
 *   nnk_cholesky_inv:        P = (L L^T)^-1 (lower != 0, lower triangle of each input read) or
 *                            (U^T U)^-1 (lower == 0, upper triangle read) -- dpotri + mirror.  P is
 *                            exactly symmetric: one triangle is computed and mirrored.
 *   nnk_cholesky_inv_banded: P = (R R^T)^-1, only the band R[t, t-j], 0 <= j < width, read.  Bit-identical
 *                            to the reference's row recurrence on finite input (signs of zeros aside).
 * A zero or non-finite diagonal entry sets *status_word (device, zero-initialised by the caller;
 * nnk_status_decode: utt = batch item, frame = row + 1, first item / row wins); the results of that
 * item are then undefined, and no input faults.
 * NNK_REQUIRE: N, T, B >= 0; width >= 1; non-NULL pointers when there is work; P != input.
 * NNK_ERR_UNSUPPORTED: min(width, T) > 9 (l + u + 1 of every window set the MLPG kernels accept).      */
int nnk_cholesky_inv(const double* L, int32_t lower, int32_t N, int32_t B, double* P, uint64_t* status_word,
                     void* stream);
int nnk_cholesky_inv_banded(const double* R, int32_t width, int32_t T, int32_t B, double* P, uint64_t* status_word,
                            void* stream);

/* ---- delta features (SURVEY section 8f row 2; preprocessing/generic.py:229-288) ------------------
 * out[:, w*D + d] = np.correlate(x[:, d], coef_w, mode="same") per utterance of a flat (sum_T, D)
 * batch: window centred at len(coef_w) // 2, zeros outside the utterance, float64 arithmetic,
 * result in the dtype of x.  out has nw*D columns.                                                */
int nnk_delta_features(const void* x, int32_t dtype, int32_t D, int64_t x_ld, const int64_t* utt_off,
                       const int32_t* utt_len, int32_t n_utt, int32_t max_T, const nnk_windows_t* win, void* out,
                       int64_t out_ld, void* stream);

/* ---- length-masked objective metrics (SURVEY section 8f row 4; metrics/__init__.py:27-190) --------
 * Padded (B, T, D) batches X, Y (element strides item_stride / frame_stride, D contiguous), lengths
 * (B) int32 on the device or NULL (all T frames valid).  The kernels deliver the SUM (float64) and the
 * COUNT of contributing frames; mean / sqrt / dB constant are the caller's scalar finish.
 *   nnk_frame_metric kind 0: sum of per-frame ||x - y||_2      (melcd,               :59-71)
 *                    kind 1: sum of (x - y)^2 over frames x D  (mean_squared_error,  :103-110)
 *   nnk_f0_metric    kind 0: sum of (x - y)^2 over frames with src_vuv + tgt_vuv >= 2; count = voiced
 *                    kind 1: the same on exp(x), exp(y)        (lf0_mean_squared_error, :141-165)
 *                    kind 2: sum of (src_vuv != tgt_vuv)       (vuv_error,           :181-190)
 * Deterministic (fixed-order fold of per-block partials).  workspace >= nnk_metric_workspace_bytes(B, T),
 * zero-filled before its first use (each call leaves it reusable); one workspace per stream.         */
int64_t nnk_metric_workspace_bytes(int32_t B, int32_t T);
int nnk_frame_metric(const void* X, const void* Y, int32_t dtype, int32_t B, int32_t T, int32_t D,
                     int64_t item_stride, int64_t frame_stride, const int32_t* lengths, int32_t kind, double* sum_out,
                     int64_t* count_out, void* workspace, int64_t workspace_bytes, void* stream);
int nnk_f0_metric(const void* src_f0, const void* src_vuv, const void* tgt_f0, const void* tgt_vuv, int32_t dtype,
                  int32_t B, int32_t T, int64_t item_stride, int64_t frame_stride, const int32_t* lengths,
                  int32_t kind, double* sum_out, int64_t* count_out, void* workspace, int64_t workspace_bytes,
                  void* stream);

/* ---- GMM mapping in front of MLPG (baseline/gmm.py:47-247; SURVEY.md 8f row 1) ---------------------
 * Device tables of a joint source/target GMM with M mixtures over D-dimensional frames, float64:
 *   src_means, tgt_means (M, D); prec_chol (M, D, D) = sklearn precisions_cholesky_ of the source marginal
 *   (U_m, row-major [d][e]); log_const (M) = log w_m + log det U_m - D/2 log 2pi;
 *   A_t (M, D, D) = (Syx_m Sxx_m^-1)^T, row-major [j][i]; Dm (M, D) = Eq. 23 diagonal variances (may be
 *   NULL when no variances are requested).
 * nnk_gmm_logprob: lp (T, M) = log w_m + log N(x_t | mu_m, Sxx_m)  -- the per-frame predict_proba /
 *   posterior of gmm.py:116-118, 219-221 before normalisation.
 * nnk_gmm_map: mode 0 = MLPG.transform's arg-max mixture sequence (gmm.py:219-237): E[t] = Eq. 22 mean,
 *   Dv[t] = Eq. 23 variance of the chosen mixture, mix[t] = its index (Dv / mix may be NULL);
 *   mode 1 = MLPGBase._transform_frame (gmm.py:97-121): E[t] = posterior-weighted mean, Eq. 13.     */
typedef struct nnk_gmm {
  const double* src_means;
  const double* tgt_means;
  const double* prec_chol;
  const double* log_const;
  const double* A_t;
  const double* Dm;
  int32_t M, D;
} nnk_gmm_t;
int nnk_gmm_logprob(const nnk_gmm_t* gmm, const double* x, int64_t x_ld, int32_t T, double* lp, void* stream);
int nnk_gmm_map(const nnk_gmm_t* gmm, const double* x, int64_t x_ld, int32_t T, const double* lp, int32_t mode, double* E,
                double* Dv, int32_t* mix, void* stream);

/* ---- trajectory EM of GMM voice conversion (baseline.gmm.MLPG.transform_em; csrc/nnk_gmm_traj.cu) --------------
 * float64.  The model (Toda, Black & Tokuda 2007, Sec. III, with the diagonal Eq. 23 variances of baseline.gmm.MLPG):
 * source frames x_t (D = nw * static_dim columns), static trajectory c (static_dim columns) and its
 * static + dynamic sequence Y_t[w * static_dim + s] = sum_{k = -l_w}^{u_w} coef[w][l_w + k] c_{t+k}[s], where
 * frames outside the utterance of t are zero.  Per mixture m:
 *   E_{m,t} = nu_m + A_m (x_t - mu_m)                    (gmm->tgt_means, gmm->A_t, gmm->src_means; Eq. 22)
 *   lw_{t,m} = lp[t][m] + log_norm[m][e_t] - 1/2 sum_{d in K_t} (Y_t - E_{m,t})_d^2 inv_Dm[m][d]
 * with lp from nnk_gmm_logprob and inv_Dm = 1 / D_m.  Like nnk_mlpg_fwd, which gives the dynamic windows zero
 * precision on the first and last H frames of an utterance (H = max_w max(l_w, u_w)) and on every frame when H = 0
 * (the reference's precisions[-0:] is the whole column), the columns K_t of frame t are all D columns (e_t = 0)
 * except on those edge frames, where they are the static_dim columns of window 0
 * (e_t = 1); log_norm[m][e] = -1/2 (sum_{d in K} log D_m,d + |K| log 2 pi) over the same columns.
 *
 * nnk_gmm_traj_em, one CTA per tile of NNK_GMM_TRAJ_TILE frames of one utterance:
 *   mode NNK_GMM_TRAJ_EM (E-step): gamma_{t,m} = softmax_m lw_{t,m};
 *     V[t][d] = 1 / P_t,d with P_t,d = sum_m gamma_{t,m} inv_Dm[m][d];
 *     E_bar[t][d] = (sum_m gamma_{t,m} E_{m,t,d} inv_Dm[m][d]) / P_t,d;
 *     both (T, D) row-major, the layout nnk_mlpg_fwd reads as means / variances.
 *   mode NNK_GMM_TRAJ_OBJECTIVE: E_bar and V are not touched (may be NULL).
 *   Both modes: ll_part[tile] = sum over the tile's frames, in frame order, of log sum_m exp lw_{t,m}
 *     (ll_part may be NULL in mode EM).  Utterance u owns the tiles tile_off[u] .. tile_off[u+1] - 1, in frame
 *     order; the per-utterance objective is their sum.
 * Tables (device int32, n_utt + 1 entries each): utterance u is frames utt_off[u] .. utt_off[u+1] - 1 with
 * utt_off[0] = 0, utt_off[n_utt] = T; tile_off[0] = 0, tile_off[u+1] - tile_off[u] =
 * ceil(len_u / NNK_GMM_TRAJ_TILE), tile_off[n_utt] = n_tiles.
 * Errors: NNK_ERR_ARG for NULL pointers, bad sizes or strides, D != win.nw * static_dim, a bad window set or
 * mode; NNK_ERR_UNSUPPORTED for D > 96 or more than 65535 mixtures; all before anything touches the device. */
#define NNK_GMM_TRAJ_EM 0
#define NNK_GMM_TRAJ_OBJECTIVE 1
#define NNK_GMM_TRAJ_TILE 32

typedef struct nnk_gmm_traj_args {
  const double* x;            /* device (T, x_ld) source frames, D = gmm->D columns                         */
  int64_t x_ld;
  const double* lp;           /* device (T, M) from nnk_gmm_logprob                                         */
  const double* c;            /* device (T, c_ld) current static trajectory, static_dim columns              */
  int64_t c_ld;
  int32_t T;
  int32_t n_utt;
  const int32_t* utt_off;     /* device (n_utt + 1)                                                         */
  const int32_t* tile_off;    /* device (n_utt + 1)                                                         */
  int32_t n_tiles;
  int32_t static_dim;
  nnk_windows_t win;
  int32_t mode;               /* NNK_GMM_TRAJ_EM / NNK_GMM_TRAJ_OBJECTIVE                                    */
  const double* inv_Dm;       /* device (M, D) 1 / D_m                                                      */
  const double* log_norm;     /* device (M, 2): all columns, static columns only                            */
  double* E_bar;              /* device (T, D), mode EM                                                     */
  double* V;                  /* device (T, D), mode EM                                                     */
  double* ll_part;            /* device (n_tiles), or NULL in mode EM                                       */
} nnk_gmm_traj_args_t;

int nnk_gmm_traj_em(const nnk_gmm_t* gmm, const nnk_gmm_traj_args_t* args, void* stream);

/* ---- GMM training: EM for full-covariance mixtures (sklearn.mixture.GaussianMixture.fit) ----------------
 * N frames of D features (D <= 128), K components (K <= 128); all parameters are float64 device arrays,
 * X is float32 (widened on load) or float64.  One EM iteration is
 *   nnk_gmm_em_estep   : resp (N, K) = exp(log_resp) from weights / means / prec_chol, *lower_bound = mean of the
 *                        per-frame log-likelihood (sklearn's _e_step + _compute_lower_bound);
 *   nnk_gmm_em_mstep   : from resp: means (K, D), covariances (K, D, D) with reg_covar on the diagonal and, per
 *                        weight_norm, weights = nk / N (0, sklearn's _initialize), nk / sum nk (1, its _m_step) or
 *                        left alone (2);
 *   nnk_gmm_em_factor  : factor != 0: prec_chol = L^-T with covariances = L L^T (sklearn's
 *                        _compute_precision_cholesky); factor == 0: prec_chol is the caller's.  Either way it
 *                        derives the per-component constants the next nnk_gmm_em_estep reads from the workspace,
 *                        so it must run after any change of weights, means or prec_chol.
 * A non-positive Cholesky pivot sets *status (zeroed by the caller) to 1 and leaves prec_chol undefined.
 * Every reduction runs in a fixed order: identical inputs give bit-identical outputs.  All three take their
 * scratch from `workspace` (>= nnk_gmm_em_workspace_bytes(N, D, K); 0 = unsupported sizes), which carries
 * state from nnk_gmm_em_factor to nnk_gmm_em_estep and from nnk_gmm_em_mstep's statistics to its covariances. */
typedef struct nnk_gmm_em_args {
  const void* X;              /* device (N, x_ld) frames                                               */
  int64_t N, x_ld;
  int32_t dtype;              /* NNK_F32 / NNK_F64 of X                                                */
  int32_t D, K;
  int32_t weight_norm;        /* nnk_gmm_em_mstep: 0 = nk / N, 1 = nk / sum(nk), 2 = keep weights      */
  int32_t factor;             /* nnk_gmm_em_factor: 1 = factor covariances, 0 = prec_chol given        */
  double reg_covar;
  double* resp;               /* device (N, K)                                                         */
  double* weights;            /* device (K)                                                            */
  double* means;              /* device (K, D)                                                         */
  double* covariances;        /* device (K, D, D)                                                      */
  double* prec_chol;          /* device (K, D, D) upper factors U, U U^T = covariance^-1               */
  double* lower_bound;        /* device (1)                                                            */
  int32_t* status;            /* device (1)                                                            */
  void* workspace;
  size_t workspace_bytes;
} nnk_gmm_em_args_t;
size_t nnk_gmm_em_workspace_bytes(int64_t N, int32_t D, int32_t K);
int nnk_gmm_em_estep(const nnk_gmm_em_args_t* args, void* stream);
int nnk_gmm_em_mstep(const nnk_gmm_em_args_t* args, void* stream);
int nnk_gmm_em_factor(const nnk_gmm_em_args_t* args, void* stream);

/* ---- k-means initialisation of the GMM fit (sklearn.cluster.KMeans(n_init=1) / kmeans_plusplus) -----------
 * N frames of D features (D <= 128), K clusters (K <= 128, N >= K); X is float32 (widened on load) or float64,
 * every other array float64 on the device.  With centre != 0 (KMeans.fit) every kernel reads x - mean(X) and the
 * centres are kept in those centred coordinates; with centre == 0 (kmeans_plusplus) the raw rows.
 *   nnk_kmeans_prepare      : mean (D) = column means (zeros when centre == 0); status[NNK_KM_VAR_MEAN] =
 *                             mean(var(X, axis=0)) (centre != 0), the scale of KMeans' tolerance;
 *   nnk_kmeans_seed         : k-means++ with 2 + int(log K) local trials: centers (K, D) and indices (K).  The
 *                             random draws come from the caller: `first` (the first centre) and rand
 *                             ((K - 1) x trials uniforms in [0, 1)), so a host RandomState is consumed as
 *                             scikit-learn consumes it;
 *   nnk_kmeans_lloyd        : update != 0: one Lloyd iteration from centers -- labels (N), cluster sums (K, D),
 *                             weights (K), status[NNK_KM_CHANGED] labels that changed, status[NNK_KM_EMPTY]
 *                             empty clusters; without empty clusters centers becomes the averages and
 *                             status[NNK_KM_SHIFT] = sum of squared centre shifts.  With empty clusters centers
 *                             is left alone: the caller relocates them (nnk_kmeans_relocate_dist, its own fix of
 *                             sums / weights) and calls nnk_kmeans_average.  update == 0: labels only;
 *   nnk_kmeans_relocate_dist: dist (N) = squared distance of every row to centers[label];
 *   nnk_kmeans_average      : centers = sums / weights (an empty cluster copies the heaviest one), status shift;
 *   nnk_kmeans_inertia      : status[NNK_KM_INERTIA] = sum of squared distances to centers[label],
 *                             status[NNK_KM_DISTINCT] = distinct labels, out_centers = centers + mean.
 * labels must hold -1 (or the previous labels) before the first Lloyd iteration.  Every reduction runs in a fixed
 * order: identical inputs give bit-identical outputs.  Sizes outside the limits are NNK_ERR_UNSUPPORTED. */
#define NNK_KM_CHANGED 0
#define NNK_KM_EMPTY 1
#define NNK_KM_SHIFT 2
#define NNK_KM_INERTIA 3
#define NNK_KM_DISTINCT 4
#define NNK_KM_VAR_MEAN 5
#define NNK_KM_STATUS_LEN 8
typedef struct nnk_kmeans_args {
  const void* X;              /* device (N, x_ld) frames                                               */
  int64_t N, x_ld;
  int32_t dtype;              /* NNK_F32 / NNK_F64 of X                                                */
  int32_t D, K;
  int32_t centre;             /* 1 = KMeans (centred rows), 0 = kmeans_plusplus (raw rows)             */
  int32_t update;             /* nnk_kmeans_lloyd: 1 = assign and update, 0 = assign only              */
  int64_t first;              /* nnk_kmeans_seed: index of the first centre                            */
  const double* rand;         /* device (K - 1, trials): nnk_kmeans_seed's uniform draws               */
  double* centers;            /* device (K, D)                                                         */
  double* sums;               /* device (K, D) cluster sums                                            */
  double* weights;            /* device (K) cluster weights                                            */
  int32_t* labels;            /* device (N)                                                            */
  int64_t* indices;           /* device (K) k-means++ seeds                                            */
  double* mean;               /* device (D)                                                            */
  double* dist;               /* device (N) nnk_kmeans_relocate_dist output                            */
  double* out_centers;        /* device (K, D) nnk_kmeans_inertia output                               */
  double* status;             /* device (NNK_KM_STATUS_LEN)                                            */
  void* workspace;
  size_t workspace_bytes;     /* >= nnk_kmeans_workspace_bytes(N, D, K); 0 = unsupported sizes          */
} nnk_kmeans_args_t;
size_t nnk_kmeans_workspace_bytes(int64_t N, int32_t D, int32_t K);
int nnk_kmeans_prepare(const nnk_kmeans_args_t* args, void* stream);
int nnk_kmeans_seed(const nnk_kmeans_args_t* args, void* stream);
int nnk_kmeans_lloyd(const nnk_kmeans_args_t* args, void* stream);
int nnk_kmeans_relocate_dist(const nnk_kmeans_args_t* args, void* stream);
int nnk_kmeans_average(const nnk_kmeans_args_t* args, void* stream);
int nnk_kmeans_inertia(const nnk_kmeans_args_t* args, void* stream);

/* ---- Merlin post-filter (postfilters/__init__.py:7-62) ------------------------------------------------
 * Per frame c of a flat (N, D) batch (rows at stride ld, float32 or float64), weight w (D doubles on the
 * device): out = w * c with out[0] += log(r0(c) / r0(w * c)) / 2, where r0 = c2acr(freqt(., order, -alpha),
 * 0, fftlen) -- the reference's freqt / c2acr / mc2b / b2mc chain collapsed (mc2b and b2mc are exact
 * inverses outside coefficient 0).  r0 runs on a float64 basis B = Cos F ((fftlen/2 + 1) x D) that
 * nnk_postfilter_basis builds once per (alpha, D, order, fftlen) into `basis` (device, basis_elems =
 * nnk_postfilter_basis_elems(D, fftlen) doubles, opaque order).  Arithmetic is float64, out has the dtype
 * of mgc.  fftlen must be a power of two (SPTK's fftr), 0 <= order <= fftlen - 1 (c2acr's buffer);
 * D > 128 or fftlen > 8192 is NNK_ERR_UNSUPPORTED.  nnk_postfilter_basis_elems returns 0 for such sizes. */
int64_t nnk_postfilter_basis_elems(int32_t D, int32_t fftlen);
int nnk_postfilter_basis(double alpha, int32_t D, int32_t order, int32_t fftlen, double* basis, int64_t basis_elems,
                         void* stream);
int nnk_postfilter_apply(const void* mgc, int32_t dtype, int64_t N, int32_t D, int64_t ld, const double* weight,
                         int32_t fftlen, const double* basis, int64_t basis_elems, void* out, int64_t out_ld,
                         void* stream);

/* ---- corpus normalisation (preprocessing/generic.py:496-828) -----------------------------------------
 * nnk_frame_stats folds the rows of n_utt utterances into a running per-column state (device, float64,
 * 1 + 4*D doubles, in and out): [count, mean[D], m2[D], min[D], max[D]], m2 = sum of squared deviations
 * (= var * count).  Utterance u is rows utt_off[u] .. of a row-major float32 / float64 matrix (row stride
 * ld elements, int64 offsets on the device); it has min(utt_off[u+1] - utt_off[u], lengths[u], max_rows)
 * valid rows (lengths: int32 on the device, NULL = no limit, negative = 0); no other row is read.  The
 * incoming state is merged first (Chan's pairwise formula), so chunks stream through one state.  min / max
 * start from the state's min / max (+inf / -inf for a fresh state).  A NaN propagates into its column's
 * mean, m2, min and max.  Deterministic: fixed tiles, fixed-order fold of per-block partials.
 * workspace >= nnk_frame_stats_workspace_bytes(n_utt, max_rows, D), any contents (reset on the stream).
 *
 * nnk_column_affine: per-column affine map of a contiguous (n_rows, D) matrix in the dtype `dtype`
 * (x may be float32 while dtype is float64; a, b are D-vectors in `dtype` on the device):
 *   form 0: out = (x - a[c]) / b[c]   (scale, inv_minmax_scale)
 *   form 1: out = x * b[c] + a[c]     (inv_scale, minmax_scale)
 * IEEE round-to-nearest for every operation and no contraction: bit-identical to the NumPy expression. */
int64_t nnk_frame_stats_workspace_bytes(int32_t n_utt, int32_t max_rows, int32_t D);
int nnk_frame_stats(const void* X, int32_t dtype, int32_t D, int64_t ld, const int64_t* utt_off,
                    const int32_t* lengths, int32_t n_utt, int32_t max_rows, double* state, void* workspace,
                    int64_t workspace_bytes, void* stream);
int nnk_column_affine(const void* x, int32_t x_dtype, int32_t dtype, int64_t n_rows, int32_t D, const void* a,
                      const void* b, int32_t form, void* out, void* stream);

/* ---- waveform and F0 preprocessing (csrc/nnk_wave.cu; DESIGN.md 3.13) -------------------------------
 * nnk_f0_interp: preprocessing.interp1d on B padded rows of T_max frames (row-major, contiguous); row b
 * is interpolated over [0, lengths[b]) (lengths NULL: T_max), later frames are copied.  kind 0 linear,
 * 1 slinear, 2 zero, 3 nearest, 4 nearest-up, 5 previous, 6 next.  Bit-identical to scipy.
 * nnk_preemphasis: pre-emphasis (inverse 0) or its inverse (inverse 1) along rows of T_max samples,
 * row b over [0, lengths[b]); bit-identical to scipy.signal.lfilter in the input dtype.  The inverse
 * needs the workspace and a 2-word device counter (chunks rerun, samples rewritten by the repair walk).
 * nnk_mulaw: mode 0 mulaw, 1 inv_mulaw, 2 mulaw_quantize (int64 out), 3 inv_mulaw_quantize; variant
 * 0 = float32 NumPy chain (float64 result), 1 = float32 chain, 2 = float64 chain.                    */
int64_t nnk_f0_interp_workspace_bytes(int32_t B, int32_t T_max);
int nnk_f0_interp(const void* x, void* out, int32_t dtype, int32_t B, int32_t T_max, const int32_t* lengths,
                  int32_t kind, void* workspace, int64_t workspace_bytes, void* stream);
int64_t nnk_preemphasis_workspace_bytes(int32_t dtype, int64_t rows, int64_t T_max, double coef, int32_t inverse);
int nnk_preemphasis(const void* x, void* out, int32_t dtype, int64_t rows, int64_t T_max, const int32_t* lengths,
                    double coef, int32_t inverse, void* workspace, int64_t workspace_bytes,
                    unsigned long long* counters, void* stream);
int nnk_mulaw(const void* x, int32_t in_type, void* out, int32_t mode, int32_t variant, int64_t n, double mu,
              void* stream);

/* ---- modulation spectrum (preprocessing/modspec.py; csrc/nnk_modspec.cu; DESIGN.md 3.16) -----------------------
 * nnk_modspec: one CTA per (utterance b, feature column d).  The column's first len_b frames (lengths[b], or
 * T_in when lengths is NULL; later frames are never read) are zero-padded to n and transformed with an n-point
 * real FFT in shared memory (n / 2-point complex FFT and split); Y = fwd_scale * X is the spectrum in the
 * norm's scaling.  K = n / 2 + 1 bins; all arrays are row-major (B, rows, D).
 *   mode 0 (power):   out  = |Y_k|^2, (B, K, D); out2 = Y_k / |Y_k| as interleaved (re, im), (B, K, D, 2),
 *                     or NULL.  A zero bin has phase (+1, 0), or (-1, 0) when its real part is -0.
 *   mode 1 (smooth):  bins k >= limit_bin become Y_k / |Y_k| (log_domain) or 0, then
 *                     out = inv_scale * irfft_unnormalised(Y)[:len_b], (B, T_out, D).
 *   mode 2 (inverse): in = |Y|^2 (B, K, D), in2 = phase (B, K, D, 2); Y = sqrt(in) * in2;
 *                     out = inv_scale * irfft_unnormalised(Y)[:len_b], (B, T_out, D).  The imaginary parts of
 *                     bins 0 and n / 2 are ignored, as numpy.fft.irfft does.
 *   mode 3 (grad):    in2 = dL/d|Y|^2 (B, K, D); out = dL/dx = 2 fwd_scale Re(sum_k G_k conj(Y_k) e^{-2 pi i k t / n})
 *                     for t < len_b, (B, T_out, D).
 *   mode 4 (log power): out = log(max(|Y_k|^2, tiny)), (B, K, D), tiny the smallest normal number of the dtype
 *                     (FLT_MIN, DBL_MIN); out2 must be NULL.  No inverse FFT, like mode 0.
 *   mode 5 (post-filter): in2 = (a, c) interleaved, (K, D, 2), shared by every utterance.  Bin 0 is kept; a bin
 *                     k >= 1 of zero power stays 0, any other becomes Y_k / |Y_k| exp(s' / 2) with
 *                     s' = a s + c, s = log(max(|Y_k|^2, tiny)); then, as mode 1,
 *                     out = inv_scale * irfft_unnormalised(Y)[:len_b], (B, T_out, D).  out2 must be NULL.
 * Frames len_b <= t < T_out of out are written as 0.  n is 256, 512, 1024, 2048 or 4096 (else NNK_ERR_ARG);
 * every len_b must be <= n and <= T_out (<= T_in for the modes that read x). */
#define NNK_MS_POWER 0
#define NNK_MS_SMOOTH 1
#define NNK_MS_INVERSE 2
#define NNK_MS_GRAD 3
#define NNK_MS_LOGPOWER 4
#define NNK_MS_POSTFILTER 5
int nnk_modspec(int32_t mode, int32_t dtype, int32_t n, const void* in, const void* in2, void* out, void* out2,
                int32_t B, int32_t T_in, int32_t T_out, int32_t D, const int32_t* lengths, double fwd_scale,
                double inv_scale, int32_t limit_bin, int32_t log_domain, void* stream);

/* ---- parameter generation considering the modulation spectrum (paramgen.mlpg_ms_batch; csrc/nnk_ms_gen.cu;
 * DESIGN.md 3.18) -----------------------------------------------------------------------------------------------
 * nnk_mlpg_ms: per chain c (one smoothed output column s = c.out_col of one utterance of T <= n frames) and with
 * tau, P, b and c_m = P^-1 b exactly as nnk_mlpg_fwd builds them (edge rule included), Y = rfft(c, n) and
 * s_k(c) = log(max(|Y_k|^2, DBL_MIN)), maximises
 *   F(c) = omega (b^T c - c^T P c / 2) - 1/2 sum_{k=1}^{n/2} q_k (s_k(c) - nu_k)^2,
 *   nu_k = ms_mean[k * args->out_ld + s],  q_k = 1 / ms_var[k * args->out_ld + s]  (q_k = 0 when ms_var is inf)
 * from c0 = c_m by n_iter trials: g = grad of the MS term at c, h = P^-1 g, delta = (c_m - c) + h / omega,
 * c' = c + alpha delta is kept when F(c') >= F(c), otherwise alpha halves (alpha starts at `step`; a rejected
 * trial still counts).  Bin 0 has no term; a bin of power <= DBL_MIN adds a constant and no gradient.
 * omega = weight, or 1 / (nw T) when weight == 0.  Pass-through chains are copied.
 *
 * Everything is float64: args->dtype must be NNK_F64 (callers widen float32 inputs once) and args->out_off
 * NULL.  Every utterance must have T <= n frames (args->max_T <= n); longer ones are left unwritten.  One call
 * enqueues, on `stream` and without a host synchronisation, 2 + 2 n_iter launches: nnk_mlpg_fwd into the
 * workspace, one launch that copies c_m to out and forms the first gradient, then per trial one nnk_mlpg_solve
 * (float64 right-hand side) and one launch of ms_gen_kernel (csrc/nnk_ms_gen.cu).  Non-positive pivots set the
 * status word as for nnk_mlpg_fwd.  The workspace must hold nnk_mlpg_ms_workspace_bytes(): the MLPG factor
 * scratch of the whole batch, c_m and h ((n_rows, out_ld) each), g ((n_rows, n_chain)) and two numbers per
 * chain (F and alpha).  Per-chain sums run in a fixed order inside one CTA, so a chain's result does not depend
 * on the batch around it and repeated calls give the same bits. */
typedef struct nnk_mlpg_ms {
  const double* ms_mean; /* device (n / 2 + 1, args->out_ld): nu, finite where ms_var is finite          */
  const double* ms_var;  /* device (n / 2 + 1, args->out_ld): > 0, inf exempts the bin                    */
  int32_t n;             /* DFT length: 256, 512, 1024, 2048 or 4096                                      */
  int32_t n_iter;        /* >= 0 trials                                                                   */
  double step;           /* > 0 initial step alpha                                                        */
  double weight;         /* omega > 0, or 0 => 1 / (nw T) per utterance                                   */
  int64_t n_rows;        /* rows of means / vars / out (utt_off[n_utt] at most); sizes the workspace      */
} nnk_mlpg_ms_t;

int nnk_mlpg_ms(const nnk_mlpg_args_t* args, const nnk_mlpg_ms_t* ms, void* stream);
size_t nnk_mlpg_ms_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, int64_t n_rows, int64_t out_ld,
                                   const nnk_windows_t* win);

/* ---- segment-level modulation spectrum (postfilters.modspec_*(segment=L), paramgen.mlpg_ms_batch(segment=L);
 * csrc/nnk_ms_segment.cu, csrc/nnk_ms_gen.cu; DESIGN.md 3.16, 3.18) --------------------------------------------
 * nnk_ms_segment: the segment-level MS of Takamichi et al. (ICASSP 2014) over a padded batch x (B, T, D),
 * row-major, in dtype (NNK_F32 / NNK_F64).  Utterance b has len_b = min(max(lengths[b], 0), T) frames
 * (lengths NULL: T); later frames are never read.  With the hop H = L / 2 and the periodic Hann window
 * w_m = 0.5 - 0.5 cos(2 pi m / L), utterance b has J_b = ceil(len_b / H) + 1 segments (0 when len_b = 0);
 * segment j starts at frame (j - 1) H, frames outside [0, len_b) are 0, and Y_j = rfft(w * x[seg j], n),
 * K = n / 2 + 1 bins, s_jk = log(max(|Y_jk|^2, tiny)).
 *   mode 0 (log power):   out (S, D, K) in dtype, S = sum_b J_b: row seg_off[b] + j, column d, bin k holds
 *                         s_jk of column d.  seg_off (B,) int64 on the device, the exclusive prefix sums of J_b
 *                         computed from the same lengths; table is unused (may be NULL).
 *   mode 1 (post-filter): table (K, D, 2) in dtype holds (a, c); every bin k >= 1 of non-zero power becomes
 *                         C_jk = Y_jk / |Y_jk| exp((a s_jk + c) / 2), bin 0 and zero-power bins as for
 *                         nnk_modspec's post-filter; out (B, T, D) = sum_j irfft(C_j, n)[t - (j - 1) H] over
 *                         the segments with 0 <= t - (j - 1) H < L for t < len_b, 0 for len_b <= t < T.
 *                         seg_off is unused (may be NULL).
 * n is 32, 64, 128, 256 or 512 and L even with 4 <= L <= n (else NNK_ERR_ARG).  Every output element is
 * written exactly once, without atomics: repeated calls give the same bits.
 *
 * nnk_mlpg_ms_segment: parameter generation considering the segment-level MS (paramgen.mlpg_ms_batch(segment=L),
 * DESIGN.md 3.18).  args, ms, tau, P, b, c_m = P^-1 b, omega, the start point c0 = c_m and the trials are exactly
 * those of nnk_mlpg_ms; only the MS term differs.  Per chain (one smoothed output column s = c.out_col of one
 * utterance of T >= 1 frames, any T), with the segments of nnk_ms_segment (H = L / 2, J = ceil(T / H) + 1,
 * segment j starts at frame (j - 1) H, frames outside [0, T) are 0, periodic Hann window w),
 * Y_j = rfft(w * c[seg j], n) and s_jk = log(max(|Y_jk|^2, DBL_MIN)), it maximises
 *   F(c) = omega (b^T c - c^T P c / 2) - 1/(2 J) sum_j sum_{k=1}^{n/2} q_k (s_jk - nu_k)^2
 * (nu_k, q_k from ms->ms_mean / ms->ms_var as for nnk_mlpg_ms): the mean of the utterance level's term over the J
 * segments, edge segments included.  Bin 0 has no term; a bin of power <= DBL_MIN adds a constant and no
 * gradient; ms_var = inf exempts a bin.  The gradient at frame t = (j - 1) H + m (0 <= m < L) is
 *   g_t = 1/J sum_{j containing t} w_m [n irfft(C_j, n)]_m,  C_jk = -q_k (s_jk - nu_k) / |Y_jk|^2 Y_jk
 * (C_j,n/2 doubled, C_j0 = 0): every frame lies in two segments, so g_t is one addition of two terms.
 * ms->n is 32, 64, 128, 256 or 512 and L even with 4 <= L <= n; there is no limit on args->max_T.  NNK_ERR_ARG:
 * args or ms NULL, dtype not NNK_F64, out_off not NULL, a negative size, a bad n or L, n_iter < 0, step <= 0,
 * weight < 0 or NaN, a NULL device pointer or NULL ms_mean / ms_var.  The workspace is
 * nnk_mlpg_ms_workspace_bytes() of the same arguments.  One call enqueues 2 + 2 n_iter launches on `stream`
 * without a host synchronisation, whatever the batch and T: nnk_mlpg_fwd, one launch that copies c_m to out and
 * forms the first gradient, then per trial one nnk_mlpg_solve and one launch of ms_gen_segment_kernel
 * (csrc/nnk_ms_gen.cu).  Non-positive pivots set the status word as for nnk_mlpg_ms.  Sums run in a fixed order
 * inside one CTA per chain, so a chain's bits do not depend on the batch and repeated calls give the same bits. */
#define NNK_MSSEG_LOGPOWER 0
#define NNK_MSSEG_POSTFILTER 1
int nnk_ms_segment(int32_t mode, int32_t dtype, int32_t n, int32_t L, const void* x, const void* table, void* out,
                   int32_t B, int32_t T, int32_t D, const int32_t* lengths, const int64_t* seg_off, void* stream);
int nnk_mlpg_ms_segment(const nnk_mlpg_args_t* args, const nnk_mlpg_ms_t* ms, int32_t L, void* stream);

/* ---- parameter generation from mixture outputs (paramgen.mlpg_mixture_batch; csrc/nnk_mix_gen.cu;
 * DESIGN.md 3.19) -----------------------------------------------------------------------------------------------
 * nnk_mix_gen: one launch of mix_gen_kernel, the E-step side of the EM of paramgen.mlpg_mixture_batch (Tokuda et
 * al., ICASSP 2000).  Frame r (a row of the batch) has M components: log-weights lw[r, m] (log_weights,
 * (n_rows, M)), means mu[r, m, i] and variances s2[r, m, i] (means / vars, (n_rows, M, D)), all of `dtype` and
 * row-major; float32 inputs are widened in registers and every operation is float64.  Utterance u has rows
 * utt_off[u] .. utt_off[u] + utt_len[u] - 1 and the tiles tile_off[u] .. tile_off[u + 1] - 1 of
 * NNK_MIX_GEN_TILE frames (n_tiles = tile_off[n_utt]); rows outside every utterance are never read or written.
 * col_map[i] describes input column i:
 *   -1                        the column takes no part (no chain reads it);
 *   (out_col << 3) | 0        a copied column: Y_t[i] = c[t, out_col];
 *   (out_col << 3) | (w + 1)  window w of a smoothed column: Y_t[i] = sum_j coef_w[j] c[t + j, out_col], with
 *                             c = 0 outside the utterance.
 * On the first and last H = max_w max(l_w, u_w) frames of an utterance, and on every frame when H = 0, only the
 * copied columns and those of window 0 count; elsewhere every column with col_map >= 0 counts.
 *   NNK_MIX_GEN_SELECT:    per frame the component a with the largest lw (the lowest index on ties) goes to
 *                          E[r, :] = mu[r, a, :], V[r, :] = s2[r, a, :]; every component's log-normaliser
 *                          lnorm[r, m] = lw[r, m] - 1/2 sum_{counted i} (log s2[r, m, i] + log 2 pi) goes to
 *                          lnorm.  Data errors set *status_word (below).
 *   NNK_MIX_GEN_ESTEP:     with l[r, m] = lnorm[r, m] - 1/2 sum_{counted i} (Y_r[i] - mu[r, m, i])^2 / s2[r, m, i]
 *                          and gamma its softmax over m: P = sum_m gamma / s2, E[r, i] = (sum_m gamma mu / s2) / P
 *                          and V[r, i] = 1 / P for every column with col_map >= 0 (0 and 1 for the others).
 *                          With ll_part, ll_part[tile] = sum over the tile's frames, in frame order, of
 *                          log sum_m exp(l[r, m]).
 *   NNK_MIX_GEN_OBJECTIVE: ll_part only (required).
 * c (rows of c_ld doubles, the first c_cols staged per tile) is read by ESTEP and OBJECTIVE only.
 * Status word (device, zeroed by the caller): 0, or ~((row << 2) | kind) of the first failing row, lowest kind
 * first: kind 1 = a NaN or +inf log-weight, 2 = every log-weight -inf, 3 = a variance of a column with
 * col_map >= 0 that is not positive and finite.  Results of a failing call are undefined but never fault.
 * Errors: NNK_ERR_ARG for NULL pointers, bad sizes, a bad mode, dtype or window set; NNK_ERR_UNSUPPORTED for
 * D > NNK_MIX_GEN_MAX_D or M > NNK_MIX_GEN_MAX_M; all before anything touches the device.  Every output element
 * is written by one thread in a fixed order: repeated calls give the same bits. */
#define NNK_MIX_GEN_SELECT 0
#define NNK_MIX_GEN_ESTEP 1
#define NNK_MIX_GEN_OBJECTIVE 2
#define NNK_MIX_GEN_TILE 32    /* frames per tile */
#define NNK_MIX_GEN_MAX_D 256  /* input columns   */
#define NNK_MIX_GEN_MAX_M 64   /* components      */

typedef struct nnk_mix_gen_args {
  const void* log_weights; /* device (n_rows, M) of dtype                                                   */
  const void* means;       /* device (n_rows, M, D) of dtype                                                */
  const void* vars;        /* device (n_rows, M, D) of dtype                                                */
  int32_t dtype;           /* NNK_F32 / NNK_F64                                                             */
  int32_t M;               /* components, 1 .. NNK_MIX_GEN_MAX_M                                            */
  int32_t D;               /* input columns, 1 .. NNK_MIX_GEN_MAX_D                                         */
  int32_t n_utt;           /* >= 1                                                                          */
  const int32_t* utt_off;  /* device (n_utt): first row of each utterance                                   */
  const int32_t* utt_len;  /* device (n_utt): frames of each utterance                                      */
  const int32_t* tile_off; /* device (n_utt + 1): first tile of each utterance                              */
  int32_t n_tiles;         /* tile_off[n_utt]                                                               */
  const int32_t* col_map;  /* device (D)                                                                    */
  nnk_windows_t win;
  int32_t mode;            /* NNK_MIX_GEN_SELECT / _ESTEP / _OBJECTIVE                                      */
  const double* c;         /* device, ESTEP / OBJECTIVE: current trajectories, row r at c + r * c_ld        */
  int64_t c_ld;
  int32_t c_cols;          /* columns of c the column map addresses (out_col < c_cols <= c_ld)             */
  double* lnorm;           /* device (n_rows, M): written by SELECT, read by ESTEP / OBJECTIVE              */
  double* E;               /* device (n_rows, D): written by SELECT / ESTEP                                 */
  double* V;               /* device (n_rows, D): written by SELECT / ESTEP                                 */
  double* ll_part;         /* device (n_tiles) or NULL (ESTEP); required for OBJECTIVE                      */
  uint64_t* status_word;   /* device, SELECT                                                                */
} nnk_mix_gen_args_t;

int nnk_mix_gen(const nnk_mix_gen_args_t* args, void* stream);

/* ---- trajectory-model log-likelihood (paramgen.trajectory_log_likelihood_batch; csrc/nnk_mlpg.cu;
 * DESIGN.md 3.20) -----------------------------------------------------------------------------------------------
 * nnk_mlpg_traj_ll: one launch of mlpg_kernel in MODE_TLL / MODE_TLL_GRAD per workspace wave.  Per chain c of
 * utterance u (a static column, exactly as nnk_mlpg_fwd sees it: T frames, tau_{t,w} = 1 / var with the edge rule
 * of nnk_mlpg_fwd, mu_{t,w}, P = sum_w W_w^T diag(tau_w) W_w, b = sum_w W_w^T (tau_w mu_w), cbar = P^-1 b,
 * P = L D L^T with pivots d_t) and its target static trajectory x (x_t at targets[(out_off or utt_off)[u] + t) *
 * tgt_ld + chains[c].out_col]), the Gaussian trajectory model N(x; cbar, P^-1) (Zen, Tokuda & Kitamura 2007) has
 * the log-likelihood
 *
 *   l = 1/2 sum_t log d_t - 1/2 sum_{t,w} tau_{t,w} (u_{t,w} - ubar_{t,w})^2 - (T/2) log 2 pi,
 *   u_{t,w} = (W_w x)_t,  ubar_{t,w} = (W_w cbar)_t,
 *
 * written to ll[u * n_chain + c] (0 for copied chains, flags & 1).  With grad != 0 the gradients are written too,
 * with w_t row t of W_w and Sigma = P^-1:
 *
 *   dl/dmu_{t,w}   = tau_{t,w} (u_{t,w} - ubar_{t,w})                                         -> grad_means
 *   dl/dvar_{t,w}  = -tau_{t,w}^2 / 2 [w_t^T Sigma w_t - (u_{t,w} - mu_{t,w})^2 + (ubar_{t,w} - mu_{t,w})^2]
 *   dl/dx          = -P (x - cbar) = -sum_w W_w^T (dl/dmu_{.,w})                               -> grad_targets
 *
 * grad_means has the rows of means (utt_off[u] + t) and columns chains[c].in_col + w * win_stride with row stride
 * gm_ld; grad_targets has the rows and columns of the targets with row stride gx_ld; both are of `dtype`.  Per-frame
 * variances (var_ld > 0): grad_vars has the layout of grad_means with row stride gv_ld, of `dtype`.  Global (D,)
 * variances (var_ld == 0): grad_vars is a float64 (n_utt, gv_ld) array and grad_vars[u * gv_ld + column] is the
 * sum of the per-frame values over the utterance's frames.  Only the elements of solved chains at frames
 * 0 .. T - 1 are written: the caller zeroes the others.  Where the edge rule sets tau to zero, both gradients are 0.
 * Every sum runs in a fixed order in one thread, so a chain's results do not depend on the batch and repeated calls
 * give the same bits.  Arithmetic is float64; float32 inputs are widened exactly as nnk_mlpg_fwd widens them.
 * Targets and means are not checked: non-finite values give NaN.  A pivot d_t <= 0 sets the status word as
 * nnk_mlpg_fwd does.  Errors: NNK_ERR_ARG for NULL pointers or bad sizes, NNK_ERR_UNSUPPORTED for a window set no
 * instance serves, NNK_ERR_WORKSPACE for a workspace below one utterance's share of
 * nnk_mlpg_traj_ll_workspace_bytes; all before anything is launched.  args->out, grad_out, go_ld and go_f64 are
 * not used. */
typedef struct nnk_traj_ll {
  const void* targets; /* device, dtype: target static trajectories (rows and columns of the nnk_mlpg_fwd output) */
  int64_t tgt_ld;      /* row stride of targets, in elements                                                      */
  double* ll;          /* device (n_utt, n_chain) float64                                                         */
  int32_t grad;        /* 0: ll only; 1: ll and the three gradients                                               */
  void* grad_means;    /* device, dtype, rows and columns of means                                                */
  int64_t gm_ld;
  void* grad_vars;     /* device: per-frame, dtype, rows and columns of vars; global, float64 (n_utt, gv_ld)      */
  int64_t gv_ld;
  void* grad_targets;  /* device, dtype, rows and columns of targets                                              */
  int64_t gx_ld;
} nnk_traj_ll_t;

int nnk_mlpg_traj_ll(const nnk_mlpg_args_t* args, const nnk_traj_ll_t* tl, void* stream);
size_t nnk_mlpg_traj_ll_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

/* ---- sampling from the trajectory model (paramgen.trajectory_sample_batch; csrc/nnk_mlpg.cu; DESIGN.md 3.21) ---
 * nnk_mlpg_traj_sample: one launch of mlpg_kernel in MODE_SAMPLE per workspace wave.  Per chain c of utterance u
 * (a static column, exactly as nnk_mlpg_fwd sees it: T frames, tau_{t,w} = 1 / var with the edge rule of
 * nnk_mlpg_fwd, P = sum_w W_w^T diag(tau_w) W_w, b = sum_w W_w^T (tau_w mu_w), and the top-down factorisation
 * P = L D L^T with unit lower L, pivots d_t, multipliers l_j[t] = L[t+j][t] and zs_t = (L^-1 b)_t / d_t),
 * sample s = 0 .. n_samples - 1 is
 *
 *   y_t = zs_t + scale * z_{s,t} / sqrt(d_t) - sum_{j=1..S} l_j[t] y_{t+j}      (t = T-1 .. 0, y_t = 0 for t >= T)
 *
 * that is y = L^-T (D^-1 L^-1 b + scale D^-1/2 z) ~ N(cbar, scale^2 P^-1), cbar = P^-1 b, for z ~ N(0, I).  It is
 * written in the dtype of the inputs to args->out + s * sample_stride at row (out_off or utt_off)[u] + t, column
 * chains[c].out_col, row stride out_ld.  With scale = 0 the recurrence is nnk_mlpg_fwd's backward sweep term for
 * term.  Copied chains (flags & 1) get the means column, unchanged and without noise, in every sample.  Elements
 * no chain writes are not touched.  Arithmetic is float64; float32 inputs are widened exactly as nnk_mlpg_fwd
 * widens them.
 *
 * The noise z_{s,t} of chain c of utterance u is a pure function of (seed, key_u, s, t, out_col = chains[c].out_col):
 * it does not depend on the batch around the utterance, the layout, the padding, the dtype, n_samples or the
 * workspace waves.  Normative definition:
 *
 *   Philox4x32-10 (Salmon, Moraes, Dror & Shaw, SC 2011) with multipliers M0 = 0xD2511F53, M1 = 0xCD9E8D57 and key
 *   increments W0 = 0x9E3779B9, W1 = 0xBB67AE85.  A round maps the counter (c0, c1, c2, c3) to
 *     (hi(M1 * c2) ^ c1 ^ k0, lo(M1 * c2), hi(M0 * c0) ^ c3 ^ k1, lo(M0 * c0))
 *   (hi / lo: upper / lower 32 bits of the 64-bit product); after each of the first nine rounds the key becomes
 *   (k0 + W0, k1 + W1) mod 2^32.  Ten rounds give the output words (r0, r1, r2, r3).
 *     key      (k0, k1)         = (seed mod 2^32, seed >> 32)
 *     counter  (c0, c1, c2, c3) = (t >> 1, out_col, s, key_u),   key_u = keys ? keys[u] : u
 *   u is the caller's utterance index (the index into utt_off), never a position in args->order.
 *     N_U = (r0 >> 6) * 2^26 + (r1 >> 6),   U = (N_U + 0.5) * 2^-52   in (0, 1)
 *     N_V = (r2 >> 6) * 2^26 + (r3 >> 6),   V = N_V * 2^-52           in [0, 1)
 *     R = sqrt(-2 log U),   z_{s,t} = R cos(2 pi V) for even t,  R sin(2 pi V) for odd t   (Box & Muller 1958)
 *   so one Philox call serves frames 2k and 2k + 1 of one chain and sample.  Known answers of the rounds
 *   (Random123's philox4x32-10 vectors): counter 0, key 0 -> 6627e8d5 e169c58d bc57ac4c 9b00dbd8; all ones ->
 *   408f276d 41c83b0e a20bc7c6 6d5451fd; counter 243f6a88 85a308d3 13198a2e 03707344, key a4093822 299f31d0 ->
 *   d16cfe09 94fdcceb 5001e420 24126ea1.
 *
 * A pivot d_t <= 0 sets the status word as nnk_mlpg_fwd does.  Errors: NNK_ERR_ARG for NULL pointers, bad sizes,
 * n_samples < 1, sample_stride < 0 or a scale that is negative or not finite; NNK_ERR_UNSUPPORTED for a window set
 * no instance serves; NNK_ERR_WORKSPACE for a workspace below one utterance's share of
 * nnk_mlpg_traj_sample_workspace_bytes; all before anything is launched.  args->grad_out, go_ld and go_f64 are
 * not used. */
typedef struct nnk_traj_sample {
  int64_t sample_stride; /* elements between samples in args->out                                        */
  int32_t n_samples;     /* >= 1                                                                           */
  uint64_t seed;
  const uint32_t* keys;  /* device (n_utt,), or NULL for key_u = u                                         */
  double scale;          /* >= 0, finite                                                                   */
} nnk_traj_sample_t;

int nnk_mlpg_traj_sample(const nnk_mlpg_args_t* args, const nnk_traj_sample_t* ts, void* stream);
size_t nnk_mlpg_traj_sample_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

/* ---- the gradient of MLPG in its means and variances (paramgen.mlpg_vjp_batch; csrc/nnk_mlpg.cu;
 * DESIGN.md 3.22) -----------------------------------------------------------------------------------------------
 * nnk_mlpg_vjp: one launch of mlpg_kernel in MODE_VJP per workspace wave.  Per chain c of utterance u (a static
 * column, exactly as nnk_mlpg_fwd sees it: T frames, tau_{t,w} = 1 / var with the edge rule of nnk_mlpg_fwd,
 * mu_{t,w}, P = sum_w W_w^T diag(tau_w) W_w, b = sum_w W_w^T (tau_w mu_w), cbar = P^-1 b, the trajectory
 * nnk_mlpg_fwd writes) and the gradient o = dL/dcbar of a loss L with respect to that trajectory (o_t at
 * grad_out[((out_off or utt_off)[u] + t) * go_ld + chains[c].out_col], of `dtype`), with g = P^-1 o:
 *
 *   dL/dmu_{t,w}  = tau_{t,w} (W_w g)_t                                                      -> grad_means
 *   dL/dvar_{t,w} = -tau_{t,w}^2 (W_w g)_t (mu_{t,w} - (W_w cbar)_t)                          -> grad_vars
 *
 * (Wu & Wang 2006: minimum generation error training through MLPG in both).  Where the edge rule sets tau to zero,
 * both gradients are 0.  Copied chains (flags & 1) pass o through: dL/dmu = o, and their dL/dvar is not written.
 * grad_means has the rows of means (utt_off[u] + t) and columns chains[c].in_col + w * win_stride with row stride
 * gm_ld, of `dtype`.  Per-frame variances (var_ld > 0): grad_vars has the layout of grad_means with row stride
 * gv_ld, of `dtype`.  Global (D,) variances (var_ld == 0): grad_vars is a float64 (n_utt, gv_ld) array and
 * grad_vars[u * gv_ld + column] is the sum of the per-frame values over the utterance's frames.  Only the elements
 * of chains at frames 0 .. T - 1 are written: the caller zeroes the others.  Every sum runs in a fixed order in one
 * thread, so a chain's results do not depend on the batch and repeated calls give the same bits.  Arithmetic is
 * float64; float32 inputs are widened exactly as nnk_mlpg_fwd widens them, and the results are stored in `dtype`.
 * Means and grad_out are not checked: non-finite values give NaN.  A pivot d_t <= 0 sets the status word as
 * nnk_mlpg_fwd does.  Errors: NNK_ERR_ARG for NULL pointers or bad sizes, NNK_ERR_UNSUPPORTED for a window set no
 * instance serves, NNK_ERR_WORKSPACE for a workspace below one utterance's share of nnk_mlpg_vjp_workspace_bytes;
 * all before anything is launched.  args->out, args->grad_out, args->go_ld, args->out_ld and args->go_f64 are not
 * used. */
typedef struct nnk_mlpg_vjp {
  const void* grad_out; /* device, dtype: dL/dcbar (rows and columns of the nnk_mlpg_fwd output)                  */
  int64_t go_ld;        /* row stride of grad_out, in elements                                                     */
  void* grad_means;     /* device, dtype, rows and columns of means                                                */
  int64_t gm_ld;
  void* grad_vars;      /* device: per-frame, dtype, rows and columns of vars; global, float64 (n_utt, gv_ld)      */
  int64_t gv_ld;
} nnk_mlpg_vjp_t;

int nnk_mlpg_vjp(const nnk_mlpg_args_t* args, const nnk_mlpg_vjp_t* vj, void* stream);
size_t nnk_mlpg_vjp_workspace_bytes(int32_t n_utt, int32_t n_chain, int32_t max_T, const nnk_windows_t* win);

/* ---- sharded batches (SURVEY.md 8e; the reference has no multi-device path) ------------------------
 * Copies n_seg row segments (whole utterances) between two row-major device matrices:
 * dst[dst_row[s] + r, 0:cols] = src[src_row[s] + r, 0:cols] for r < len[s].  Used to bring the
 * all-gathered trajectories (shard order: bucket, rank, utterance) back into the caller's utterance
 * order, i.e. the order the reference's per-utterance loop over paramgen.mlpg
 * (paramgen/_mlpg.py:92) would have produced them in.  elem_bytes 4 or 8; n_seg <= 65535 per call. */
int nnk_segment_copy(const void* src, void* dst, int32_t elem_bytes, int64_t cols, int64_t src_ld, int64_t dst_ld,
                     const int64_t* src_row, const int64_t* dst_row, const int32_t* len, int32_t n_seg,
                     int32_t max_len, void* stream);

/* Peer-memory transport of a sharded result (one process per GPU of one NVLink / NVSwitch box):
 * a cudaMalloc allocation per rank, shared through CUDA IPC handles; nnk_peer_copy pushes a byte range
 * into a peer's mapping with copy-engine DMA over NVLink (no SMs: it overlaps the solve kernels, which
 * an NCCL all-gather kernel cannot while they hold every SM slot).  The 64-byte handle travels between
 * the processes by any host channel (torch.distributed here).                                       */
int nnk_peer_alloc(size_t bytes, void** ptr);
int nnk_peer_free(void* ptr);
int nnk_peer_export(const void* ptr, unsigned char* handle64);
int nnk_peer_open(const unsigned char* handle64, void** ptr);
int nnk_peer_close(void* ptr);
int nnk_peer_copy(void* dst_peer, const void* src_local, size_t bytes, void* stream);

const char* nnk_last_error(void);
int nnk_abi_version(void);
/* Number of kernel launches this library has issued since load (bench.py's gpu_launches).       */
int64_t nnk_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* NNK_B200_H */
