// nnk_mlpg.cuh -- declarations shared by the MLPG kernels (nnk_mlpg.cu, nnk_mlpg_as.cuh).
#pragma once
#include "nnk_common.cuh"

namespace nnk {

// MODE_GV: the forward solve followed by the global-variance refinement of nnk_mlpg_gv (mlpg_kernel only).
// MODE_TLL / MODE_TLL_GRAD: the trajectory-model log-likelihood of nnk_mlpg_traj_ll, without / with its
// gradients (mlpg_kernel only).  MODE_SAMPLE: samples of the trajectory model of nnk_mlpg_traj_sample (mlpg_kernel
// only).  MODE_VJP: the gradients of the forward solve in its means and variances, nnk_mlpg_vjp (mlpg_kernel only).
enum { MODE_FWD = 0, MODE_GRAD = 1, MODE_SOLVE = 2, MODE_GV = 3, MODE_TLL = 4, MODE_TLL_GRAD = 5, MODE_SAMPLE = 6,
       MODE_VJP = 7 };

// scratch columns per frame of one work item: the S + 1 factor columns, in MODE_GV four more (pivot d, c_m, and
// the current / trial trajectory), in the MODE_TLL pair one more (1 / d), in MODE_SAMPLE one more (1 / sqrt(d)), in
// MODE_VJP one more ((L^-1 o)_t / d_t)
template <int MODE, int NT>
struct WsCols {
  static constexpr int value =
      NT + (MODE == MODE_GV ? 4
            : (MODE == MODE_TLL || MODE == MODE_TLL_GRAD || MODE == MODE_SAMPLE || MODE == MODE_VJP) ? 1 : 0);
};

template <int NW, int L, int U>
struct WinTab {
  static constexpr int S = L + U;
  static constexpr int NT = L + U + 1;
  double c[NW][NT];         // c[w][L + k] = W_w[t, t + k]   (zero padded to the common (L, U))
  double q[NW][S + 1][NT];  // q[w][m][i] = c[w][i] * c[w][i + m]
  int nw;                   // real number of windows (<= NW)
  int m_edge;               // max_w max(l_w, u_w): dynamic windows get zero precision at that many
                            // edge frames (paramgen/_mlpg.py:177, 190-193)
};

template <typename Tin, int NW, int L, int U>
struct MlpgParams {
  const Tin* means;
  const Tin* vars;
  const void* go;
  int go_f64;
  void* out;
  int64_t in_ld, var_ld, go_ld, out_ld;
  const int64_t* utt_off;
  const int64_t* out_off;  // first output row per utterance (NULL: utt_off)
  const int32_t* utt_len;
  const int32_t* order;
  const nnk_chain_t* chains;
  int n_utt, n_chain, n_groups, max_T, urank0;
  double* ws;
  unsigned long long* status;
  WinTab<NW, L, U> win;
  // MODE_GV only (see nnk_mlpg_gv_t); the other modes leave them zero
  const double* gv_mean;
  const double* gv_var;
  double gv_step, gv_weight;
  int gv_n_iter;
};

// MODE_TLL / MODE_TLL_GRAD: MlpgParams plus the targets and outputs of nnk_traj_ll_t.  Only those instances take
// it (KernelParams), so every other instance keeps MlpgParams and its parameter layout.
template <typename Tin, int NW, int L, int U>
struct TllParams : MlpgParams<Tin, NW, L, U> {
  const Tin* targets;
  int64_t tgt_ld;
  double* ll;  // (n_utt, n_chain)
  Tin* grad_means;
  int64_t gm_ld;
  void* grad_vars;  // Tin rows of gv_ld, or (n_utt, gv_ld) float64 partials for global variances
  int64_t gv_ld;
  Tin* grad_targets;
  int64_t gx_ld;
};

// MODE_SAMPLE: MlpgParams plus the sample count, stride, seed, keys and scale of nnk_traj_sample_t
template <typename Tin, int NW, int L, int U>
struct SampleParams : MlpgParams<Tin, NW, L, U> {
  int64_t sample_stride;  // elements between samples in out
  int n_samples;
  unsigned long long seed;
  const uint32_t* keys;  // (n_utt,) or NULL: key_u = u
  double scale;
};

// MODE_VJP: MlpgParams (grad_out and go_ld in go / go_ld, of Tin) plus the outputs of nnk_mlpg_vjp_t
template <typename Tin, int NW, int L, int U>
struct VjpParams : MlpgParams<Tin, NW, L, U> {
  Tin* grad_means;
  int64_t gm_ld;
  void* grad_vars;  // Tin rows of gv_ld, or (n_utt, gv_ld) float64 partials for global variances
  int64_t gv_ld;
};

template <typename Tin, int NW, int L, int U, int MODE>
struct KernelParams {
  using type = MlpgParams<Tin, NW, L, U>;
};
template <typename Tin, int NW, int L, int U>
struct KernelParams<Tin, NW, L, U, MODE_TLL> {
  using type = TllParams<Tin, NW, L, U>;
};
template <typename Tin, int NW, int L, int U>
struct KernelParams<Tin, NW, L, U, MODE_TLL_GRAD> {
  using type = TllParams<Tin, NW, L, U>;
};
template <typename Tin, int NW, int L, int U>
struct KernelParams<Tin, NW, L, U, MODE_SAMPLE> {
  using type = SampleParams<Tin, NW, L, U>;
};
template <typename Tin, int NW, int L, int U>
struct KernelParams<Tin, NW, L, U, MODE_VJP> {
  using type = VjpParams<Tin, NW, L, U>;
};

}  // namespace nnk
