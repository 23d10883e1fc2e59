// nnk_dtw.cu -- DTW / FastDTW alignment on sm_90a: one thread block per utterance pair walks the
// anti-diagonals of the accumulated-cost matrix (wavefront), local cost computed in registers.
//
// Replaces the per-pair body of DTWAligner.transform / IterativeDTWAligner.transform
// (preprocessing/alignment.py:48-54, :136-143):
//       dist, path = fastdtw(x, y, radius=self.radius, dist=self.dist)
// i.e. the third-party `fastdtw` package (slaypni/fastdtw; unpinned dependency, setup.py:139) whose
// published algorithm is restated here: inputs as float64; recursion until a series is shorter
// than radius+2 (full DTW there); halve by averaging adjacent frames; project the coarse path,
// dilated by `radius`, onto the fine grid; DP restricted to that per-row window
//       D[i,j] = dt + first-min(D[i-1,j], D[i,j-1], D[i-1,j-1])      (order: up, left, diagonal)
// and backtrack.  radius < 0 selects the exact DTW (full window) -- the same kernel with the window
// test compiled out.  The whole recursion of one pair runs inside one CTA: coarse levels, window
// expansion, DP and backtrack never leave the SM except for the float64 level copies of the series
// (L2-resident scratch) and, in exact mode, the 1 byte/cell back-pointers.
//
// Local cost (cost_kind): 1 = metrics.melcd(x, y) on two frames = (10/ln10*sqrt2) * sqrt(sum((x-y)^2))
// (metrics/__init__.py:5,52-57), 0 = the default lambda x, y: norm(x - y) (alignment.py:35).  The
// squared differences are summed in float64 in the exact order of numpy's pairwise add-reduce so
// that costs, ties and therefore back-track indices are bit-identical to the CPU oracle.
#include <math_constants.h>
#include <stdlib.h>

#include "nnk_common.cuh"

namespace nnk {

// The parameters of all four kernels: the common part, then each path's own fields.
struct DtwParams {
  const void* X;
  const void* Y;
  int is_f64;  // fastdtw_kernel only: the exact kernels take the dtype as a template parameter
  int64_t x_pair_stride, y_pair_stride;
  int x_ld, y_ld, D;
  const int32_t* len_x;
  const int32_t* len_y;
  const int32_t* order;
  int cost_kind, radius;
  int32_t* path_i;
  int32_t* path_j;
  int path_ld;
  int32_t* path_len;
  double* dist;
  long long* cells;
  int max_tx, max_ty;
  double logdb;
  // FastDTW
  unsigned char* ws;
  size_t ws_pair_bytes, series_doubles;
  int smem_bp_cap;  // bytes of back-pointer space available in shared memory
  size_t cost_cap;  // doubles of per-pair cost buffer
  unsigned long long* prof;  // optional [8] cycle counters (NNK_DTW_PROF=1): build, window, cost, wavefront, backtrack
  // exact, two-pass: the chunk being run
  int first;             // rank of the chunk's first pair in `order`
  int n_pairs;           // pairs in this chunk
  double* cost;          // [chunk][max_tx * max_ty]
  unsigned char* bp;     // [chunk][max_tx * max_ty]
  // exact, fused
  uint32_t* bp_words;    // [pair slot][max_tx][wpr]
  int wpr;               // back-pointer words per row = ceil(max_ty / 16)
};

// A pair with an empty series has an empty path.
__device__ __forceinline__ void store_empty_pair(const DtwParams& p, int pair) {
  if (threadIdx.x == 0) { p.path_len[pair] = 0; p.dist[pair] = 0.0; if (p.cells) p.cells[pair] = 0; }
}

// The back-track wrote path_i / path_j[:n] from the last cell back: reverse them in place (all NT threads of
// the block), then store the length (-1: the path did not fit path_ld) and the cell count.
template <int NT>
__device__ __forceinline__ void store_path(const DtwParams& p, int pair, int n, long long cells) {
  if (n > 0) {
    int32_t* pi = p.path_i + (size_t)pair * p.path_ld;
    int32_t* pj = p.path_j + (size_t)pair * p.path_ld;
    for (int a = threadIdx.x; a < n / 2; a += NT) {
      const int b = n - 1 - a;
      const int32_t ti = pi[a], tj = pj[a];
      pi[a] = pi[b]; pj[a] = pj[b];
      pi[b] = ti; pj[b] = tj;
    }
  }
  if (threadIdx.x == 0) {
    p.path_len[pair] = n;
    if (p.cells) p.cells[pair] = cells;
  }
}

// One cell of the recurrence, D[i,j] = first-min(up, left, diagonal), each candidate being that predecessor
// plus the cell's cost: the fastdtw package's tie order.  `dir` is the 2-bit back-pointer: 0 up, 1 left,
// 2 diagonal.  Callers add the cost to each predecessor next to its load: adding it here, after all three
// loads, gives dtw_dp_kernel<16> 107 registers instead of 76 (CUDA 12.9).
struct Relaxed {
  double best;
  uint32_t dir;
};
__device__ __forceinline__ Relaxed relax(double up, double left, double diag) {
  Relaxed r{up, 0};
  if (left < r.best) { r.best = left; r.dir = 1; }
  if (diag < r.best) { r.best = diag; r.dir = 2; }
  return r;
}

// doubles per staged frame: even, and stride/2 odd, so that LDS.128 is bank-conflict free
__host__ __device__ __forceinline__ int dtw_row_stride(int D) {
  int dp = (D + 1) & ~1;
  if (((dp >> 1) & 1) == 0) dp += 2;
  return dp;
}

// numpy DOUBLE_pairwise_sum order over a[k] = (x[k]-y[k])^2 without materialising a[]; the operands
// are widened to float64 first (fastdtw: np.asanyarray(x, dtype='float')), which is exact
template <typename T>
__device__ __forceinline__ double sq(const T* __restrict__ x, const T* __restrict__ y, int k) {
  const double z = __dsub_rn((double)x[k], (double)y[k]);
  return __dmul_rn(z, z);  // never contracted into an FMA: numpy multiplies, then adds
}
template <typename T>
__device__ __forceinline__ double strided8(const T* x, const T* y, int j, int n8) {
  double r = sq(x, y, j);
  for (int i = 8; i < n8; i += 8) r = __dadd_rn(r, sq(x, y, i + j));
  return r;
}
template <typename T>
__device__ double pairwise_block(const T* x, const T* y, int n) {  // n <= 128
  if (n < 8) {
    double res = -0.0;
    for (int i = 0; i < n; ++i) res = __dadd_rn(res, sq(x, y, i));
    return res;
  }
  const int n8 = n - (n % 8);
  const double s01 = __dadd_rn(strided8(x, y, 0, n8), strided8(x, y, 1, n8));
  const double s23 = __dadd_rn(strided8(x, y, 2, n8), strided8(x, y, 3, n8));
  const double s0123 = __dadd_rn(s01, s23);
  const double s45 = __dadd_rn(strided8(x, y, 4, n8), strided8(x, y, 5, n8));
  const double s67 = __dadd_rn(strided8(x, y, 6, n8), strided8(x, y, 7, n8));
  double res = __dadd_rn(s0123, __dadd_rn(s45, s67));
  for (int i = n8; i < n; ++i) res = __dadd_rn(res, sq(x, y, i));
  return res;
}
template <typename T>
__device__ double pairwise_sumsq(const T* x, const T* y, int n) {
  if (n <= 128) return pairwise_block(x, y, n);
  int n2 = n / 2;
  n2 -= n2 % 8;
  return __dadd_rn(pairwise_sumsq(x, y, n2), pairwise_sumsq(x + n2, y + n2, n - n2));
}

// pairwise_sumsq for a frame of x held in registers, D in [8*NB8, 8*NB8 + 7] (ntail = D - 8*NB8): the
// eight accumulators over blocks 0..NB8-1, numpy's fold of them, then the tail in order
template <int NB8>
__device__ __forceinline__ double sumsq_reg(const double (&xreg)[NB8 * 8 + 8], const double* yr, int ntail) {
  double r[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) { const double z = __dsub_rn(xreg[q], yr[q]); r[q] = __dmul_rn(z, z); }
#pragma unroll
  for (int bk = 1; bk < NB8; ++bk) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const double z = __dsub_rn(xreg[bk * 8 + q], yr[bk * 8 + q]);
      r[q] = __dadd_rn(r[q], __dmul_rn(z, z));
    }
  }
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                         __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
#pragma unroll
  for (int e = 0; e < 7; ++e)
    if (e < ntail) { const double z = __dsub_rn(xreg[NB8 * 8 + e], yr[NB8 * 8 + e]); res = __dadd_rn(res, __dmul_rn(z, z)); }
  return res;
}

// the local cost from the sum of squares: cost_kind 0 = euclid, 1 = melcd
__device__ __forceinline__ double local_cost(double sumsq, int kind, double logdb) {
  const double r = sqrt(sumsq);
  return kind == 1 ? __dmul_rn(logdb, r) : r;
}

// ---- FastDTW (radius >= 1): one CTA (4 warps) per pair, the whole recursion inside the CTA ---------
// Per level:   (C) all 128 threads evaluate the local cost of every window cell, eight lanes per
//                  cell (numpy's pairwise order, see below), into a float64 cost buffer -- this is
//                  the bulk of the arithmetic and has no dependence on the recurrence;
//              (D) warp 0 walks the anti-diagonals with ONE LANE PER ACTIVE ROW (row i lives in lane
//                  i & 31): the three predecessors come from the lane's own registers and from the
//                  neighbouring lane by shuffle, the cell's cost from a small shared-memory ring that
//                  cp.async fills FD_PD diagonals ahead, so the serial part of a diagonal is a few
//                  dozen instructions;
//              (B) thread 0 backtracks and records the per-row extents the next finer level needs.
// A level whose rows are wider than the lane / ring budget (never for small radii) runs (D) with the
// straightforward loop over cells instead.
constexpr int FD_BLOCK = 128;
constexpr int FD_PD = 7;       // cost prefetch distance in diagonals (ring of FD_PD + 1 = 8 slots)
constexpr int FD_MAXW = 24;    // most rows active on one diagonal the lane-per-row path takes (+ FD_PD < 32)

__device__ __forceinline__ void cp_async8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}

// lanes 8m..8m+7 hold r_0..r_7: lane 8m ends with numpy's ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7))
__device__ __forceinline__ double fold8_lanes(double r) {
  r = __dadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 1));
  r = __dadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 2));
  return __dadd_rn(r, __shfl_xor_sync(0xffffffffu, r, 4));
}

#define FD_TICK(slot)                                                            \
  do {                                                                           \
    if (p.prof && tid == 0) {                                                    \
      const long long now_ = clock64();                                          \
      atomicAdd(p.prof + (slot), (unsigned long long)(now_ - tick_));            \
      tick_ = now_;                                                              \
    }                                                                            \
  } while (0)

__global__ void __launch_bounds__(FD_BLOCK) fastdtw_kernel(const DtwParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  long long tick_ = clock64();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int pair = p.order ? p.order[blockIdx.x] : blockIdx.x;
  const int Tx0 = p.len_x[pair], Ty0 = p.len_y[pair];
  const int D = p.D;
  if (Tx0 <= 0 || Ty0 <= 0) { store_empty_pair(p, pair); return; }
  // ---- shared memory carve-up -------------------------------------------------------------------
  const int mtx = p.max_tx;
  double* cring = reinterpret_cast<double*>(smem);            // [FD_PD + 1][32] prefetched costs
  int* lo = reinterpret_cast<int*>(cring + (FD_PD + 1) * 32);
  int* hi = lo + mtx;
  int* off = hi + mtx;             // [mtx + 1] row offsets into bp / cost buffer
  int* jmn = off + mtx + 1;        // [mtx/2 + 1] coarse path extents per coarse row
  int* jmx = jmn + mtx / 2 + 1;
  unsigned char* bp_s = reinterpret_cast<unsigned char*>(jmx + mtx / 2 + 1);
  __shared__ int s_n, s_wmax;
  __shared__ long long s_cells;

  unsigned char* wsp = p.ws + (size_t)pair * p.ws_pair_bytes;
  double* xs = reinterpret_cast<double*>(wsp);
  double* ys = xs + p.series_doubles;
  double* Dglob = ys + p.series_doubles;                                   // [3][mtx] DP diagonals of the slow path
  double* cbuf = Dglob + 3 * (size_t)mtx;                                  // [cost_cap] local costs of one level
  unsigned char* bp_g = reinterpret_cast<unsigned char*>(cbuf + p.cost_cap);

  // ---- level 0 = the inputs widened to float64 (fastdtw: np.asanyarray(x, dtype='float')) --------
  {
    const int64_t xb = (int64_t)pair * p.x_pair_stride, yb = (int64_t)pair * p.y_pair_stride;
#pragma unroll 4
    for (int r = warp; r < Tx0; r += FD_BLOCK / 32)
      for (int e = lane; e < D; e += 32) {
        const int64_t src = xb + (int64_t)r * p.x_ld + e;
        xs[(size_t)r * D + e] = p.is_f64 ? reinterpret_cast<const double*>(p.X)[src] : (double)reinterpret_cast<const float*>(p.X)[src];
      }
#pragma unroll 4
    for (int r = warp; r < Ty0; r += FD_BLOCK / 32)
      for (int e = lane; e < D; e += 32) {
        const int64_t src = yb + (int64_t)r * p.y_ld + e;
        ys[(size_t)r * D + e] = p.is_f64 ? reinterpret_cast<const double*>(p.Y)[src] : (double)reinterpret_cast<const float*>(p.Y)[src];
      }
  }
  // ---- coarser levels: __reduce_by_half, until one side is shorter than radius + 2 ----------------
  int nlev = 1;
  {
    const int min_time = p.radius + 2;
    int tx = Tx0, ty = Ty0;
    size_t xo = 0, yo = 0;
    __syncthreads();
    while (tx >= min_time && ty >= min_time) {
      const int hx = tx / 2, hy = ty / 2;
      const double* xin = xs + xo; const double* yin = ys + yo;
      double* xout = xs + xo + (size_t)tx * D; double* yout = ys + yo + (size_t)ty * D;
#pragma unroll 4
      for (int r = warp; r < hx; r += FD_BLOCK / 32)
        for (int e = lane; e < D; e += 32)
          xout[(size_t)r * D + e] = (xin[(size_t)(2 * r) * D + e] + xin[(size_t)(2 * r + 1) * D + e]) / 2;
#pragma unroll 4
      for (int r = warp; r < hy; r += FD_BLOCK / 32)
        for (int e = lane; e < D; e += 32)
          yout[(size_t)r * D + e] = (yin[(size_t)(2 * r) * D + e] + yin[(size_t)(2 * r + 1) * D + e]) / 2;
      xo += (size_t)tx * D; yo += (size_t)ty * D;
      tx = hx; ty = hy;
      ++nlev;
      __syncthreads();
    }
  }
  if (tid == 0) s_cells = 0;
  __syncthreads();
  FD_TICK(0);

  // ---- levels, coarsest first ---------------------------------------------------------------------
  for (int lev = nlev - 1; lev >= 0; --lev) {
    int Tx = Tx0, Ty = Ty0;
    size_t xo = 0, yo = 0;
    for (int l = 0; l < lev; ++l) { xo += (size_t)Tx * D; yo += (size_t)Ty * D; Tx /= 2; Ty /= 2; }
    const double* xl = xs + xo;
    const double* yl = ys + yo;
    // window: full rectangle at the coarsest level, else __expand_window of the coarser path
    if (lev == nlev - 1) {
      for (int i = tid; i < Tx; i += FD_BLOCK) { lo[i] = 0; hi[i] = Ty; }
    } else {
      const int cx = Tx / 2, r = p.radius;  // coarse rows 0..cx-1 all carry path cells
      for (int i = tid; i < Tx; i += FD_BLOCK) {
        const int a = i >> 1;
        int mn = INT_MAX, mx = -1;
        for (int aa = max(0, a - r); aa <= min(cx - 1, a + r); ++aa) { mn = min(mn, jmn[aa]); mx = max(mx, jmx[aa]); }
        int l = 2 * (mn - r), h = 2 * (mx + r) + 2;
        if (mx < 0) { l = 0; h = 0; }
        lo[i] = max(0, l);
        hi[i] = min(Ty, h);
      }
    }
    __syncthreads();
    if (warp == 0) {  // exclusive prefix sum of the row widths (warp scan, 32 rows per step)
      int carry = 0;
      for (int base = 0; base < Tx; base += 32) {
        const int i = base + lane;
        const int wdt = (i < Tx) ? max(0, hi[i] - lo[i]) : 0;
        int incl = wdt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        if (i < Tx) off[i] = carry + incl - wdt;
        carry += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (lane == 0) { off[Tx] = carry; s_cells += carry; s_wmax = 0; }
    }
    for (int a = tid; a < Tx; a += FD_BLOCK) { if (a < mtx / 2 + 1) { jmn[a] = INT_MAX; jmx[a] = -1; } }
    __syncthreads();
    // exact maximum number of rows active on one diagonal: the span grows only when a row enters
    // (diagonal k = i + lo[i]); the lowest row still active then is the first r with r + hi[r] > k
    // (r + hi[r] is increasing), found by binary search -- all rows in parallel.
    {
      int smax = 0;
      for (int i = tid; i < Tx; i += FD_BLOCK) {
        const int k = i + lo[i];
        int a = 0, b = i;  // first r in [0, i] with r + hi[r] > k
        while (a < b) {
          const int m = (a + b) >> 1;
          if (m + hi[m] > k) b = m; else a = m + 1;
        }
        smax = max(smax, i - a + 1);
      }
      smax = __reduce_max_sync(0xffffffffu, smax);
      if (lane == 0) atomicMax(&s_wmax, smax);
    }
    __syncthreads();
    const int ncells = off[Tx];
    const bool bp_in_smem = ncells <= p.smem_bp_cap;
    const bool fast_d = (s_wmax <= FD_MAXW) && ((size_t)ncells <= p.cost_cap);
    unsigned char* bp = bp_in_smem ? bp_s : bp_g;
    FD_TICK(1);

    // ---- (C) local costs of every window cell, eight lanes per cell -------------------------------
    // lane l of a group accumulates the strided partial sum r_l of numpy's pairwise reduction (elements
    // l, l+8, l+16, ...); a three-step butterfly combines r_0..r_7 in exactly numpy's association
    // ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)); lane 0 adds the tail and takes the square root.
    if (fast_d) {
      const int grp = tid >> 3, gl = tid & 7;  // 16 groups of 8 lanes
      const int n8 = D - (D % 8), ntail = D - n8;
      const bool batched = (D >= 8 && D <= 32);  // <= 4 strided elements per lane: one batch of loads per cell
      int ci = 0;                                 // row cursor of this group
      for (int c0 = 0; c0 < ncells; c0 += 2 * (FD_BLOCK / 8)) {
        // two cells per group per trip so that their loads overlap
        int ii[2], jj[2], cidx[2];
        bool val[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int c = c0 + u * (FD_BLOCK / 8) + grp;
          val[u] = c < ncells;
          const int cc = val[u] ? c : ncells - 1;
          while (off[ci + 1] <= cc) ++ci;
          ii[u] = ci; jj[u] = lo[ci] + (cc - off[ci]); cidx[u] = c;
        }
        if (batched) {
          double xv[2][4], yv[2][4], xt[2], yt[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const double* xr = xl + (size_t)ii[u] * D;
            const double* yr = yl + (size_t)jj[u] * D;
#pragma unroll
            for (int m = 0; m < 4; ++m) {
              const int e = gl + 8 * m;
              xv[u][m] = (e < n8) ? xr[e] : 0.0;
              yv[u][m] = (e < n8) ? yr[e] : 0.0;
            }
            xt[u] = (gl < ntail) ? xr[n8 + gl] : 0.0;  // tail element n8 + gl, fetched by lane gl
            yt[u] = (gl < ntail) ? yr[n8 + gl] : 0.0;
          }
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            double z = __dsub_rn(xv[u][0], yv[u][0]);
            double r = __dmul_rn(z, z);
#pragma unroll
            for (int m = 1; m < 4; ++m)
              if (gl + 8 * m < n8) { z = __dsub_rn(xv[u][m], yv[u][m]); r = __dadd_rn(r, __dmul_rn(z, z)); }
            r = fold8_lanes(r);
            z = __dsub_rn(xt[u], yt[u]);
            const double at = __dmul_rn(z, z);
            for (int e = 0; e < ntail; ++e) r = __dadd_rn(r, __shfl_sync(0xffffffffu, at, e, 8));  // tail, in order
            if (val[u] && gl == 0) cbuf[cidx[u]] = local_cost(r, p.cost_kind, p.logdb);
          }
        } else {
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const double* xr = xl + (size_t)ii[u] * D;
            const double* yr = yl + (size_t)jj[u] * D;
            double r;
            if (D >= 8 && D <= 128) {
              r = fold8_lanes(strided8(xr, yr, gl, n8));
              for (int e = n8; e < D; ++e) r = __dadd_rn(r, sq(xr, yr, e));
            } else {
              r = pairwise_sumsq(xr, yr, D);
            }
            const double dt = local_cost(r, p.cost_kind, p.logdb);
            if (val[u] && gl == 0) cbuf[cidx[u]] = dt;
          }
        }
      }
      __threadfence_block();
    }
    __syncthreads();

    FD_TICK(2);
    const int ndiag = Tx + Ty - 1;
    if (warp == 0 && fast_d) {
      // ---- (D) wavefront, one lane per active row -------------------------------------------------
      // Every lane follows ONE row at a time: the row congruent to its lane index inside the 32-row band
      // [imin, imin + 32) (the band of rows that are, or are about to become, active).  The row's window
      // (lo, hi, offset) and its predecessor's window are cached in registers and reloaded only when the band
      // has moved past the row (every ~64 diagonals), so the per-diagonal step touches shared memory only
      // for the prefetched cost, the back-pointer and the two band-edge tests -- which are cached as well
      // (n_in = diagonal at which row imax + 1 enters, n_out = diagonal at which row imin leaves).
      int imin = 0, imax = -1;
      int n_in = (Tx > 0) ? lo[0] : INT_MAX;          // row 0 enters at diagonal 0 + lo[0]
      int n_out = (Tx > 0) ? hi[0] : INT_MAX;         // row imin leaves at diagonal imin + hi[imin]
      int my_row = -1;
      int r_lo = 0, r_hi = 0, r_off = 0, p_lo = 0, p_hi = 0;  // my row's window / offset, previous row's window
      double D1 = CUDART_INF, D2 = CUDART_INF;                  // my row on diagonals k-1, k-2
      bool fresh = false;
      auto follow = [&](int base) {  // (re)load the cached row of this lane for the band starting at `base`
        const int r = base + ((lane - base) & 31);
        if (r != my_row) {
          my_row = r;
          if (r < Tx) {
            r_lo = lo[r]; r_hi = hi[r]; r_off = off[r];
            p_lo = r > 0 ? lo[r - 1] : 0; p_hi = r > 0 ? hi[r - 1] : 0;
          } else {
            r_lo = 0; r_hi = 0; r_off = 0; p_lo = 0; p_hi = 0;  // beyond the last row: empty window
          }
          fresh = true;  // D1 / D2 still hold the OLD row's last two diagonals: the neighbouring lane reads them
        }                //   for two more steps, so they are only reset when the new row becomes active
      };
      auto prefetch = [&](int kk) {  // cost of this lane's cached row on diagonal kk -> ring slot of that diagonal
        const int jj = kk - my_row;
        if (kk < ndiag && jj >= r_lo && jj < r_hi)
          cp_async8(cring + (size_t)(kk % (FD_PD + 1)) * 32 + lane, cbuf + r_off + (jj - r_lo));
        asm volatile("cp.async.commit_group;" ::: "memory");
      };
      follow(0);
      for (int kk = 0; kk < FD_PD; ++kk) prefetch(kk);
      double dist_last = 0.0;
      for (int k = 0; k < ndiag; ++k) {
        while (n_in <= k) { ++imax; n_in = (imax + 1 < Tx) ? imax + 1 + lo[imax + 1] : INT_MAX; }
        while (n_out <= k) { ++imin; n_out = (imin < Tx) ? imin + hi[imin] : INT_MAX; }
        // a row that has left the band has no cell on any later diagonal: its lane moves on to row + 32.
        // (Its prefetches for diagonals k .. k + FD_PD - 1 found an empty window and copied nothing.)
        follow(imin);
        prefetch(k + FD_PD);
        asm volatile("cp.async.wait_group %0;" ::"n"(FD_PD) : "memory");
        __syncwarp();
        const int i = my_row;
        const bool active = i <= imax && i < Tx;
        if (active && fresh) { D1 = CUDART_INF; D2 = CUDART_INF; fresh = false; }  // the row enters
        const double upv = __shfl_sync(0xffffffffu, D1, (lane + 31) & 31);
        const double dgv = __shfl_sync(0xffffffffu, D2, (lane + 31) & 31);
        double newD = CUDART_INF;
        if (active) {
          const int j = k - i;
          const double dt = cring[(size_t)(k % (FD_PD + 1)) * 32 + lane];
          const bool vu = i > 0 && j >= p_lo && j < p_hi;
          const bool vl = j - 1 >= r_lo;
          const bool vd = i > 0 && j - 1 >= p_lo && j - 1 < p_hi;
          const Relaxed c = relax((vu ? upv : CUDART_INF) + dt, (vl ? D1 : CUDART_INF) + dt,
                                  ((i == 0 && j == 0) ? 0.0 : (vd ? dgv : CUDART_INF)) + dt);
          newD = c.best;
          bp[(size_t)(r_off + j - r_lo)] = (unsigned char)c.dir;
          if (i == Tx - 1 && j == Ty - 1) dist_last = c.best;
        }
        D2 = D1;
        D1 = newD;
      }
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      // the last cell (Tx-1, Ty-1) lives in lane (Tx-1) & 31
      dist_last = __shfl_sync(0xffffffffu, dist_last, (Tx - 1) & 31);
      if (lane == 0 && lev == 0) p.dist[pair] = dist_last;
      __threadfence_block();
    } else if (warp == 0 && !fast_d) {
      // ---- slow path: loop over the cells of each diagonal, frames and DP diagonals in global memory ----
      int imin = 0, imax = -1;
      for (int k = 0; k < ndiag; ++k) {
        while (imax + 1 < Tx && imax + 1 + lo[imax + 1] <= k) ++imax;
        while (imin < Tx && imin + hi[imin] <= k) ++imin;
        double* dk = Dglob + (size_t)(k % 3) * mtx;
        const double* d1 = Dglob + (size_t)((k + 2) % 3) * mtx;
        const double* d2 = Dglob + (size_t)((k + 1) % 3) * mtx;
        for (int i = imin + lane; i <= imax; i += 32) {
          const int j = k - i;
          const double dt = local_cost(pairwise_sumsq(xl + (size_t)i * D, yl + (size_t)j * D, D), p.cost_kind, p.logdb);
          const bool vu = i > 0 && j >= lo[i - 1] && j < hi[i - 1];
          const bool vl = j - 1 >= lo[i];
          const bool vd = i > 0 && j - 1 >= lo[i - 1] && j - 1 < hi[i - 1];
          const Relaxed c = relax((vu ? d1[i - 1] : CUDART_INF) + dt, (vl ? d1[i] : CUDART_INF) + dt,
                                  ((i == 0 && j == 0) ? 0.0 : (vd ? d2[i - 1] : CUDART_INF)) + dt);
          dk[i] = c.best;
          bp[(size_t)(off[i] + j - lo[i])] = (unsigned char)c.dir;
        }
        __threadfence_block();
        __syncwarp();
      }
      if (lane == 0 && lev == 0) p.dist[pair] = Dglob[(size_t)((ndiag - 1) % 3) * mtx + (Tx - 1)];
    }
    __syncthreads();
    FD_TICK(3);

    // ---- (B) backtrack (one thread; the path is a dependent chain) ----------------------------------
    if (tid == 0) {
      int i = Tx - 1, j = Ty - 1, n = 0;
      bool ok = true;
      int32_t* pi = p.path_i + (size_t)pair * p.path_ld;
      int32_t* pj = p.path_j + (size_t)pair * p.path_ld;
      // the window of the current row and of the row above live in registers (the row above is fetched when
      // the path moves up, one row before it is needed), the per-row column extent of the path is
      // accumulated in registers and stored once per row: one dependent shared-memory load per step
      int clo = lo[i], chi = hi[i], coff = off[i];
      int plo = i > 0 ? lo[i - 1] : 0, phi = i > 0 ? hi[i - 1] : 0, poff = i > 0 ? off[i - 1] : 0;
      int cmin = j, cmax = j;
      while (i >= 0 && j >= 0) {
        if (j < clo || j >= chi) { ok = false; break; }
        if (lev == 0) {
          if (n >= p.path_ld) { ok = false; break; }
          pi[n] = i; pj[n] = j;
        } else {
          cmin = min(cmin, j);
          cmax = max(cmax, j);
        }
        ++n;
        const unsigned char dir = bp[(size_t)(coff + j - clo)];
        if (dir != 0) --j;
        if (dir != 1) {  // the path leaves row i
          if (lev != 0) { jmn[i] = min(jmn[i], cmin); jmx[i] = max(jmx[i], cmax); cmin = j; cmax = j; }
          --i;
          clo = plo; chi = phi; coff = poff;
          if (i > 0) { plo = lo[i - 1]; phi = hi[i - 1]; poff = off[i - 1]; }
        }
      }
      if (lev != 0 && ok && i >= 0) { jmn[i] = min(jmn[i], cmin); jmx[i] = max(jmx[i], cmax); }  // path ended by j < 0
      s_n = ok ? n : -1;
    }
    __syncthreads();
    FD_TICK(4);
  }
  store_path<FD_BLOCK>(p, pair, s_n, s_cells);
}

// ---- exact DTW (radius < 0): cost pass + wavefront pass --------------------------------------------
// The local cost of a cell does not depend on the recurrence, so the exact mode is split in two:
//   dtw_cost_kernel : one thread per cell, all cells of all pairs in parallel, float64 cost written
//                     in DIAGONAL-MAJOR order (cell (i, k-i) of diagonal k at diag_off(k) + i - imin(k));
//   dtw_dp_kernel   : one CTA per pair walks the anti-diagonals; a diagonal's costs and back-pointers
//                     are contiguous, so every access of the wavefront is coalesced; three rolling
//                     diagonals of D live in shared memory; thread 0 backtracks at the end.
// number of cells on diagonals 0 .. k-1 of a Tx x Ty rectangle
__device__ __forceinline__ long long diag_off(int k, int Tx, int Ty) {
  const long long a = min(Tx, Ty), b = max(Tx, Ty);
  if (k <= a) return (long long)k * (k + 1) / 2;
  if (k <= b) return a * (a + 1) / 2 + (k - a) * a;
  const long long m = k - b;
  return a * (a + 1) / 2 + (b - a) * a + m * a - m * (m + 1) / 2;
}

// Tiled cost pass.  A block owns a TI x TJ tile of cells: the TI frames of x and TJ frames of y are
// staged ONCE in shared memory as float64 (coalesced loads, one conversion per element instead of
// one per cell); thread t owns row i0 + t and sweeps the tile along anti-diagonals (lane l of a warp
// is at column j0 + c - l in step c), so the 32 costs a warp produces per step belong to one
// diagonal and land contiguously in the diagonal-major cost buffer.  Per cell: numpy's pairwise sum
// with its eight static accumulators, float64, no FMA contraction.
constexpr int DTW_TI = 128, DTW_TJ = 64;

// NB8 = number of 8-element blocks of the pairwise reduction known at compile time (D in
// [8*NB8, 8*NB8 + 7]); NB8 == 0 selects pairwise_sumsq's run-time loops (D < 8 or D > 39).
template <typename T, int NB8>
__global__ void __launch_bounds__(DTW_TI) dtw_cost_kernel(const DtwParams p) {
  extern __shared__ __align__(16) unsigned char smem_c[];
  const int slot = blockIdx.y;
  const int pair = p.order ? p.order[p.first + slot] : p.first + slot;
  const int Tx = p.len_x[pair], Ty = p.len_y[pair];
  if (Tx <= 0 || Ty <= 0) return;
  const int tiles_j = (p.max_ty + DTW_TJ - 1) / DTW_TJ;
  const int i0 = (blockIdx.x / tiles_j) * DTW_TI, j0 = (blockIdx.x % tiles_j) * DTW_TJ;
  if (i0 >= Tx || j0 >= Ty) return;
  const int D = p.D, DP = dtw_row_stride(D);
  double* xs = reinterpret_cast<double*>(smem_c);  // [TI][DP]
  double* ys = xs + (size_t)DTW_TI * DP;           // [TJ][DP]
  const int tid = threadIdx.x;
  const T* X = reinterpret_cast<const T*>(p.X) + (int64_t)pair * p.x_pair_stride;
  const T* Y = reinterpret_cast<const T*>(p.Y) + (int64_t)pair * p.y_pair_stride;
  const int ni = min(DTW_TI, Tx - i0), nj = min(DTW_TJ, Ty - j0);
  for (int e = tid; e < ni * D; e += DTW_TI) {
    const int r = e / D, k = e - r * D;
    xs[(size_t)r * DP + k] = (double)X[(int64_t)(i0 + r) * p.x_ld + k];
  }
  for (int e = tid; e < nj * D; e += DTW_TI) {
    const int r = e / D, k = e - r * D;
    ys[(size_t)r * DP + k] = (double)Y[(int64_t)(j0 + r) * p.y_ld + k];
  }
  __syncthreads();
  const int lane = tid & 31, wbase = tid & ~31;
  const int i = i0 + tid;
  const double* xr = xs + (size_t)tid * DP;
  double* cost = p.cost + (size_t)slot * ((size_t)p.max_tx * p.max_ty);
  // this thread's frame of x stays in registers for the whole tile when the block count is static
  double xreg[NB8 > 0 ? NB8 * 8 + 8 : 1];
  if (NB8 > 0) {
#pragma unroll
    for (int e = 0; e < NB8 * 8 + 8; ++e) xreg[e] = (e < D) ? xr[e] : 0.0;
  }
  const int ntail = D - NB8 * 8;
  const int nsteps = DTW_TJ + 31;
  const bool row_ok = i < Tx;
  for (int c = 0; c < nsteps; ++c) {
    const int jl = c - lane;  // column inside the tile
    const int k = i0 + wbase + j0 + c;  // diagonal of every lane of this warp in this step
    if (row_ok && jl >= 0 && jl < nj) {
      const double* yr = ys + (size_t)jl * DP;
      double res;
      if constexpr (NB8 > 0) res = sumsq_reg<NB8>(xreg, yr, ntail);
      else res = pairwise_sumsq(xr, yr, D);
      cost[(size_t)diag_off(k, Tx, Ty) + (i - max(0, k - (Ty - 1)))] = local_cost(res, p.cost_kind, p.logdb);
    }
  }
}

template <int MC>
__global__ void __launch_bounds__(256) dtw_dp_kernel(const DtwParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* Dbuf = reinterpret_cast<double*>(smem);  // [3][max_tx]
  __shared__ int s_n;
  const int tid = threadIdx.x;
  const int slot = blockIdx.x;
  const int pair = p.order ? p.order[p.first + slot] : p.first + slot;
  const int Tx = p.len_x[pair], Ty = p.len_y[pair];
  if (Tx <= 0 || Ty <= 0) { store_empty_pair(p, pair); return; }
  const int mtx = p.max_tx;
  const double* cost = p.cost + (size_t)slot * ((size_t)p.max_tx * p.max_ty);
  unsigned char* bp = p.bp + (size_t)slot * ((size_t)p.max_tx * p.max_ty);
  const int ndiag = Tx + Ty - 1;
  long long off = 0;
  // the costs of diagonal k+1 are fetched while diagonal k is being relaxed (MC cells per thread)
  double cnext[MC];
  {
    const int imax0 = 0;
#pragma unroll
    for (int m = 0; m < MC; ++m) cnext[m] = (tid + 256 * m <= imax0) ? cost[tid + 256 * m] : 0.0;
  }
  for (int k = 0; k < ndiag; ++k) {
    const int imin = max(0, k - (Ty - 1)), imax = min(Tx - 1, k);
    const int ncur = imax - imin + 1;
    double ccur[MC];
#pragma unroll
    for (int m = 0; m < MC; ++m) ccur[m] = cnext[m];
    if (k + 1 < ndiag) {
      const int nmin = max(0, k + 1 - (Ty - 1)), nmax = min(Tx - 1, k + 1);
      const double* cn = cost + off + ncur;
#pragma unroll
      for (int m = 0; m < MC; ++m) cnext[m] = (tid + 256 * m <= nmax - nmin) ? cn[tid + 256 * m] : 0.0;
    }
    double* dk = Dbuf + (size_t)(k % 3) * mtx;
    const double* d1 = Dbuf + (size_t)((k + 2) % 3) * mtx;
    const double* d2 = Dbuf + (size_t)((k + 1) % 3) * mtx;
#pragma unroll
    for (int m = 0; m < MC; ++m) {
      const int i = imin + tid + 256 * m;
      if (i <= imax) {
        const int j = k - i;
        const double dt = ccur[m];
        const Relaxed c = relax((i > 0 ? d1[i - 1] : CUDART_INF) + dt, (j > 0 ? d1[i] : CUDART_INF) + dt,
                                ((i == 0 && j == 0) ? 0.0 : ((i > 0 && j > 0) ? d2[i - 1] : CUDART_INF)) + dt);
        dk[i] = c.best;
        bp[off + (i - imin)] = (unsigned char)c.dir;
      }
    }
    off += ncur;
    __syncthreads();
  }
  if (tid == 0) {
    __threadfence_block();
    int i = Tx - 1, j = Ty - 1, n = 0;
    bool ok = true;
    p.dist[pair] = Dbuf[(size_t)((ndiag - 1) % 3) * mtx + (Tx - 1)];
    int32_t* pi = p.path_i + (size_t)pair * p.path_ld;
    int32_t* pj = p.path_j + (size_t)pair * p.path_ld;
    while (i >= 0 && j >= 0) {
      if (n >= p.path_ld) { ok = false; break; }
      pi[n] = i; pj[n] = j;
      ++n;
      const int k = i + j;
      const unsigned char dir = bp[diag_off(k, Tx, Ty) + (i - max(0, k - (Ty - 1)))];
      if (dir == 0) --i;
      else if (dir == 1) --j;
      else { --i; --j; }
    }
    s_n = ok ? n : -1;
  }
  __syncthreads();
  store_path<256>(p, pair, s_n, (long long)Tx * Ty);
}

// ---- exact DTW, fused (the production path for frames of 8..39 dims that fit shared memory) -----------------
// One CTA (16 warps) per pair; the local cost of a cell is computed in registers at the moment the
// recurrence needs it -- there is NO Tx x Ty cost matrix in HBM (the two-kernel path above wrote and
// re-read 8 bytes per cell: 5 GB per configs[3] batch against 0.25 GB of algorithmic traffic).
//   * all of Y (float64, conflict-free row stride) is staged ONCE in shared memory;
//   * the rows of X are cut into groups of 32; warp w owns groups w, w + 16, ...  Lane l of the warp owns
//     row i = 32 g + l, keeps its frame of X in registers (float64) and walks the columns: at step s it
//     relaxes cell (i, j = s - l) -- the warp is one 32-cell anti-diagonal wavefront that streams over all
//     Ty columns with every lane busy.  Predecessors: left = the lane's own register, up / diagonal = the
//     neighbouring lane's register by shuffle; lane 0 takes them from the last row of the previous group;
//   * groups are a software pipeline, not lock-stepped: lane 31 publishes its row into a small ring in
//     shared memory (DTW_CW columns per boundary) together with a progress counter, the warp that owns
//     the next group polls it every DTW_POLL steps (and publishes how far it has read, so the producer
//     never overwrites unread columns).  No __syncthreads inside the recurrence: a first version that
//     advanced one diagonal of 512 rows per barrier left half of the warps idle (the triangle ramps) and
//     stalled at the barrier;
//   * cost: numpy's pairwise order, float64, no FMA contraction (bit-exact), two columns per loop trip so
//     that the sqrt chain of one cell overlaps the element-wise work of the next;
//   * back-pointers are 2 bits per cell, packed by the owning lane into one 32-bit word per 16 columns,
//     row-major in an L2-resident scratch (200 KB per pair instead of 1 byte per cell);
//   * the back-track is a pointer chase: warp 0 loads a 32-row x 32-column window of back-pointer words
//     with one coalesced round trip, walks it by shuffles, and reloads when the path leaves the window.
constexpr int DTW_FR = 512;
constexpr int DTW_NWARP = DTW_FR / 32;
constexpr int DTW_CW = 128;    // columns per boundary ring
constexpr int DTW_NBR = DTW_NWARP + 1;  // boundary rings (one per group in flight + the one being read)
constexpr int DTW_POLL = 8;    // steps between progress checks / publications
constexpr int DTW_TRIP = 2;    // columns per loop trip (cost evaluations in flight per lane)
static_assert(DTW_POLL % DTW_TRIP == 0, "progress checks fall on trip boundaries");

template <typename T, int NB8>
__global__ void __launch_bounds__(DTW_FR, 1) dtw_fused_kernel(const DtwParams p) {
  extern __shared__ __align__(16) unsigned char smem_f[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int slot = blockIdx.x;
  const int pair = p.order ? p.order[slot] : slot;
  const int Tx = p.len_x[pair], Ty = p.len_y[pair];
  if (Tx <= 0 || Ty <= 0) { store_empty_pair(p, pair); return; }
  const int D = p.D, DP = dtw_row_stride(D);
  const int max_groups = (p.max_tx + 31) / 32;
  double* Ys = reinterpret_cast<double*>(smem_f);              // [max_ty][DP]
  double* Bnd = Ys + (size_t)p.max_ty * DP;                    // [DTW_NBR][DTW_CW] last rows of the groups in flight
  volatile int* prog = reinterpret_cast<volatile int*>(Bnd + DTW_NBR * DTW_CW);  // [groups] columns published by group g
  volatile int* cons = prog + max_groups + 1;                                   // [groups] columns group g has read
  const T* X = reinterpret_cast<const T*>(p.X) + (int64_t)pair * p.x_pair_stride;
  const T* Y = reinterpret_cast<const T*>(p.Y) + (int64_t)pair * p.y_pair_stride;
  for (int e = tid; e < Ty * D; e += DTW_FR) {
    const int r = e / D, k = e - r * D;
    Ys[(size_t)r * DP + k] = (double)Y[(int64_t)r * p.y_ld + k];
  }
  for (int e = tid; e < 2 * (max_groups + 1); e += DTW_FR) prog[e] = 0;
  __syncthreads();
  uint32_t* bp = p.bp_words + (size_t)slot * ((size_t)p.max_tx * p.wpr);
  const int ntail = D - NB8 * 8;
  const int ngroups = (Tx + 31) / 32;
  const int nsteps = Ty + 31;
  for (int g = warp; g < ngroups; g += DTW_NWARP) {
    const int i = g * 32 + lane;
    const bool row_ok = i < Tx;
    double xreg[NB8 * 8 + 8];
#pragma unroll
    for (int e = 0; e < NB8 * 8 + 8; ++e) xreg[e] = (row_ok && e < D) ? (double)X[(int64_t)i * p.x_ld + e] : 0.0;
    const double* bprev = Bnd + (size_t)((g + DTW_NBR - 1) % DTW_NBR) * DTW_CW;  // written by group g - 1
    double* bcur = Bnd + (size_t)(g % DTW_NBR) * DTW_CW;                          // read by group g + 1
    const bool feeds = (g + 1 < ngroups);
    double myD = CUDART_INF;     // D[i][j-1] of the lane's current column (left)
    double uprev = CUDART_INF;   // D[i-1][j-1] (diagonal) = what the neighbour held one step earlier
    uint32_t bpw = 0;
    uint32_t* bprow = bp + (size_t)i * p.wpr;
    for (int s0 = 0; s0 < nsteps; s0 += DTW_TRIP) {
      if ((s0 & (DTW_POLL - 1)) == 0) {
        // (1) publish: lane 0 has consumed boundary columns < s0; lane 31 has produced columns <= s0 - 32
        __syncwarp();
        if (lane == 0 && g > 0) cons[g] = s0;
        if (lane == 31 && feeds) { __threadfence_block(); prog[g] = max(0, s0 - 31); }
        // (2) wait: the previous group must have published the columns lane 0 reads in the next DTW_POLL
        //     steps; the next group must have read the ring slots lane 31 is about to overwrite
        if (g > 0) {
          const int need = min(Ty, s0 + DTW_POLL);
          while (prog[g - 1] < need) __nanosleep(40);
        }
        if (feeds) {
          const int j_hi = s0 + DTW_POLL - 1 - 31;  // last column lane 31 writes before the next check
          while (j_hi - DTW_CW + 2 > cons[g + 1]) __nanosleep(40);
        }
        __threadfence_block();
        __syncwarp();
      }
      // ---- local costs of this lane's cells of steps s0, s0 + 1 (branch-free, columns clamped) ----
      double cst[DTW_TRIP];
#pragma unroll
      for (int q = 0; q < DTW_TRIP; ++q) {
        const int jc = min(max(s0 + q - lane, 0), Ty - 1);
        cst[q] = local_cost(sumsq_reg<NB8>(xreg, Ys + (size_t)jc * DP, ntail), p.cost_kind, p.logdb);
      }
      // ---- two relaxation steps ----
#pragma unroll
      for (int q = 0; q < DTW_TRIP; ++q) {
        const int s = s0 + q;
        const int j = s - lane;
        // up = D[i-1][j]: the neighbouring lane finished that cell in the previous step
        double u = __shfl_up_sync(0xffffffffu, myD, 1);
        if (lane == 0) {
          if (g > 0) {
            u = (s < Ty) ? bprev[s & (DTW_CW - 1)] : CUDART_INF;
            uprev = (s > 0 && s <= Ty) ? bprev[(s - 1) & (DTW_CW - 1)] : CUDART_INF;
          } else {
            u = CUDART_INF;
            uprev = (s == 0) ? 0.0 : CUDART_INF;  // the virtual cell before (0, 0)
          }
        }
        if (row_ok && j >= 0 && j < Ty) {
          const double dt = cst[q];
          const Relaxed c = relax(u + dt, myD + dt, uprev + dt);  // myD == +inf before the lane's first column
          myD = c.best;
          if (lane == 31 && feeds) bcur[j & (DTW_CW - 1)] = c.best;
          bpw |= c.dir << (2 * (j & 15));
          if ((j & 15) == 15 || j == Ty - 1) { bprow[j >> 4] = bpw; bpw = 0; }
          if (i == Tx - 1 && j == Ty - 1) p.dist[pair] = c.best;
        }
        uprev = u;
      }
    }
    if (lane == 31 && feeds) { __threadfence_block(); prog[g] = Ty; }
    if (lane == 0 && g > 0) cons[g] = nsteps + DTW_CW;
    __syncwarp();
  }
  __syncthreads();
  // ---- back-track (warp 0) ----
  __shared__ int s_n;
  if (warp == 0) {
    int i = Tx - 1, j = Ty - 1, n = 0;
    bool ok = true;
    int32_t* pi = p.path_i + (size_t)pair * p.path_ld;
    int32_t* pj = p.path_j + (size_t)pair * p.path_ld;
    while (ok && i >= 0 && j >= 0) {
      const int bi = i, bw = j >> 4;
      const int r = bi - lane;
      const uint32_t w0 = (r >= 0) ? __ldcg(bp + (size_t)r * p.wpr + bw) : 0u;
      const uint32_t w1 = (r >= 0 && bw > 0) ? __ldcg(bp + (size_t)r * p.wpr + bw - 1) : 0u;
      while (i >= 0 && j >= 0 && bi - i < 32 && (j >> 4) >= bw - 1) {
        if (n >= p.path_ld) { ok = false; break; }
        if (lane == 0) { pi[n] = i; pj[n] = j; }
        ++n;
        const bool second = (j >> 4) != bw;
        const uint32_t word = __shfl_sync(0xffffffffu, second ? w1 : w0, bi - i);
        const uint32_t dir = (word >> (2 * (j & 15))) & 3u;
        if (dir == 0) --i;
        else if (dir == 1) --j;
        else { --i; --j; }
      }
    }
    if (lane == 0) s_n = ok ? n : -1;
  }
  __syncthreads();
  store_path<DTW_FR>(p, pair, s_n, (long long)Tx * Ty);
}

static size_t dtw_fused_smem(int max_tx, int max_ty, int D) {
  const size_t groups = (size_t)(max_tx + 31) / 32;
  return sizeof(double) * ((size_t)max_ty * dtw_row_stride(D) + (size_t)DTW_NBR * DTW_CW) + sizeof(int) * 2 * (groups + 1) + 16;
}
// the fused kernel serves frames of 8..39 dimensions whose Y series fits shared memory as float64;
// max_dyn is the dynamic shared memory a block may request: the opt-in limit less the kernel's static part
static bool dtw_fused_ok(int max_tx, int max_ty, int D, size_t max_dyn) {
  return D >= 8 && D < 40 && dtw_fused_smem(max_tx, max_ty, D) <= max_dyn;
}
// the instances for a dtype and a count of 8-element blocks of the frame (nb8 = D / 8 inside 8..39, else 0)
static const void* dtw_fused_instance(bool f64, int nb8) {
  switch (nb8) {
    case 1: return f64 ? (const void*)dtw_fused_kernel<double, 1> : (const void*)dtw_fused_kernel<float, 1>;
    case 2: return f64 ? (const void*)dtw_fused_kernel<double, 2> : (const void*)dtw_fused_kernel<float, 2>;
    case 3: return f64 ? (const void*)dtw_fused_kernel<double, 3> : (const void*)dtw_fused_kernel<float, 3>;
    default: return f64 ? (const void*)dtw_fused_kernel<double, 4> : (const void*)dtw_fused_kernel<float, 4>;
  }
}
static const void* dtw_cost_instance(bool f64, int nb8) {
  switch (nb8) {
    case 1: return f64 ? (const void*)dtw_cost_kernel<double, 1> : (const void*)dtw_cost_kernel<float, 1>;
    case 2: return f64 ? (const void*)dtw_cost_kernel<double, 2> : (const void*)dtw_cost_kernel<float, 2>;
    case 3: return f64 ? (const void*)dtw_cost_kernel<double, 3> : (const void*)dtw_cost_kernel<float, 3>;
    case 4: return f64 ? (const void*)dtw_cost_kernel<double, 4> : (const void*)dtw_cost_kernel<float, 4>;
    default: return f64 ? (const void*)dtw_cost_kernel<double, 0> : (const void*)dtw_cost_kernel<float, 0>;
  }
}
// opts `fn` in to `smem` bytes of dynamic shared memory, then launches it with the parameters `p`
static cudaError_t dtw_launch(const void* fn, dim3 grid, int block, size_t smem, cudaStream_t st, DtwParams p) {
  const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  void* args[] = {&p};
  return cudaLaunchKernel(fn, grid, dim3(block), args, smem, st);
}
// pairs per chunk of the exact mode: 9 bytes per cell (float64 cost + back-pointer), <= ~2 GiB per chunk
static int dtw_exact_chunk(int n_pairs, int max_tx, int max_ty) {
  const size_t per = (size_t)max_tx * (size_t)max_ty * 9;
  size_t ch = per ? ((size_t)2 << 30) / per : 1;
  if (ch < 1) ch = 1;
  return (int)(ch < (size_t)n_pairs ? ch : (size_t)n_pairs);
}

// X_aligned[n, :L] = X[n, path[n, :L]]; rows L.. are zero (alignment.py:52-54, 72-73)
template <typename T>
__global__ void gather_rows_kernel(const T* __restrict__ X, int64_t x_pair_stride, int x_ld, const int32_t* __restrict__ path,
                                   int path_ld, const int32_t* __restrict__ path_len, T* __restrict__ out,
                                   int64_t out_pair_stride, int out_rows, int D) {
  const int pair = blockIdx.y;
  const int L = path_len[pair];
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)out_rows * D; e += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(e / D), k = (int)(e % D);
    T v = T(0);
    if (r < L) v = X[(int64_t)pair * x_pair_stride + (int64_t)path[(int64_t)pair * path_ld + r] * x_ld + k];
    out[(int64_t)pair * out_pair_stride + (int64_t)r * D + k] = v;
  }
}

// trim_zeros_frames(x, eps, trim='b') lengths (preprocessing/generic.py:312-323): last frame whose
// sum_d |x| (accumulated in the input dtype, numpy pairwise order for D <= 128) is >= eps, plus one.
template <typename T>
__device__ T abs_pairwise(const T* a, int n) {
  if (n < 8) {
    T res = T(0);
    for (int i = 0; i < n; ++i) res += fabs(a[i]);
    return res;
  }
  if (n <= 128) {
    T r[8];
    for (int j = 0; j < 8; ++j) r[j] = fabs(a[j]);
    int i;
    for (i = 8; i < n - (n % 8); i += 8)
      for (int j = 0; j < 8; ++j) r[j] += fabs(a[i + j]);
    T res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (; i < n; ++i) res += fabs(a[i]);
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return abs_pairwise(a, n2) + abs_pairwise(a + n2, n - n2);
}

template <typename T>
__global__ void trim_len_kernel(const T* __restrict__ X, int64_t pair_stride, int ld, int Tn, int D, T eps, int32_t* __restrict__ len) {
  const int pair = blockIdx.x;
  __shared__ int s_last;
  if (threadIdx.x == 0) s_last = 0;
  __syncthreads();
  int last = 0;
  for (int t = threadIdx.x; t < Tn; t += blockDim.x) {
    const T s = abs_pairwise(X + (int64_t)pair * pair_stride + (int64_t)t * ld, D);
    if (!(s < eps)) last = max(last, t + 1);
  }
  atomicMax(&s_last, last);
  __syncthreads();
  if (threadIdx.x == 0) len[pair] = s_last;
}

static size_t dtw_series_doubles(int max_t, int D) { return (size_t)2 * (size_t)max_t * D + 8; }

static size_t dtw_smem_bytes(int max_tx, int bp_cap) {
  size_t b = sizeof(double) * (FD_PD + 1) * 32;
  b += sizeof(int) * ((size_t)max_tx * 2 + (max_tx + 1) + 2 * (max_tx / 2 + 1)) + (size_t)bp_cap;
  return b + 16;
}

static size_t dtw_fast_cells_bound(int max_tx, int max_ty, int radius) {
  // window cells of one level <= 4 (2r+1) (coarse path length + 2r+1); the coarsest level is a full
  // rectangle of at most (2(r+2)) x ... cells, covered by the same bound for every realistic size
  const size_t r2 = (size_t)(2 * radius + 1);
  return 4 * r2 * ((size_t)(max_tx + max_ty) / 2 + r2 + 2) + 64;
}

}  // namespace nnk

using namespace nnk;

extern "C" size_t nnk_dtw_workspace_bytes(int32_t n_pairs, int32_t max_tx, int32_t max_ty, int32_t D, int32_t radius) {
  const int mt = max_tx > max_ty ? max_tx : max_ty;
  if (radius < 0) {
    // exact, two-pass fallback: chunked float64 cost matrix + back-pointers, diagonal-major;
    // exact, fused: 2-bit back-pointers only, (max_ty / 16 + 1) words per row, every pair at once
    const size_t ch = (size_t)dtw_exact_chunk(n_pairs, max_tx, max_ty);
    const size_t two_pass = ((ch * (size_t)max_tx * (size_t)max_ty * 9 + 255) / 256 * 256) + 256;
    const size_t fused = (size_t)n_pairs * (size_t)max_tx * (size_t)((max_ty + 15) / 16) * 4 + 256;
    return two_pass > fused ? two_pass : fused;
  }
  size_t per = 2 * dtw_series_doubles(mt, D) * sizeof(double) + 3 * (size_t)max_tx * sizeof(double);
  per += dtw_fast_cells_bound(max_tx, max_ty, radius) * sizeof(double);  // cost buffer of one level
  per += (size_t)max_tx * (size_t)max_ty < ((size_t)64 << 20) ? (size_t)max_tx * (size_t)max_ty : ((size_t)64 << 20);
  per = (per + 255) / 256 * 256;
  return per * (size_t)n_pairs;
}

extern "C" int nnk_dtw_align(const nnk_dtw_args_t* a, void* stream) {
  NNK_REQUIRE(a != nullptr, NNK_ERR_ARG, "args is NULL");
  NNK_REQUIRE(a->n_pairs >= 0 && a->D > 0 && a->max_tx >= 0 && a->max_ty >= 0, NNK_ERR_ARG, "bad size");
  if (a->n_pairs == 0 || a->max_tx == 0 || a->max_ty == 0) return NNK_OK;
  NNK_REQUIRE(a->X && a->Y && a->len_x && a->len_y && a->path_i && a->path_j && a->path_len && a->dist && a->workspace,
              NNK_ERR_ARG, "NULL device pointer");
  NNK_REQUIRE(a->dtype == NNK_F32 || a->dtype == NNK_F64, NNK_ERR_ARG, "bad dtype");
  NNK_REQUIRE(a->cost_kind == 0 || a->cost_kind == 1, NNK_ERR_UNSUPPORTED, "cost_kind must be 0 (euclid) or 1 (melcd)");
  NNK_REQUIRE(a->path_ld >= a->max_tx + a->max_ty - 1, NNK_ERR_ARG, "path_ld < max_tx + max_ty - 1");
  NNK_REQUIRE(a->radius != 0, NNK_ERR_UNSUPPORTED, "radius 0 is not supported (fastdtw itself fails on odd lengths)");
  DeviceGuard guard(a->X);
  cudaStream_t st = (cudaStream_t)stream;
  const bool full = a->radius < 0;
  const int mt = a->max_tx > a->max_ty ? a->max_tx : a->max_ty;
  DtwParams p{};
  p.X = a->X; p.Y = a->Y; p.is_f64 = a->dtype == NNK_F64;
  p.x_pair_stride = a->x_pair_stride; p.y_pair_stride = a->y_pair_stride; p.x_ld = a->x_ld; p.y_ld = a->y_ld; p.D = a->D;
  p.len_x = a->len_x; p.len_y = a->len_y; p.order = a->order; p.cost_kind = a->cost_kind; p.radius = a->radius;
  p.path_i = a->path_i; p.path_j = a->path_j; p.path_ld = a->path_ld; p.path_len = a->path_len; p.dist = a->dist;
  p.cells = (long long*)a->cells; p.max_tx = a->max_tx; p.max_ty = a->max_ty;
  p.logdb = 10.0 / log(10.0) * sqrt(2.0);  // metrics/__init__.py:5
  const size_t need = nnk_dtw_workspace_bytes(a->n_pairs, a->max_tx, a->max_ty, a->D, a->radius);
  NNK_REQUIRE(a->workspace_bytes >= need, NNK_ERR_WORKSPACE, "DTW workspace too small");
  int dev = 0, max_smem = 0;
  NNK_CUDA_CHECK(cudaGetDevice(&dev));
  NNK_CUDA_CHECK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int nb8 = (a->D >= 8 && a->D < 40) ? a->D / 8 : 0;  // registers hold a frame of up to 39 dims
  size_t fused_dyn = 0;  // dynamic shared memory the fused instance for this D may request
  if (full && nb8 > 0) {
    cudaFuncAttributes fa;
    NNK_CUDA_CHECK(cudaFuncGetAttributes(&fa, dtw_fused_instance(p.is_f64, nb8)));
    fused_dyn = (size_t)max_smem > fa.sharedSizeBytes ? (size_t)max_smem - fa.sharedSizeBytes : 0;
  }
  if (full && dtw_fused_ok(a->max_tx, a->max_ty, a->D, fused_dyn)) {
    p.bp_words = reinterpret_cast<uint32_t*>(a->workspace);
    p.wpr = (a->max_ty + 15) / 16;
    NNK_CUDA_CHECK(dtw_launch(dtw_fused_instance(p.is_f64, nb8), a->n_pairs, DTW_FR, dtw_fused_smem(a->max_tx, a->max_ty, a->D), st, p));
    count_launch();
    NNK_CUDA_CHECK(cudaGetLastError());
    return NNK_OK;
  }
  if (full) {
    const size_t smem = sizeof(double) * 3 * (size_t)a->max_tx + 16;
    NNK_REQUIRE(smem <= (size_t)max_smem, NNK_ERR_UNSUPPORTED, "sequence too long for the wavefront buffers in shared memory");
    NNK_REQUIRE(a->max_tx <= 256 * 16, NNK_ERR_UNSUPPORTED, "exact DTW supports up to 4096 frames");
    const int mc = (a->max_tx + 255) / 256;
    const void* dp_fn = mc <= 4 ? (const void*)dtw_dp_kernel<4> : mc <= 8 ? (const void*)dtw_dp_kernel<8> : (const void*)dtw_dp_kernel<16>;
    const size_t csmem = (size_t)(DTW_TI + DTW_TJ) * dtw_row_stride(a->D) * sizeof(double);
    NNK_REQUIRE(csmem <= (size_t)max_smem, NNK_ERR_UNSUPPORTED, "feature dimension too large for the cost tiles");
    const int tiles_i = (a->max_tx + DTW_TI - 1) / DTW_TI, tiles_j = (a->max_ty + DTW_TJ - 1) / DTW_TJ;
    const int ch = dtw_exact_chunk(a->n_pairs, a->max_tx, a->max_ty);
    const size_t cells = (size_t)a->max_tx * (size_t)a->max_ty;
    p.cost = reinterpret_cast<double*>(a->workspace);
    p.bp = reinterpret_cast<unsigned char*>(a->workspace) + (size_t)ch * cells * sizeof(double);
    for (int first = 0; first < a->n_pairs; first += ch) {
      p.first = first;
      p.n_pairs = (a->n_pairs - first < ch) ? a->n_pairs - first : ch;
      const dim3 grid((unsigned)(tiles_i * tiles_j), (unsigned)p.n_pairs);
      NNK_CUDA_CHECK(dtw_launch(dtw_cost_instance(p.is_f64, nb8), grid, DTW_TI, csmem, st, p));
      NNK_CUDA_CHECK(dtw_launch(dp_fn, p.n_pairs, 256, smem, st, p));
      count_launch(2);
      NNK_CUDA_CHECK(cudaGetLastError());
    }
    return NNK_OK;
  } else {
    size_t bound = dtw_fast_cells_bound(a->max_tx, a->max_ty, a->radius);
    size_t smem = dtw_smem_bytes(a->max_tx, (int)bound);
    if (smem > (size_t)max_smem / 4) {  // keep >= 4 CTAs per SM; overflow back-pointers go to global scratch
      const size_t base = dtw_smem_bytes(a->max_tx, 0);
      NNK_REQUIRE(base + 1024 <= (size_t)max_smem, NNK_ERR_UNSUPPORTED, "sequence too long for shared memory");
      bound = ((size_t)max_smem / 4 > base + 1024) ? (size_t)max_smem / 4 - base : 1024;
      smem = dtw_smem_bytes(a->max_tx, (int)bound);
    }
    p.ws = (unsigned char*)a->workspace;
    p.ws_pair_bytes = need / (size_t)a->n_pairs;
    p.series_doubles = dtw_series_doubles(mt, a->D);
    p.smem_bp_cap = (int)bound;
    p.cost_cap = dtw_fast_cells_bound(a->max_tx, a->max_ty, a->radius);
    static unsigned long long* d_prof = nullptr;
    if (getenv("NNK_DTW_PROF")) {
      if (!d_prof) NNK_CUDA_CHECK(cudaMalloc(&d_prof, 8 * sizeof(unsigned long long)));
      NNK_CUDA_CHECK(cudaMemsetAsync(d_prof, 0, 8 * sizeof(unsigned long long), st));
      p.prof = d_prof;
    }
    NNK_CUDA_CHECK(dtw_launch((const void*)fastdtw_kernel, a->n_pairs, FD_BLOCK, smem, st, p));
    if (p.prof) {  // debug only: synchronises
      unsigned long long h[8];
      NNK_CUDA_CHECK(cudaMemcpyAsync(h, d_prof, sizeof(h), cudaMemcpyDeviceToHost, st));
      NNK_CUDA_CHECK(cudaStreamSynchronize(st));
      fprintf(stderr, "[nnk fastdtw cycles/pair] build=%llu window=%llu cost=%llu wavefront=%llu backtrack=%llu\n",
              h[0] / a->n_pairs, h[1] / a->n_pairs, h[2] / a->n_pairs, h[3] / a->n_pairs, h[4] / a->n_pairs);
    }
  }
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int nnk_gather_rows(const void* X, int32_t dtype, int64_t x_pair_stride, int32_t x_ld, const int32_t* path,
                               int32_t path_ld, const int32_t* path_len, void* out, int64_t out_pair_stride,
                               int32_t out_rows, int32_t D, int32_t n_pairs, void* stream) {
  NNK_REQUIRE(X && path && path_len && out, NNK_ERR_ARG, "NULL pointer");
  if (n_pairs == 0 || out_rows == 0 || D == 0) return NNK_OK;
  DeviceGuard guard(X);
  cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((unsigned)(((int64_t)out_rows * D + 255) / 256), (unsigned)n_pairs);
  if (grid.x > 1024) grid.x = 1024;
  if (dtype == NNK_F32)
    gather_rows_kernel<float><<<grid, 256, 0, st>>>((const float*)X, x_pair_stride, x_ld, path, path_ld, path_len, (float*)out, out_pair_stride, out_rows, D);
  else
    gather_rows_kernel<double><<<grid, 256, 0, st>>>((const double*)X, x_pair_stride, x_ld, path, path_ld, path_len, (double*)out, out_pair_stride, out_rows, D);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}

extern "C" int nnk_trim_lengths(const void* X, int32_t dtype, int64_t pair_stride, int32_t ld, int32_t T, int32_t D,
                                double eps, int32_t n_pairs, int32_t* len, void* stream) {
  NNK_REQUIRE(X && len, NNK_ERR_ARG, "NULL pointer");
  if (n_pairs == 0) return NNK_OK;
  DeviceGuard guard(X);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == NNK_F32) trim_len_kernel<float><<<n_pairs, 128, 0, st>>>((const float*)X, pair_stride, ld, T, D, (float)eps, len);
  else trim_len_kernel<double><<<n_pairs, 128, 0, st>>>((const double*)X, pair_stride, ld, T, D, eps, len);
  count_launch();
  NNK_CUDA_CHECK(cudaGetLastError());
  return NNK_OK;
}
