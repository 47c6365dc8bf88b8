/*
 * mplb_trajsolve.cu — batched TrajSolver / PolySolver on the GPU (SURVEY section 8f.4, first half).
 *
 * Reference: TrajSolver<Dim>::solve (MPL/include/mpl_traj_solver/traj_solver.h:73-109), PolySolver<Dim>::solve
 * (MPL/src/mpl_traj_solver/poly_solver.cpp:23-221), PolyTraj<Dim>::toPrimitives (MPL/src/mpl_traj_solver/poly_traj.cpp:75-92):
 * the closed-form minimum-derivative polynomial spline through a waypoint list (Richter-style unconstrained QP):
 *   A (boundary-derivative matrix), Q (cost Hessian), M (raw -> [fixed | free] derivative selection),
 *   X = A^-1 M, R = X^T Q X, Dp = -Rpp^-1 Rpf Df, d = M [Df; Dp], p_s = A_s^-1 d_s, coeff_k = p_k k!.
 *
 * The reference builds every matrix dense at (segments*N)^2 and calls Eigen's PartialPivLU on them.  A and Q are block
 * diagonal (one N x N block per segment, N = 2, 4, 6) and M has a single 1 per row, so here one CTA owns one trajectory
 * and works on the blocks only:
 *   phase 1  one thread per segment: A_s, its partial-pivot LU, A_s^-1 column by column, T_s = A_s^-T Q_s
 *   phase 2  one thread per entry of the free rows of R: the running sum over the (at most two) segments both
 *            derivatives touch, in the dense product's summation order
 *   phase 3  Rpf * Df, then a CTA-parallel partial-pivot LU of Rpp with the right-hand side carried as extra columns
 *            (pivot search by warp 0, row swap / scaling / rank-1 update by all threads) and the back substitution
 *   phase 4  one thread per (segment, axis): p = A_s^-1 d_s and the six Primitive coefficients
 * Skipping the structural zeros is exact in IEEE arithmetic (x - 0*y = x, acc + 0 = acc for finite values), every
 * element receives the same operations in the same order as the dense textbook algorithm (first maximal pivot; forward
 * substitution ascending, back substitution descending with a division by the diagonal), products and sums are explicit
 * __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn, so the result is bit-identical to the CPU checker's restatement of the dense
 * algorithm (tests/test_gpu_trajsolver.py; that checker is pinned to the reference's own sources).  Against a real Eigen build the difference is Eigen's blocking of the large dense
 * products (rounding level); tests state the tolerance.
 *
 * Work space per CTA: 3*S*N^2 + Wd*(ncol + 1) ... doubles (S segments, Wd = W*N/2 derivatives); it lives in shared memory
 * when it fits the opt-in limit and in a global scratch buffer (L2 resident) otherwise.  Position axes and yaw are two
 * independent solves: blockIdx.y selects which.
 *
 * FP64 pipe / latency bound, not HBM bound: 36 trajectories of 36 waypoints are ~1 MB of traffic.  Algorithmic bytes per
 * trajectory: W * 112 B of waypoints + S * 8 B of times read, S * (Dim + 1) * 48 B written.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mplb.h"
#include "mplb_internal.h"
#include "mplb_ref.h"

namespace {

constexpr int TS_THREADS = 256;
constexpr int TS_MAXN = 6;

struct TsJob {
  int wp_off;   /* first waypoint of this trajectory in the concatenated list */
  int n_wp;     /* W */
  int seg_off;  /* first segment in the concatenated dts / coefs */
  int pad;
  long long ws_off; /* global scratch offset in doubles, per (trajectory, solve) */
};

struct TsView { /* carve-up of one CTA's work space */
  double *Alu, *Ainv, *T, *D, *Rf, *B;
  int *piv, *newid, *att, *misc;
};

__host__ __device__ inline size_t ts_ws_doubles(int W, int N, int ncol) {
  const size_t S = W - 1, Wd = (size_t)W * N / 2;
  size_t d = 3 * S * N * N + Wd * ncol /*D*/ + Wd * Wd /*Rf upper bound*/ + Wd * ncol /*B*/;
  size_t ints = 2 * S * N + 2 * Wd + 8;
  return d + (ints + 1) / 2;
}

__device__ inline TsView ts_carve(double *ws, int W, int N, int ncol) {
  const size_t S = W - 1, Wd = (size_t)W * N / 2;
  TsView v;
  v.Alu = ws; ws += S * N * N;
  v.Ainv = ws; ws += S * N * N;
  v.T = ws; ws += S * N * N;
  v.D = ws; ws += Wd * ncol;
  v.Rf = ws; ws += Wd * Wd;
  v.B = ws; ws += Wd * ncol;
  int *iw = reinterpret_cast<int *>(ws);
  v.piv = iw; iw += S * N;
  v.newid = iw; iw += S * N;
  v.att = iw; iw += 2 * Wd;
  v.misc = iw;
  return v;
}

__device__ inline double ts_power(double t, int n) { /* math.h:197-203 */
  double tn = 1;
  while (n > 0) { tn = __dmul_rn(tn, t); n--; }
  return tn;
}

/* N x N partial-pivot LU of one segment block (column-major a[r + c*N]), Eigen's unblocked order */
__device__ void ts_block_lu(double *a, int *piv, int N) {
  for (int k = 0; k < N; k++) {
    int p = k;
    double best = fabs(a[k + k * N]);
    for (int r = k + 1; r < N; r++) {
      const double v = fabs(a[r + k * N]);
      if (v > best) { best = v; p = r; }
    }
    piv[k] = p;
    if (best != 0) {
      if (p != k)
        for (int c = 0; c < N; c++) { const double t = a[k + c * N]; a[k + c * N] = a[p + c * N]; a[p + c * N] = t; }
      const double d = a[k + k * N];
      for (int r = k + 1; r < N; r++) a[r + k * N] = __ddiv_rn(a[r + k * N], d);
    }
    for (int c = k + 1; c < N; c++)
      for (int r = k + 1; r < N; r++) a[r + c * N] = __dsub_rn(a[r + c * N], __dmul_rn(a[r + k * N], a[k + c * N]));
  }
}

/* x := A^-1 x for one right-hand side, through the block's LU */
__device__ void ts_block_solve(const double *a, const int *piv, int N, double *x) {
  for (int k = 0; k < N; k++)
    if (piv[k] != k) { const double t = x[k]; x[k] = x[piv[k]]; x[piv[k]] = t; }
  for (int i = 0; i < N; i++) {
    double acc = x[i];
    for (int j = 0; j < i; j++) acc = __dsub_rn(acc, __dmul_rn(a[i + j * N], x[j]));
    x[i] = acc;
  }
  for (int i = N - 1; i >= 0; i--) {
    double acc = x[i];
    for (int j = N - 1; j > i; j--) acc = __dsub_rn(acc, __dmul_rn(a[i + j * N], x[j]));
    x[i] = __ddiv_rn(acc, a[i + i * N]);
  }
}

/* One solve (position axes: ncol = dim, order from `control`; yaw: ncol = 1, order from `yaw_control`). */
__global__ void __launch_bounds__(TS_THREADS)
k_traj_solve(const TsJob *jobs, const mplb_waypoint *wps, const double *dts, double *coefs, int dim, int Npos, int Rpos,
             int Nyaw, int Ryaw, int yaw_control, double *gscratch, int smem_doubles) {
  extern __shared__ double ts_smem[];
  const TsJob job = jobs[blockIdx.x];
  const bool is_yaw = blockIdx.y == 1;
  const int N = is_yaw ? Nyaw : Npos, R_ = is_yaw ? Ryaw : Rpos, ncol = is_yaw ? 1 : dim;
  const int W = job.n_wp, S = W - 1, H = N / 2, Wd = W * H;
  const int tid = threadIdx.x, nt = blockDim.x;
  if (W < 2) return;
  const size_t need = ts_ws_doubles(W, N, ncol);
  double *ws = need <= (size_t)smem_doubles ? ts_smem : gscratch + job.ws_off + (is_yaw ? ts_ws_doubles(W, Npos, dim) : 0);
  const TsView v = ts_carve(ws, W, N, ncol);
  const mplb_waypoint *wp = wps + job.wp_off;
  const double *dt = dts + job.seg_off;
  int *s_nfixed = v.misc, *s_pivrow = v.misc + 1;

  /* use_xxx of waypoint w, derivative k (traj_solver.h:88-97 for yaw: interior Control::VEL, ends yaw_control) */
  auto use = [&](int w, int k) -> bool {
    const int c = is_yaw ? ((w == 0 || w == W - 1) ? yaw_control : 1) : wp[w].control;
    return (c >> k) & 1;
  };
  auto value = [&](int w, int k, int a) -> double {
    if (is_yaw) return k == 0 ? wp[w].yaw : 0.0;
    const mplb_waypoint &q = wp[w];
    return k == 0 ? q.pos[a] : k == 1 ? q.vel[a] : k == 2 ? q.acc[a] : q.jrk[a];
  };

  /* ---- permutation table (ps:90-160): raw id -> new id, fixed derivatives first; thread 0, O(W) */
  if (tid == 0) {
    int nfixed = 0;
    for (int w = 0; w < W; w++)
      for (int k = 0; k < H; k++) nfixed += use(w, k) ? 1 : 0;
    int raw = 0, fix = 0, fre = 0;
    for (int i = 0; i < 2 * Wd; i++) v.att[i] = -1;
    for (int w = 0; w < W; w++) {
      const bool interior = w > 0 && w < W - 1;
      for (int k = 0; k < H; k++) {
        const bool u = use(w, k);
        const int nid = u ? fix : nfixed + fre;
        v.newid[raw] = nid;
        v.att[2 * nid] = raw; /* attachments in ascending raw (= ascending segment) order */
        if (interior) { v.newid[raw + H] = nid; v.att[2 * nid + 1] = raw + H; }
        if (u) { /* Df (ps:189-203) */
          for (int a = 0; a < ncol; a++) v.D[nid * ncol + a] = value(w, k, a);
          fix++;
        } else fre++;
        raw++;
      }
      if (interior) raw += H;
    }
    *s_nfixed = nfixed;
  }
  /* ---- phase 1: per-segment blocks */
  for (int s = tid; s < S; s += nt) {
    double *a = v.Alu + (size_t)s * N * N, *ai = v.Ainv + (size_t)s * N * N, *t = v.T + (size_t)s * N * N;
    const double seg_time = dt[s];
    for (int i = 0; i < N * N; i++) a[i] = 0;
    for (int n = 0; n < N; n++) { /* ps:43-58 */
      if (n < H) {
        int val = 1;
        for (int m = 0; m < n; m++) val *= (n - m);
        a[n + n * N] = val;
      }
      for (int r = 0; r < H; r++)
        if (r <= n) {
          int val = 1;
          for (int m = 0; m < r; m++) val *= (n - m);
          a[(H + r) + n * N] = __dmul_rn((double)val, ts_power(seg_time, n - r));
        }
    }
    ts_block_lu(a, v.piv + s * N, N);
    for (int c = 0; c < N; c++) { /* column c of A_s^-1 = solve(e_c) */
      double x[TS_MAXN];
      for (int i = 0; i < N; i++) x[i] = i == c ? 1.0 : 0.0;
      ts_block_solve(a, v.piv + s * N, N, x);
      for (int i = 0; i < N; i++) ai[i + c * N] = x[i];
    }
    /* T_s(col, c) = sum_k Ainv(k, col) * Q_s(k, c), k ascending (ps:60-68 for Q, ps:175 for the product) */
    for (int col = 0; col < N; col++)
      for (int c = 0; c < N; c++) {
        double acc = 0;
        for (int k = 0; k < N; k++) {
          double q = 0;
          if (k >= R_ && c >= R_) {
            int val = 1;
            for (int m = 0; m < R_; m++) val *= (k - m) * (c - m);
            const int e = k + c - 2 * R_ + 1;
            q = __ddiv_rn(__dmul_rn((double)val, ts_power(seg_time, e)), (double)e);
          }
          acc = __dadd_rn(acc, __dmul_rn(ai[k + col * N], q));
        }
        t[col + c * N] = acc;
      }
  }
  __syncthreads();
  const int nfixed = *s_nfixed, nfree = Wd - nfixed;
  double *Rf = v.Rf; /* free rows of R: Rf[a * Wd + j] = R(nfixed + a, j) */
  double *B = v.B;   /* nfree x ncol */

  if (W > 2 && nfree > 0) {
    /* ---- phase 2: R(i, j) = sum_c (X^T Q)(i, c) X(c, j), c ascending over the segments that carry both i and j */
    for (int e = tid; e < nfree * Wd; e += nt) {
      const int a = e / Wd, j = e - a * Wd, i = nfixed + a;
      double acc = 0;
      for (int ia = 0; ia < 2; ia++) {
        const int ri = v.att[2 * i + ia];
        if (ri < 0) continue;
        const int s = ri / N;
        int rj = -1;
        for (int ja = 0; ja < 2; ja++) {
          const int r = v.att[2 * j + ja];
          if (r >= 0 && r / N == s) rj = r;
        }
        if (rj < 0) continue;
        const double *t = v.T + (size_t)s * N * N, *ai = v.Ainv + (size_t)s * N * N;
        const int li = ri - s * N, lj = rj - s * N;
        for (int c = 0; c < N; c++) acc = __dadd_rn(acc, __dmul_rn(t[li + c * N], ai[c + lj * N]));
      }
      Rf[(size_t)a * Wd + j] = acc;
    }
    __syncthreads();
    /* ---- phase 3a: B = Rpf * Df (ps:210), f ascending */
    for (int e = tid; e < nfree * ncol; e += nt) {
      const int a = e / ncol, col = e - a * ncol;
      double acc = 0;
      for (int f = 0; f < nfixed; f++) acc = __dadd_rn(acc, __dmul_rn(Rf[(size_t)a * Wd + f], v.D[f * ncol + col]));
      B[a * ncol + col] = acc;
    }
    __syncthreads();
    /* ---- phase 3b: partial-pivot LU of Rpp = Rf[:, nfixed:], right-hand side carried along */
    double *P = Rf + nfixed; /* P(r, c) = P[r * Wd + c] */
    for (int k = 0; k < nfree; k++) {
      if (tid < 32) { /* first row of maximal magnitude in column k */
        double best = -1.0;
        int p = k;
        for (int r = k + tid; r < nfree; r += 32) {
          const double val = fabs(P[(size_t)r * Wd + k]);
          if (val > best) { best = val; p = r; }
        }
        for (int o = 16; o > 0; o >>= 1) {
          const double ob = __shfl_down_sync(0xffffffffu, best, o);
          const int op = __shfl_down_sync(0xffffffffu, p, o);
          if (ob > best || (ob == best && op < p)) { best = ob; p = op; }
        }
        if (tid == 0) { s_pivrow[0] = p; s_pivrow[1] = best != 0 ? 1 : 0; }
      }
      __syncthreads();
      const int p = s_pivrow[0];
      const bool nonzero = s_pivrow[1] != 0;
      if (p != k) { /* swap rows k and p: all nfree columns (L part included, as Eigen does) and the right-hand side */
        for (int c = tid; c < nfree + ncol; c += nt) {
          double *x = c < nfree ? &P[(size_t)k * Wd + c] : &B[k * ncol + (c - nfree)];
          double *y = c < nfree ? &P[(size_t)p * Wd + c] : &B[p * ncol + (c - nfree)];
          const double t = *x; *x = *y; *y = t;
        }
        __syncthreads();
      }
      if (nonzero) {
        const double d = P[(size_t)k * Wd + k];
        for (int r = k + 1 + tid; r < nfree; r += nt) P[(size_t)r * Wd + k] = __ddiv_rn(P[(size_t)r * Wd + k], d);
        __syncthreads();
      }
      const int rem = nfree - k - 1, width = rem + ncol;
      for (int e = tid; e < rem * width; e += nt) {
        const int r = k + 1 + e / width, cc = e % width;
        const double l = P[(size_t)r * Wd + k];
        if (cc < rem) {
          const int c = k + 1 + cc;
          P[(size_t)r * Wd + c] = __dsub_rn(P[(size_t)r * Wd + c], __dmul_rn(l, P[(size_t)k * Wd + c]));
        } else {
          const int c = cc - rem;
          B[r * ncol + c] = __dsub_rn(B[r * ncol + c], __dmul_rn(l, B[k * ncol + c]));
        }
      }
      __syncthreads();
    }
    /* ---- phase 3c: back substitution, column oriented (j descending), then Dp = -x (ps:210-212) */
    for (int j = nfree - 1; j >= 0; j--) {
      if (tid < ncol) B[j * ncol + tid] = __ddiv_rn(B[j * ncol + tid], P[(size_t)j * Wd + j]);
      __syncthreads();
      for (int e = tid; e < j * ncol; e += nt) {
        const int i = e / ncol, c = e - i * ncol;
        B[i * ncol + c] = __dsub_rn(B[i * ncol + c], __dmul_rn(P[(size_t)i * Wd + j], B[j * ncol + c]));
      }
      __syncthreads();
    }
    for (int e = tid; e < nfree * ncol; e += nt) v.D[(nfixed + e / ncol) * ncol + e % ncol] = -B[e];
  } else {
    for (int e = tid; e < nfree * ncol; e += nt) v.D[(nfixed + e / ncol) * ncol + e % ncol] = 0.0;
  }
  __syncthreads();
  /* ---- phase 4: p = A_s^-1 d_s (ps:215-221), coeff(k) = p(k) * k!, reversed (poly_traj.cpp:80-86) */
  for (int e = tid; e < S * ncol; e += nt) {
    const int s = e / ncol, a = e - s * ncol;
    double x[TS_MAXN];
    for (int i = 0; i < N; i++) x[i] = v.D[v.newid[s * N + i] * ncol + a];
    ts_block_solve(v.Alu + (size_t)s * N * N, v.piv + s * N, N, x);
    double *o = coefs + ((size_t)(job.seg_off + s) * (dim + 1) + (is_yaw ? dim : a)) * 6;
    int fact = 1;
    double c6[6] = {0, 0, 0, 0, 0, 0};
    for (int k = 0; k < N; k++) {
      if (k > 0) fact *= k;
      c6[k] = __dmul_rn(x[k], (double)fact);
    }
    for (int k = 0; k < 6; k++) o[k] = c6[5 - k];
  }
}

bool ts_orders(int control, int *N, int *R) { /* traj_solver.h:21-27 */
  const int c = control & 0xf;
  if (c == 1) { *N = 2; *R = 1; return true; }
  if (c == 3) { *N = 4; *R = 2; return true; }
  if (c == 7) { *N = 6; *R = 3; return true; }
  return false;
}

/* staging bytes of one host thread on the device that was current when they were last grown (a different current device
 * reallocates them there); freed when the thread exits */
struct TsScratch : DevBuf<char> {
  int dev = -1;
  cudaError_t reserve(size_t want) {
    int cur = 0;
    cudaError_t e = cudaGetDevice(&cur);
    if (e != cudaSuccess) return e;
    if (cur != dev) { release(); dev = cur; }
    return DevBuf<char>::reserve(want);
  }
};
thread_local TsScratch g_jobs, g_ws, g_wps, g_dts, g_coefs;
thread_local mplb_traj_solve_stats g_stats; /* what the last ts_run of this host thread launched */

/* launches the solve for `jobs` (wp_off / n_wp / seg_off filled by the caller; ws_off is assigned here) */
int ts_run(int dim, int Np, int Rp, int Ny, int Ry, int yaw_control, std::vector<TsJob> &jobs, const mplb_waypoint *d_wps,
           const double *d_dts, double *d_coefs, cudaStream_t stream) {
  g_stats = mplb_traj_solve_stats{};
  size_t ws_total = 0, ws_max = 0;
  for (TsJob &j : jobs) {
    j.ws_off = (long long)ws_total;
    const size_t a = ts_ws_doubles(j.n_wp, Np, dim), b = ts_ws_doubles(j.n_wp, Ny, 1);
    ws_total += a + b;
    ws_max = std::max(ws_max, std::max(a, b));
  }
  if (jobs.empty()) return MPLB_OK;
  int dev = 0, smem_optin = 0;
  MPLB_CUDA_TRY(cudaGetDevice(&dev));
  MPLB_CUDA_TRY(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t smem_cap = (size_t)std::max(0, smem_optin - 1024);
  const size_t smem_bytes = std::min(ws_max * sizeof(double), smem_cap) / 8 * 8;
  mplb_traj_solve_stats st{};
  st.n_traj = (int32_t)jobs.size();
  st.smem_bytes = (int64_t)smem_bytes;
  for (const TsJob &j : jobs) { /* the kernel's per-CTA test: need <= smem_bytes / 8 */
    const bool pos_g = ts_ws_doubles(j.n_wp, Np, dim) > smem_bytes / 8, yaw_g = ts_ws_doubles(j.n_wp, Ny, 1) > smem_bytes / 8;
    (pos_g ? st.pos_global : st.pos_shared)++;
    (yaw_g ? st.yaw_global : st.yaw_shared)++;
    st.max_wp = std::max(st.max_wp, (int32_t)j.n_wp);
  }
  const bool need_global = st.pos_global + st.yaw_global > 0;
  MPLB_CUDA_TRY(g_jobs.reserve(jobs.size() * sizeof(TsJob)));
  if (need_global) {
    /* the dense formulation is O(W^2) memory per trajectory like the reference's (segments*N)^2 matrices: refuse absurd sizes */
    if (ws_total * sizeof(double) > ((size_t)8 << 30)) return mplb_internal_fail(MPLB_ERR_NOMEM, "traj_solve: work space above 8 GiB (waypoint lists this long are out of this solver's range)");
    MPLB_CUDA_TRY(g_ws.reserve(ws_total * sizeof(double)));
    st.global_bytes = (int64_t)(ws_total * sizeof(double));
  }
  MPLB_CUDA_TRY(cudaMemcpyAsync(g_jobs.p, jobs.data(), jobs.size() * sizeof(TsJob), cudaMemcpyHostToDevice, stream));
  MPLB_CUDA_TRY(cudaFuncSetAttribute(k_traj_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes));
  k_traj_solve<<<dim3((unsigned)jobs.size(), 2), TS_THREADS, smem_bytes, stream>>>(
      (const TsJob *)g_jobs.p, d_wps, d_dts, d_coefs, dim, Np, Rp, Ny, Ry, yaw_control, (double *)g_ws.p, (int)(smem_bytes / 8));
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cudaStreamSynchronize(stream)); /* the job list is reused by the next call */
  g_stats = st;
  return MPLB_OK;
}

int ts_launch(int dim, int control, int yaw_control, int n_traj, const int32_t *wp_offsets, const mplb_waypoint *d_wps,
              const double *d_dts, double *d_coefs, int32_t *n_segs, cudaStream_t stream) {
  int Np = 0, Rp = 0, Ny = 0, Ry = 0;
  const bool ok = ts_orders(control, &Np, &Rp) && (yaw_control == 1 || yaw_control == 3 || yaw_control == 7) &&
                  ts_orders(yaw_control, &Ny, &Ry);
  std::vector<TsJob> jobs;
  int seg_off = 0, unsolved_slots = 0;
  for (int i = 0; i < n_traj; i++) {
    const int W = wp_offsets[i + 1] - wp_offsets[i];
    const int slots = std::max(W - 1, 0);
    const int nseg = ok ? slots : 0; /* an uninitialised solver or < 2 waypoints give an empty Trajectory */
    if (n_segs) n_segs[i] = nseg;
    const int my_off = seg_off;
    seg_off += slots;
    unsolved_slots += slots - nseg;
    if (!nseg) continue;
    TsJob j;
    j.wp_off = wp_offsets[i] - wp_offsets[0]; j.n_wp = W; j.seg_off = my_off; j.pad = 0; j.ws_off = 0;
    jobs.push_back(j);
  }
  if (unsolved_slots) { /* only an uninitialised solver leaves slots unsolved, and then it leaves all of them: zero them like
                          the host variant does, and return once that is done as a solve would */
    MPLB_CUDA_TRY(cudaMemsetAsync(d_coefs, 0, (size_t)seg_off * (dim + 1) * 6 * sizeof(double), stream));
    if (jobs.empty()) MPLB_CUDA_TRY(cudaStreamSynchronize(stream));
  }
  return ts_run(dim, Np, Rp, Ny, Ry, yaw_control, jobs, d_wps, d_dts, d_coefs, stream);
}

/* Trajectory::getWaypoints (trajectory.h:277-289) of every plan of a batch, written as the waypoint lists the solver reads:
 * waypoint j < n_seg = the stored coord of segment j's parent (Primitive::evaluate(0) returns the coefficients c5, c4, c3, c2
 * = that state exactly), waypoint n_seg = the last primitive evaluated at its duration (pr:321-331 in the reference's term
 * order, mplb_ref.h); the two ends keep the plan's control flags, the interior ones become Control::VEL (map_planner_node.cpp:217-219).
 * Plan i is read with cfgs[cfg_id ? cfg_id[i] : 0].
 * pick == NULL: one thread per (plan, waypoint), plan i owns slots [i * (max_seg + 1), ...) of wps and [i * max_seg, ...) of dts,
 *   t = j dt (the solver reads only the dts).
 * pick != NULL: one thread per plan, the single waypoint pick[i] into wps[i] with the plan's control flags and t the running sum
 *   0 + dt + ... + dt of getWaypoints (the next start of map_replanner_node.cpp:243-253); ok[i] = 0 and wps[i] untouched where the
 *   plan failed, was truncated (n_seg > max_seg) or has no waypoint pick[i]. */
__global__ void k_gather_waypoints(const mplb_result *res, const int *actions, const double *segs, int n, int max_seg,
                                   const MplbTrajCfg *cfgs, const int *cfg_id, const int *pick, mplb_waypoint *wps, double *dts, int *ok) {
  const int per = pick ? 1 : max_seg + 1;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)n * per) return;
  const int i = (int)(idx / per);
  const int j = pick ? pick[i] : (int)(idx % per);
  const int ns = res[i].n_seg;
  const bool have = res[i].status == MPLB_PLAN_OK && ns >= 1 && ns <= max_seg && j >= 0 && j <= ns;
  if (pick) ok[i] = have ? 1 : 0;
  if (!have) return;
  const MplbTrajCfg c = cfgs[cfg_id ? cfg_id[i] : 0];
  const int dim = c.dim, plan_control = c.control;
  const double dt = c.dt;
  mplb_waypoint w;
  memset(&w, 0, sizeof(w));
  if (j < ns) {
    const double *st = segs + ((size_t)i * max_seg + j) * 13;
    for (int k = 0; k < 3; k++) { w.pos[k] = st[k]; w.vel[k] = st[3 + k]; w.acc[k] = st[6 + k]; w.jrk[k] = st[9 + k]; }
    w.yaw = st[12];
    if (!pick) dts[(size_t)i * max_seg + j] = dt;
  } else {
    const double *st = segs + ((size_t)i * max_seg + ns - 1) * 13;
    const int a = actions[(size_t)i * max_seg + ns - 1];
    mplb_ref::Prim pr;
    double e[13];
    mplb_ref::prim_build(dim, c.ord, st, c.U + a * 3, pr);
    mplb_ref::prim_eval(dim, pr, dt, e);
    for (int k = 0; k < dim; k++) { w.pos[k] = e[k]; w.vel[k] = e[3 + k]; w.acc[k] = e[6 + k]; w.jrk[k] = e[9 + k]; }
    if ((plan_control & 16) && c.Uyaw) /* pr_yaw_.p(t) = c4 t + c5 with the zero terms in front, then normalize_angle */
      w.yaw = mplb_ref::normalize_angle(mplb_ref::dadd(mplb_ref::dmul(c.Uyaw[a], dt), st[12]));
  }
  if (pick) {
    double t = 0.0; /* trajectory.h:280-287 */
    for (int m = 0; m < j; m++) t = __dadd_rn(t, dt);
    w.t = t;
    w.control = plan_control;
    wps[i] = w;
  } else {
    w.t = __dmul_rn((double)j, dt);
    w.control = (j == 0 || j == ns) ? plan_control : MPLB_CONTROL_VEL;
    wps[(size_t)i * per + j] = w;
  }
}

/* the gather of every waypoint, then one solve over the plans that are complete in the rows */
int refine_run(int dim, const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const mplb_result *d_res, const int *d_acts, const double *d_segs,
               int n, int max_seg, int control, int yaw_control, double *d_coefs, int32_t *n_segs, cudaStream_t stream);

thread_local TsScratch g_pwps, g_pdts, g_pU, g_pres;

int refine_run(int dim, const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const mplb_result *d_res, const int *d_acts, const double *d_segs,
               int n, int max_seg, int control, int yaw_control, double *d_coefs, int32_t *n_segs, cudaStream_t stream) {
  int Np = 0, Rp = 0, Ny = 0, Ry = 0;
  const bool ok = ts_orders(control, &Np, &Rp) && (yaw_control == 1 || yaw_control == 3 || yaw_control == 7) && ts_orders(yaw_control, &Ny, &Ry);
  std::vector<mplb_result> res(n);
  MPLB_CUDA_TRY(cudaMemcpyAsync(res.data(), d_res, (size_t)n * sizeof(mplb_result), cudaMemcpyDeviceToHost, stream));
  MPLB_CUDA_TRY(cudaStreamSynchronize(stream));
  const int per = max_seg + 1;
  std::vector<TsJob> jobs;
  for (int i = 0; i < n; i++) {
    const bool good = ok && res[i].status == MPLB_PLAN_OK && res[i].n_seg >= 1 && res[i].n_seg <= max_seg;
    if (n_segs) n_segs[i] = good ? res[i].n_seg : 0;
    if (!good) continue;
    TsJob j;
    j.wp_off = i * per; j.n_wp = res[i].n_seg + 1; j.seg_off = i * max_seg; j.pad = 0; j.ws_off = 0;
    jobs.push_back(j);
  }
  MPLB_CUDA_TRY(g_pwps.reserve((size_t)n * per * sizeof(mplb_waypoint)));
  MPLB_CUDA_TRY(g_pdts.reserve((size_t)n * max_seg * sizeof(double)));
  MPLB_CUDA_TRY(cudaMemsetAsync(d_coefs, 0, (size_t)n * max_seg * (dim + 1) * 6 * sizeof(double), stream));
  const long long total = (long long)n * per;
  k_gather_waypoints<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(d_res, d_acts, d_segs, n, max_seg, d_cfgs, d_cfg_id, nullptr,
                                                                           (mplb_waypoint *)g_pwps.p, (double *)g_pdts.p, nullptr);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  return ts_run(dim, Np, Rp, Ny, Ry, yaw_control, jobs, (const mplb_waypoint *)g_pwps.p, (const double *)g_pdts.p, d_coefs, stream);
}

}  // namespace

int mplb_internal_refine(int dim, const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const void *d_results, const void *d_actions,
                         const void *d_seg_states, int n, int max_seg, int control, int yaw_control, void *d_coefs, int32_t *n_segs,
                         void *stream) {
  return refine_run(dim, d_cfgs, d_cfg_id, (const mplb_result *)d_results, (const int *)d_actions, (const double *)d_seg_states, n,
                    max_seg, control, yaw_control, (double *)d_coefs, n_segs, (cudaStream_t)stream);
}

int mplb_internal_pick_waypoints(const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const void *d_results, const void *d_actions,
                                 const void *d_seg_states, int n, int max_seg, const void *d_pick, void *d_wps, void *d_ok, void *stream) {
  k_gather_waypoints<<<(unsigned)((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      (const mplb_result *)d_results, (const int *)d_actions, (const double *)d_seg_states, n, max_seg, d_cfgs, d_cfg_id,
      (const int *)d_pick, (mplb_waypoint *)d_wps, nullptr, (int *)d_ok);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  return MPLB_OK;
}

extern "C" {

int mplb_traj_solve_last_stats(mplb_traj_solve_stats *out) {
  if (!out) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve_last_stats: null output");
  *out = g_stats;
  return MPLB_OK;
}

int mplb_traj_solve_batch_device(int dim, int control, int yaw_control, int n_traj, const int32_t *wp_offsets,
                                 const void *d_wps, const void *d_dts, void *d_coefs, int32_t *n_segs, void *stream) {
  if (dim != 2 && dim != 3) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: dim must be 2 or 3");
  if (n_traj < 0 || !wp_offsets) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: bad trajectory list");
  if (n_traj == 0) return MPLB_OK;
  for (int i = 0; i < n_traj; i++)
    if (wp_offsets[i + 1] < wp_offsets[i]) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: offsets must not decrease");
  return ts_launch(dim, control, yaw_control, n_traj, wp_offsets, (const mplb_waypoint *)d_wps, (const double *)d_dts,
                   (double *)d_coefs, n_segs, (cudaStream_t)stream);
}

int mplb_refine_trajectories_device(mplb_planner *p, const void *d_results, const void *d_actions, const void *d_seg_states, int n,
                                    int max_seg, int plan_control, int control, int yaw_control, void *d_coefs, int32_t *n_segs,
                                    void *stream_) {
  if (!p || !d_results || !d_actions || !d_seg_states || !d_coefs || n < 0 || max_seg < 1) return mplb_internal_fail(MPLB_ERR_ARG, "refine: bad argument");
  if (n == 0) return MPLB_OK;
  cudaStream_t stream = (cudaStream_t)stream_;
  MplbLpaHostCfg hc;
  mplb_internal_planner_cfg(p, &hc);
  if (hc.nU <= 0) return mplb_internal_fail(MPLB_ERR_STATE, "refine: no controls set");
  MPLB_CUDA_TRY(cudaSetDevice(hc.device));
  /* the batch's one configuration: the planner's controls and dt, the control flags it was planned with */
  MPLB_CUDA_TRY(g_pU.reserve((size_t)hc.nU * 4 * sizeof(double) + sizeof(MplbTrajCfg)));
  MplbTrajCfg *d_cfg = (MplbTrajCfg *)g_pU.p;
  double *d_U = (double *)(g_pU.p + sizeof(MplbTrajCfg));
  MPLB_CUDA_TRY(cudaMemcpyAsync(d_U, hc.U, (size_t)hc.nU * 3 * sizeof(double), cudaMemcpyHostToDevice, stream));
  double *d_Uyaw = nullptr;
  if (hc.Uyaw) {
    d_Uyaw = d_U + (size_t)hc.nU * 3;
    MPLB_CUDA_TRY(cudaMemcpyAsync(d_Uyaw, hc.Uyaw, (size_t)hc.nU * sizeof(double), cudaMemcpyHostToDevice, stream));
  }
  const int cc = plan_control & 15;
  MplbTrajCfg t;
  std::memset(&t, 0, sizeof(t));
  t.dim = hc.dim; t.ord = cc == 1 ? 1 : cc == 3 ? 2 : cc == 7 ? 3 : 4; t.control = plan_control; t.use_yaw = (plan_control & 16) ? 1 : 0;
  t.U = d_U; t.Uyaw = d_Uyaw; t.dt = hc.dt;
  MPLB_CUDA_TRY(cudaMemcpyAsync(d_cfg, &t, sizeof(t), cudaMemcpyHostToDevice, stream));
  return refine_run(hc.dim, d_cfg, nullptr, (const mplb_result *)d_results, (const int *)d_actions, (const double *)d_seg_states, n,
                    max_seg, control, yaw_control, (double *)d_coefs, n_segs, stream);
}

int mplb_refine_trajectories(mplb_planner *p, const mplb_result *results, const int32_t *actions, const double *seg_states, int n,
                             int max_seg, int plan_control, int control, int yaw_control, double *coefs, int32_t *n_segs) {
  if (!p || !results || !actions || !seg_states || !coefs || n < 0 || max_seg < 1) return mplb_internal_fail(MPLB_ERR_ARG, "refine: bad argument");
  if (n == 0) return MPLB_OK;
  MplbLpaHostCfg hc;
  mplb_internal_planner_cfg(p, &hc);
  MPLB_CUDA_TRY(cudaSetDevice(hc.device));
  const size_t nc = (size_t)n * max_seg * (hc.dim + 1) * 6;
  MPLB_CUDA_TRY(g_pres.reserve((size_t)n * sizeof(mplb_result)));
  MPLB_CUDA_TRY(g_wps.reserve((size_t)n * max_seg * sizeof(int)));         /* staging: actions */
  MPLB_CUDA_TRY(g_dts.reserve((size_t)n * max_seg * 13 * sizeof(double))); /* staging: segment states */
  MPLB_CUDA_TRY(g_coefs.reserve(nc * sizeof(double)));
  MPLB_CUDA_TRY(cudaMemcpy(g_pres.p, results, (size_t)n * sizeof(mplb_result), cudaMemcpyHostToDevice));
  MPLB_CUDA_TRY(cudaMemcpy(g_wps.p, actions, (size_t)n * max_seg * sizeof(int), cudaMemcpyHostToDevice));
  MPLB_CUDA_TRY(cudaMemcpy(g_dts.p, seg_states, (size_t)n * max_seg * 13 * sizeof(double), cudaMemcpyHostToDevice));
  const int rc = mplb_refine_trajectories_device(p, g_pres.p, g_wps.p, g_dts.p, n, max_seg, plan_control, control, yaw_control, g_coefs.p, n_segs, nullptr);
  if (rc != MPLB_OK) return rc;
  MPLB_CUDA_TRY(cudaMemcpy(coefs, g_coefs.p, nc * sizeof(double), cudaMemcpyDeviceToHost));
  return MPLB_OK;
}

int mplb_traj_solve_batch(int dim, int control, int yaw_control, int n_traj, const int32_t *wp_offsets, const mplb_waypoint *wps,
                          const double *dts, double *coefs, int32_t *n_segs) {
  if (dim != 2 && dim != 3) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: dim must be 2 or 3");
  if (n_traj < 0 || !wp_offsets || (n_traj > 0 && (!wps || !dts || !coefs)))
    return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: null buffer");
  if (n_traj == 0) return MPLB_OK;
  if (wp_offsets[0] != 0) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: wp_offsets[0] must be 0");
  const int n_wp = wp_offsets[n_traj];
  int n_seg_total = 0;
  for (int i = 0; i < n_traj; i++) {
    if (wp_offsets[i + 1] < wp_offsets[i]) return mplb_internal_fail(MPLB_ERR_ARG, "traj_solve: offsets must not decrease");
    n_seg_total += std::max(wp_offsets[i + 1] - wp_offsets[i] - 1, 0);
  }
  const size_t n_seg_slots = (size_t)std::max(n_seg_total, 1);
  MPLB_CUDA_TRY(g_wps.reserve((size_t)std::max(n_wp, 1) * sizeof(mplb_waypoint)));
  MPLB_CUDA_TRY(g_dts.reserve(n_seg_slots * sizeof(double)));
  MPLB_CUDA_TRY(g_coefs.reserve(n_seg_slots * (dim + 1) * 6 * sizeof(double)));
  MPLB_CUDA_TRY(cudaMemcpy(g_wps.p, wps, (size_t)n_wp * sizeof(mplb_waypoint), cudaMemcpyHostToDevice));
  MPLB_CUDA_TRY(cudaMemcpy(g_dts.p, dts, (size_t)n_seg_total * sizeof(double), cudaMemcpyHostToDevice));
  MPLB_CUDA_TRY(cudaMemset(g_coefs.p, 0, n_seg_slots * (dim + 1) * 6 * sizeof(double)));
  const int rc = mplb_traj_solve_batch_device(dim, control, yaw_control, n_traj, wp_offsets, g_wps.p, g_dts.p, g_coefs.p, n_segs, nullptr);
  if (rc != MPLB_OK) return rc;
  MPLB_CUDA_TRY(cudaMemcpy(coefs, g_coefs.p, (size_t)n_seg_total * (dim + 1) * 6 * sizeof(double), cudaMemcpyDeviceToHost));
  return MPLB_OK;
}
}
