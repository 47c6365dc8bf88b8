/* mplb_fleet.cu — a fleet of LPA* replanners sharded over the GPUs of a box (DESIGN.md section 6.1).
 *
 * Robot i lives on rank i mod N, the striping of mplb_plan_batch_sharded.  Every rank holds a replica of the shared map; a
 * replan cycle's map edits are exchanged so that every replica applies the same rows in global robot order, and the cycle's
 * plans are gathered to one root in robot order.  Both use the communicator's grouped ncclSend / ncclRecv (mplb.cu); links,
 * updates and getSubStateSpace stay rank-local and use the single-device batch calls. */
#include <cuda_runtime.h>

#include <climits>
#include <string>
#include <unordered_set>
#include <vector>

#include "mplb_internal.h"

namespace {

int fail(int code, const std::string &msg) { return mplb_internal_fail(code, msg.c_str()); }

/* One rank's send payload, int32 words: the n_local per-robot row counts, then the rows (3 ints each) in local robot order.
 * The robots' lists are rows offs[0] .. offs[n_local] - 1 of cells3. */
__global__ void k_fleet_pack(const int *cells3, const long long *offs, int n_local, int *payload) {
  const long long rows = offs[n_local] - offs[0];
  const long long words = n_local + 3 * rows;
  for (long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x; w < words; w += (long long)gridDim.x * blockDim.x)
    payload[w] = w < n_local ? (int)(offs[w + 1] - offs[w]) : cells3[3 * offs[0] + (w - n_local)];
}

/* The received payloads (rank r's at word woff[r], nloc[r] robots, rows[r] rows) -> the robot-ordered offsets all_offs[0 .. R]
 * and, per robot, the word of its first row in the receive buffer.  One block: thread t < N walks rank t's robots for the local
 * row prefix (and sets *bad when their counts do not add up to rows[t]); then the block scans the R counts in global robot order
 * (robot i = rank i mod N, its (i / N)-th local robot). */
__global__ void __launch_bounds__(1024) k_fleet_scan(const int *recv, const long long *woff, const int *nloc, const long long *rows,
                                                     int nranks, int R, long long *all_offs, long long *src_word, int *bad) {
  __shared__ long long part[1024];
  const int t = threadIdx.x;
  if (t == 0) *bad = 0;
  __syncthreads();
  if (t < nranks) {
    long long row = 0;
    for (int k = 0; k < nloc[t]; k++) {
      src_word[(long long)k * nranks + t] = woff[t] + nloc[t] + 3 * row;
      const int c = recv[woff[t] + k];
      if (c < 0) atomicExch(bad, 1);
      row += c;
    }
    if (row != rows[t]) atomicExch(bad, 1);
  }
  const int per = (R + blockDim.x - 1) / blockDim.x, lo = min(R, t * per), hi = min(R, lo + per);
  long long sum = 0;
  for (int i = lo; i < hi; i++) sum += recv[woff[i % nranks] + i / nranks];
  part[t] = sum;
  __syncthreads();
  for (int d = 1; d < (int)blockDim.x; d <<= 1) { /* inclusive Hillis-Steele scan of the per-thread sums */
    const long long v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  long long run = part[t] - sum;
  for (int i = lo; i < hi; i++) {
    all_offs[i] = run;
    run += recv[woff[i % nranks] + i / nranks];
  }
  if (t == blockDim.x - 1) all_offs[R] = part[t];
}

/* Output row j -> its robot i (the last i with all_offs[i] <= j) -> the row's words in the receive buffer.  Writes nothing when
 * the scan found the counts inconsistent. */
__global__ void k_fleet_merge(const int *recv, const long long *all_offs, const long long *src_word, int R, long long total,
                              const int *bad, int *all_cells3) {
  if (*bad) return;
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < total; j += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = R - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) / 2;
      if (all_offs[mid] <= j) lo = mid; else hi = mid - 1;
    }
    const long long w = src_word[lo] + 3 * (j - all_offs[lo]);
    all_cells3[3 * j] = recv[w];
    all_cells3[3 * j + 1] = recv[w + 1];
    all_cells3[3 * j + 2] = recv[w + 2];
  }
}

/* robots of rank `rank` among n_total striped over nranks */
int stripe_count(int n_total, int rank, int nranks) { return n_total > rank ? (n_total - rank + nranks - 1) / nranks : 0; }

int grid_for(long long work) { return (int)std::min<long long>((work + 255) / 256, 4096); }

/* device scratch of one merge: per-rank word offsets, robots and rows, per-robot source words, the consistency flag */
struct MergeScratch {
  long long *woff, *rows, *src;
  int *nloc, *bad;
};

/* scan + merge of the received payloads (enqueued on s): robot-ordered rows into all_cells3, R + 1 offsets into all_offs */
int merge_payloads(const int *recv, const std::vector<long long> &woff, const std::vector<int> &nloc, const std::vector<long long> &rows,
                   int R, long long total, const MergeScratch &t, void *all_cells3, void *all_offs, cudaStream_t s) {
  const int N = (int)nloc.size();
  MPLB_CUDA_TRY(cudaMemcpyAsync(t.woff, woff.data(), N * sizeof(long long), cudaMemcpyHostToDevice, s));
  MPLB_CUDA_TRY(cudaMemcpyAsync(t.rows, rows.data(), N * sizeof(long long), cudaMemcpyHostToDevice, s));
  MPLB_CUDA_TRY(cudaMemcpyAsync(t.nloc, nloc.data(), N * sizeof(int), cudaMemcpyHostToDevice, s));
  k_fleet_scan<<<1, 1024, 0, s>>>(recv, t.woff, t.nloc, t.rows, N, R, (long long *)all_offs, t.src, t.bad);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  if (total > 0) {
    k_fleet_merge<<<grid_for(total), 256, 0, s>>>(recv, (const long long *)all_offs, t.src, R, total, t.bad, (int *)all_cells3);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  return MPLB_OK;
}

/* scratch slots of a communicator used by the fleet calls */
enum { SL_MINE, SL_HDR, SL_SEND, SL_RECV, SL_OFFS, SL_MERGE, SL_RES, SL_ACT };

}  // namespace

extern "C" {

int64_t mplb_fleet_map_edit(mplb_comm *c, mplb_map *m, const void *d_cells3, const int64_t *offsets_local, int n_local, int value,
                            void *d_all_cells3, void *d_all_offsets, int64_t cap, void *stream) {
  if (!c) return fail(MPLB_ERR_ARG, "fleet map edit: null communicator");
  MplbCommView cv;
  mplb_internal_comm_view(c, &cv);
  /* an argument error of this rank is not returned at once: it travels in the header exchange, so that every rank fails alike
     instead of leaving the others waiting in the exchange */
  std::string err;
  long long rows = 0;
  if (!m || n_local < 0 || cap < 0 || (n_local > 0 && !offsets_local) || (cap > 0 && !d_all_cells3)) {
    err = "fleet map edit: null argument";
  } else {
    MplbMapView mv;
    mplb_internal_map_view(m, &mv);
    if (mv.device != cv.device) err = "fleet map edit: the map is not on the communicator's device";
    for (int k = 0; k < n_local && err.empty(); k++)
      if (offsets_local[k] < 0 || offsets_local[k + 1] < offsets_local[k] || offsets_local[k + 1] - offsets_local[k] > INT_MAX)
        err = "fleet map edit: bad cell offsets";
    if (err.empty() && n_local > 0) rows = offsets_local[n_local] - offsets_local[0];
    if (err.empty() && rows > 0 && !d_cells3) err = "fleet map edit: null cell list";
  }
  if (mplb_internal_set_device(cv.device)) return fail(MPLB_ERR_CUDA, "cannot select the communicator's device");
  /* the caller's rows are written on `stream`; the exchange runs on the communicator's own stream */
  if (err.empty() && cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess) err = "fleet map edit: the caller's stream failed";
  const cudaStream_t s = (cudaStream_t)cv.stream;
  const int N = cv.nranks;
  if (N > 1024) return fail(MPLB_ERR_ARG, "fleet map edit: more than 1024 ranks"); /* the same on every rank */
  /* exchange 1: (rows, robots, cap, flags) of every rank; flags: 1 = an argument error here, 2 = a size query (no offsets buffer) */
  const long long mine[4] = {err.empty() ? rows : 0, err.empty() ? n_local : 0, cap, (err.empty() ? 0 : 1) | (d_all_offsets ? 0 : 2)};
  long long *d_mine = (long long *)mplb_internal_comm_scratch(c, SL_MINE, sizeof(mine));
  long long *d_hdr = (long long *)mplb_internal_comm_scratch(c, SL_HDR, sizeof(mine) * N);
  if (!d_mine || !d_hdr) return MPLB_ERR_CUDA;
  MPLB_CUDA_TRY(cudaMemcpyAsync(d_mine, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  std::vector<size_t> hb(N, sizeof(mine));
  int rc = mplb_internal_comm_allgather(c, d_mine, hb.data(), d_hdr, s);
  if (rc) return rc;
  std::vector<long long> hdr(4 * (size_t)N);
  MPLB_CUDA_TRY(cudaMemcpyAsync(hdr.data(), d_hdr, hdr.size() * sizeof(long long), cudaMemcpyDeviceToHost, s));
  MPLB_CUDA_TRY(cudaStreamSynchronize(s));
  /* from here on every rank decides the same way from the same numbers, so all of them return or all of them go on */
  if (!err.empty()) return fail(MPLB_ERR_ARG, err);
  long long R = 0, total = 0;
  std::vector<long long> woff(N + 1, 0), nrows(N);
  std::vector<int> nloc(N);
  for (int r = 0; r < N; r++) {
    const long long *h = &hdr[4 * (size_t)r];
    if (h[3] & 1) return fail(MPLB_ERR_ARG, "fleet map edit: an argument error on rank " + std::to_string(r));
    if (h[2] != cap || (h[3] & 2) != (mine[3] & 2))
      return fail(MPLB_ERR_ARG, "fleet map edit: every rank must pass the same cap, and all or none of them ask for the size");
    total += h[0]; R += h[1];
    nrows[r] = h[0];
    nloc[r] = (int)h[1];
    woff[r + 1] = woff[r] + h[1] + 3 * h[0];
  }
  if (R > INT_MAX) return fail(MPLB_ERR_ARG, "fleet map edit: too many robots");
  for (int r = 0; r < N; r++)
    if (nloc[r] != stripe_count((int)R, r, N))
      return fail(MPLB_ERR_ARG, "fleet map edit: the robots per rank do not follow the striping robot i -> rank i mod N");
  if (total > INT_MAX) return fail(MPLB_ERR_ARG, "fleet map edit: more than 2^31 - 1 cells");
  /* a size query, or a cap (the same on every rank) below the total: every rank sees total > its cap, nothing is exchanged or
     applied anywhere */
  if (!d_all_offsets || total > cap) return total;
  if (R == 0) return 0;
  /* exchange 2: the payloads */
  int *send = (int *)mplb_internal_comm_scratch(c, SL_SEND, (size_t)std::max<long long>(n_local + 3 * rows, 1) * sizeof(int));
  int *recv = (int *)mplb_internal_comm_scratch(c, SL_RECV, (size_t)std::max<long long>(woff[N], 1) * sizeof(int));
  long long *d_offs = (long long *)mplb_internal_comm_scratch(c, SL_OFFS, ((size_t)n_local + 1) * sizeof(long long));
  unsigned char *ms = (unsigned char *)mplb_internal_comm_scratch(c, SL_MERGE, (2 * (size_t)N + R) * sizeof(long long) + (N + 1) * sizeof(int));
  if (!send || !recv || !d_offs || !ms) return MPLB_ERR_CUDA;
  MergeScratch t;
  t.woff = (long long *)ms; t.rows = t.woff + N; t.src = t.rows + N; t.nloc = (int *)(t.src + R); t.bad = t.nloc + N;
  if (n_local > 0) {
    MPLB_CUDA_TRY(cudaMemcpyAsync(d_offs, offsets_local, ((size_t)n_local + 1) * sizeof(long long), cudaMemcpyHostToDevice, s));
    k_fleet_pack<<<grid_for(n_local + 3 * rows), 256, 0, s>>>((const int *)d_cells3, d_offs, n_local, send);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  std::vector<size_t> pb(N);
  for (int r = 0; r < N; r++) pb[r] = (size_t)(woff[r + 1] - woff[r]) * sizeof(int);
  rc = mplb_internal_comm_allgather(c, send, pb.data(), recv, s);
  if (rc) return rc;
  rc = merge_payloads(recv, woff, nloc, nrows, (int)R, total, t, d_all_cells3, d_all_offsets, s);
  if (rc) return rc;
  /* every replica applies the same rows in the same order: mplb_map_set_cells_device, brick rebuild included; it returns once
     the cells and the bricks are written */
  rc = mplb_map_set_cells_device(m, d_all_cells3, (int)total, value, s);
  if (rc) return rc;
  if (total == 0) MPLB_CUDA_TRY(cudaStreamSynchronize(s)); /* no cell to write: the offsets are the last work */
  return total;
}

int64_t mplb_fleet_merge_device(const void *d_payloads, const int64_t *payload_words, int nranks, int n_total, void *d_all_cells3,
                                void *d_all_offsets, int64_t cap, void *stream) {
  if (nranks < 1 || nranks > 1024 || n_total < 0 || !payload_words || cap < 0 || (cap > 0 && !d_all_cells3) ||
      (n_total > 0 && !d_all_offsets))
    return fail(MPLB_ERR_ARG, "fleet merge: bad argument");
  std::vector<long long> woff(nranks + 1, 0), rows(nranks);
  std::vector<int> nloc(nranks);
  long long total = 0;
  for (int r = 0; r < nranks; r++) {
    nloc[r] = stripe_count(n_total, r, nranks);
    const long long w = payload_words[r] - nloc[r];
    if (w < 0 || w % 3) return fail(MPLB_ERR_ARG, "fleet merge: a payload's size does not fit its robots");
    rows[r] = w / 3;
    total += rows[r];
    woff[r + 1] = woff[r] + payload_words[r];
  }
  if (woff[nranks] > 0 && !d_payloads) return fail(MPLB_ERR_ARG, "fleet merge: null payloads");
  if (total > INT_MAX) return fail(MPLB_ERR_ARG, "fleet merge: more than 2^31 - 1 cells");
  if (total > cap || n_total == 0) return total;
  DevBuf<unsigned char> ms;
  MPLB_CUDA_TRY(ms.reserve((2 * (size_t)nranks + n_total) * sizeof(long long) + (nranks + 1) * sizeof(int)));
  MergeScratch t;
  t.woff = (long long *)ms.p; t.rows = t.woff + nranks; t.src = t.rows + nranks; t.nloc = (int *)(t.src + n_total);
  t.bad = t.nloc + nranks;
  const cudaStream_t s = (cudaStream_t)stream;
  int rc = merge_payloads((const int *)d_payloads, woff, nloc, rows, n_total, total, t, d_all_cells3, d_all_offsets, s);
  if (rc) return rc;
  int bad = 0;
  MPLB_CUDA_TRY(cudaMemcpyAsync(&bad, t.bad, sizeof(int), cudaMemcpyDeviceToHost, s));
  MPLB_CUDA_TRY(cudaStreamSynchronize(s));
  if (bad) return fail(MPLB_ERR_ARG, "fleet merge: a payload's robot counts do not add up to its rows");
  return total;
}

int mplb_fleet_plan(mplb_comm *c, mplb_planner **planners_local, int n_local, int n_total, const mplb_waypoint *starts_local,
                    const mplb_waypoint *goals_local, mplb_result *results, int32_t *actions, int max_seg, int root) {
  if (!c) return fail(MPLB_ERR_ARG, "fleet plan: null communicator");
  MplbCommView cv;
  mplb_internal_comm_view(c, &cv);
  /* this rank's argument checks; the verdicts of all ranks are exchanged before any planner changes, so that every rank fails
     alike instead of leaving the others waiting in the gather */
  std::string err;
  int code = MPLB_ERR_ARG;
  if (n_local < 0 || n_total < 0 || max_seg < 0 || (n_local > 0 && (!planners_local || !starts_local || !goals_local)))
    err = "fleet plan: null argument";
  else if (root < 0 || root >= cv.nranks)
    err = "fleet plan: bad root";
  else if (n_local != stripe_count(n_total, cv.rank, cv.nranks))
    err = "fleet plan: n_local does not match n_total and the striping robot i -> rank i mod N";
  else if (cv.rank == root && n_total > 0 && (!results || (max_seg > 0 && !actions)))
    err = "fleet plan: the root needs a result buffer (and an action buffer when max_seg > 0)";
  std::unordered_set<mplb_planner *> seen;
  for (int k = 0; k < n_local && err.empty(); k++) {
    mplb_planner *p = planners_local[k];
    MplbLpaHostCfg cfg;
    if (!p) { err = "fleet plan: null planner"; break; }
    if (!seen.insert(p).second) { err = "fleet plan: a planner appears twice"; break; }
    mplb_internal_planner_cfg(p, &cfg);
    if (cfg.device != cv.device) err = "fleet plan: a planner is not on the communicator's device";
    else if (!mplb_internal_lpa_enabled(p)) { err = "fleet plan: every planner must have LPA* enabled"; code = MPLB_ERR_STATE; }
  }
  if (mplb_internal_set_device(cv.device)) return fail(MPLB_ERR_CUDA, "cannot select the communicator's device");
  const cudaStream_t s = (cudaStream_t)cv.stream;
  const int N = cv.nranks;
  const long long mine[3] = {err.empty() ? 0 : 1, n_total, max_seg}; /* the verdict and the arguments every rank must share */
  long long *d_mine = (long long *)mplb_internal_comm_scratch(c, SL_MINE, sizeof(mine));
  long long *d_hdr = (long long *)mplb_internal_comm_scratch(c, SL_HDR, sizeof(mine) * N);
  if (!d_mine || !d_hdr) return MPLB_ERR_CUDA;
  MPLB_CUDA_TRY(cudaMemcpyAsync(d_mine, mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  std::vector<size_t> hb(N, sizeof(mine));
  int rc = mplb_internal_comm_allgather(c, d_mine, hb.data(), d_hdr, s);
  if (rc) return rc;
  std::vector<long long> hdr(3 * (size_t)N);
  MPLB_CUDA_TRY(cudaMemcpyAsync(hdr.data(), d_hdr, hdr.size() * sizeof(long long), cudaMemcpyDeviceToHost, s));
  MPLB_CUDA_TRY(cudaStreamSynchronize(s));
  if (!err.empty()) return fail(code, err);
  for (int r = 0; r < N; r++) {
    const long long *h = &hdr[3 * (size_t)r];
    if (h[0]) return fail(MPLB_ERR_ARG, "fleet plan: an argument error on rank " + std::to_string(r));
    if (h[1] != n_total || h[2] != max_seg) return fail(MPLB_ERR_ARG, "fleet plan: every rank must pass the same n_total and max_seg");
  }
  if (n_total == 0) return MPLB_OK;
  std::vector<mplb_result> res((size_t)std::max(n_local, 1));
  if (n_local > 0) {
    rc = mplb_lpa_plan_batch(planners_local, n_local, starts_local, goals_local, res.data());
    if (rc) return rc;
  }
  if (mplb_internal_set_device(cv.device)) return fail(MPLB_ERR_CUDA, "cannot select the communicator's device");
  /* the fixed-stride rows mplb_plan_batch_sharded gathers: per = ceil(n_total / N) records and action rows (-1 padded; a
     plan that did not succeed has no trajectory, a longer one keeps its first max_seg actions) */
  const int per = (n_total + N - 1) / N;
  std::vector<mplb_result> hres((size_t)per);
  std::vector<int32_t> hact((size_t)per * max_seg, -1);
  for (int k = 0; k < n_local; k++) {
    hres[k] = res[k];
    if (max_seg > 0 && res[k].status == MPLB_PLAN_OK) mplb_get_actions(planners_local[k], &hact[(size_t)k * max_seg], max_seg);
  }
  void *d_res = mplb_internal_comm_scratch(c, SL_RES, (size_t)per * sizeof(mplb_result));
  void *d_act = max_seg > 0 ? mplb_internal_comm_scratch(c, SL_ACT, hact.size() * sizeof(int32_t)) : nullptr;
  if (!d_res || (max_seg > 0 && !d_act)) return MPLB_ERR_CUDA;
  MPLB_CUDA_TRY(cudaMemcpyAsync(d_res, hres.data(), (size_t)per * sizeof(mplb_result), cudaMemcpyHostToDevice, s));
  if (max_seg > 0) MPLB_CUDA_TRY(cudaMemcpyAsync(d_act, hact.data(), hact.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  rc = mplb_internal_comm_gather(c, d_res, d_act, per, max_seg, root, s);
  if (rc) return rc;
  MPLB_CUDA_TRY(cudaStreamSynchronize(s));
  if (cv.rank == root) return mplb_comm_unstripe(c, n_total, per, max_seg, results, max_seg > 0 ? actions : nullptr);
  if (results) std::copy(res.begin(), res.begin() + n_local, results);
  return MPLB_OK;
}

}  // extern "C"
