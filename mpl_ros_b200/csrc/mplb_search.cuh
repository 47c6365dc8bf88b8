/*
 * mplb_search.cuh — the fused A* kernel: one CTA owns one plan; a persistent grid drains a batch.
 *
 * Reference path restated per pop (paths under motion_primitive_library/include/):
 *   GraphSearch::Astar            mpl_planner/common/graph_search.h:39-182   (pop, relax, terminate)
 *   env_map::get_succ             mpl_planner/env/env_map.h:147-172          (phase B1: one lane per control u)
 *   env_map::traverse_primitive   mpl_planner/env/env_map.h:90-132           (phase B2: one thread per sample)
 *   env_map::is_goal + rayTrace   env_map.h:25-45, mpl_collision/map_util.h:117-134
 *   priorityQueue / compare_pair  mpl_planner/common/state_space.h:15-34     (binary heap, same sift rules as
 *                                 boost::heap::d_ary_heap<arity<2>, mutable_<true>> so pop order is identical)
 *   recoverTraj                   graph_search.h:369-455 (best-predecessor rule kept as a running argmin)
 *
 * The search of one plan is a serial chain of pops, so the kernel is latency-bound per plan (dependent FP64 ops, divisions,
 * shared-memory loads, shuffles and HBM round trips; tools/ub/lat.cu measures their latencies) and throughput comes from
 * running several hundred plans at once.  One pop is organised so that almost nothing sits on the serial chain:
 *
 *   warp 0  (search)  B1 when it was not prepared one pop ahead: one lane per control — exact FP64 end state,
 *                     validation, lattice key, sample count; issues the hash-table probe of every candidate successor
 *                     (ONE HBM round trip: the table slot carries the node's g and best-predecessor g) and computes h
 *                     while they fly; after the barrier it relaxes all successors lane-parallel and performs the heap
 *                     pushes in control order with a warp-cooperative sift-up on the SHARED-MEMORY heap, then takes
 *                     the next node off the root.
 *   warps 1-6 (sample) every collision sample of every control (flat list of 8-sample granules) through a FILTERED
 *                     path: an FP64 Horner evaluation in cell units decides the voxel whenever the sample is not
 *                     within a proven guard band of a voxel boundary, otherwise the exact FP64 formula of the
 *                     reference is evaluated; warp 1 also runs the goal test and the parity hash of the current node.
 *   warp 7  (heap)    finishes the previous pop's sift-down, prefetches the new root's state row, and runs B1 for
 *                     that node (the predicted next pop) into the second expansion record while the other warps
 *                     expand the current node.
 *
 * A second set of instantiations (POT = true, |U| <= 32 and |U| > 32) adds the cost-shaping branches of env_map (search
 * region, potential map, env_map.h:104-118) and the yaw controls (primitive.h:236-253,503-525, env_map.h:121-128); the
 * plain instantiations carry none of that code.
 *
 * Exactness: every value that is stored or compared (states, costs, g, h, f, keys, voxel indices) is identical to the
 * reference's double arithmetic; filters only skip work when the exact result is provably the same.  Rare hazards
 * (two successors of one expansion mapping to one node or one table slot) drop to a serial generic routine.
 *
 * Search state of a plan lives in a private HBM arena (table, node records, state rows, heap spill); the only data
 * shared between CTAs is the read-only map (occupancy bit-bricks) and the control / sample-time tables.
 */
#pragma once
#include "mplb_device.cuh"
#include "mplb_trig.cuh"
#include "../../include/mplb.h"

namespace mplb {

/* tuning knobs (chosen on the bench workload with tools/phase_timing.py, cycles per pop) */
#ifndef MPLB_WIN
#define MPLB_WIN 1 /* table slots fetched per probe (load factor <= 1/4): at 4-6 CTAs/SM one slot wins; the second slot is
                      bandwidth and registers for a 1-in-8 case */
#endif
#ifndef MPLB_LOAD_INV
#define MPLB_LOAD_INV 4 /* table load factor bound 1/4 */
#endif
#ifndef MPLB_TINIT
#define MPLB_TINIT 1024 /* initial table slots (<= smallest tsize_max the host allocates) */
#endif
#ifndef MPLB_HCAP
#define MPLB_HCAP 512 /* heap entries kept in shared memory (|U| <= 32 instantiations): 6 CTAs of 160 threads per SM need <= 37 KB each */
#endif
#define MPLB_HCAP_SMALL 1024 /* shared-memory heap entries of the |U| > 32 instantiations when several plans share an SM */
/* The ancestor ranges of the deep-heap pushes are fetched with the bulk asynchronous copy engine (cp.async.bulk + mbarrier,
 * UBLKCP / SYNCS in SASS): one copy per tree level, <= 23 per pop.  -DMPLB_NO_BULK_PREFETCH selects the 8-byte cp.async
 * (LDGSTS) variant; the two measured within noise of each other on the |U| = 125 workload. */
#if !defined(MPLB_NO_BULK_PREFETCH) && !defined(MPLB_BULK_PREFETCH)
#define MPLB_BULK_PREFETCH 1
#endif
#ifndef MPLB_B1_INLINE
#define MPLB_B1_INLINE __forceinline__ /* __noinline__ adds cycles to every pop */
#endif
#ifndef MPLB_SIFTUP_INLINE
#define MPLB_SIFTUP_INLINE __forceinline__ /* __noinline__ adds cycles to every pop */
#endif

#define MPLB_INTERNAL_OVERFLOW 100 /* arena too small: host retries the plan in a larger tier */
#define MPLB_INTERNAL_BADCTRL 9
#define MPLB_TT_CAP 1024           /* float sample times kept in shared memory */
#define MPLB_NCAP 64               /* sample divisors n < 64 tabulated in shared memory */

/* Table slot = one 32-byte sector: key, node id and the two values every relaxation compares against. */
struct __align__(32) Slot {
  unsigned long long k0;
  unsigned int k1lo;
  unsigned int node1; /* node id + 1; 0 = empty */
  double g;           /* copy of NodeHot::g */
  double pg;          /* copy of NodeHot::pg */
};
static_assert(sizeof(Slot) == 32, "Slot must be 32 bytes");

struct __align__(32) NodeHot {
  double g, h;
  double pg;       /* g of the best predecessor (tie rule of recoverTraj, gs:391-405) */
  int heap_pos;    /* position of the live heap entry while open */
  short action;    /* action id of parent -> this */
  unsigned char flags; /* 1 = iterationopened, 2 = iterationclosed */
  unsigned char pad0;
};
static_assert(sizeof(NodeHot) == 32, "NodeHot must be 32 bytes");

/* Header of a state row, followed by NS doubles of state (the stored coord of the node). */
struct __align__(16) RowHdr {
  unsigned long long k0, k1; /* packed lattice key */
  int parent;                /* best predecessor node */
  int slot;                  /* table slot of this node (kept current across table growth) */
  int pred_head;             /* newest predecessor record of this node in the predecessor log (-1 = none; log mode only) */
  int depth;                 /* primitives between the start and this node's FIRST discoverer: its stored time is
                                start.t + depth additions of dt (em:161), which is all the prior-trajectory heuristic needs */
};
static_assert(sizeof(RowHdr) == 32, "RowHdr must be 32 bytes");

/* One predecessor record (gs:100-102), kept only in log mode: when a node's g can still change after it was relaxed
 * (eps > 1, an inconsistent heuristic) recoverTraj (gs:391-405) must see every predecessor with its FINAL g. */
struct PredRec {
  double cost; /* pred_action_cost */
  int pred;    /* pred node */
  int next;    /* previous record of the same successor (-1 = end): the list runs newest -> oldest */
  int action;  /* pred_action_id */
  int pad;
};
static_assert(sizeof(PredRec) == 24, "PredRec must be 24 bytes");

struct HeapEnt {
  double f; /* heap key (gs:54,119) */
  double g; /* copy of node g for compare_pair's tie-break (ss:19-24) */
  int node; /* bit 31 set: entry is a re-push of an already closed node (gs:135-141) */
  int pad;
};
static_assert(sizeof(HeapEnt) == 24, "HeapEnt must be 24 bytes");

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

/* cmp(a,b) of compare_pair: true iff a is worse (lower priority) than b. */
__device__ __forceinline__ bool heap_worse(double af, double ag, double bf, double bg) {
  return (af == bf) ? (ag > bg) : (af > bf);
}

struct BatchArgs {
  const mplb_waypoint *starts, *goals;
  mplb_result *results;
  int *actions;       /* [n * max_seg] or null */
  double *seg_states; /* [n * max_seg * 13] or null */
  int max_seg;
  const int *work;    /* plan ids of this tier (null = identity) */
  int n_work;
  int *work_counter;
  unsigned char *arena; /* slot s at arena + s*stride */
  size_t stride;
  int cap;       /* nodes (and heap entries, pop-log entries) per slot */
  int tsize_max; /* table slots per slot arena (power of two) */
  int hcap;      /* shared-memory heap entries of this launch (|U| > 32 instantiations; see PlanSmem) */
  int load_inv;  /* table load factor bound 1/load_inv of this tier (MPLB_LOAD_INV in the small tiers, 2 in the large ones) */
  size_t off_rows, off_heap, off_table, off_poplog, off_log;
  int log_cap; /* predecessor records per slot; 0 = the running best-predecessor is exact for this configuration */
  int want_poplog;
  int *slot_of_plan;   /* optional: which slot ran plan i (retained single plan) */
  int *overflow_count; /* plans whose arena overflowed in this tier ... */
  int *overflow_list;  /* ... and their ids, for the next (larger) tier */
  long long *phase_cycles; /* diagnostics build only (MPLB_PHASE_TIMING): 8 accumulators per plan */
};

#ifdef MPLB_PHASE_TIMING
#define MPLB_TICK(k) do { if (tid == 0) { long long t__ = clock64(); ph[k] += t__ - tlast; tlast = t__; } } while (0)
#define MPLB_COUNT(k, v) atomicAdd(&S.dbg[k], (unsigned long long)(v))
#else
#define MPLB_COUNT(k, v) do { } while (0)
#define MPLB_TICK(k) do { } while (0)
#endif

/* Everything get_succ produces for one node (B1 outputs, sampling base, sample list, collision outcomes).  With
 * |U| <= 32 there are two of them: while the search warp commits the current node, the heap warp already runs B1 for
 * the node that will be popped next (the heap root after the previous pop's sift-down is the next pop unless a
 * successor overtakes it, which measured < 0.1 % of the pops). */
template <int DIM, int ORD, int MAXU, int XS = 0>
struct ExpBuf {
  static constexpr int NP = DIM * ORD; /* polynomial part of the state, [d*DIM + ax] */
  static constexpr int NS = NP + XS;   /* + yaw slot in the cost-shaping / yaw instantiations (index NP) */
  static constexpr int GCAP = MAXU * 8; /* 8-sample granules */
  double st[NS];     /* state of the expanded node */
  unsigned long long pk0, pk1; /* its packed lattice key (a successor with the same key is the self-loop of em:158) */
  int node, ready, key_bad, n_gran;
  double y0[3];      /* filtered sampling: cell coordinate of the parent and lower coefficients, in cells */
  double Ap[3 * 3];
  double es[MAXU * NS]; /* end states, [u][d*DIM+ax] */
  unsigned long long k0[MAXU], k1[MAXU];
  int verdict[MAXU]; /* 0 self, 1 dyn, 2 blocked, 3 valid, 4 valid-no-motion, 5 needs sampling (transient) */
  int nsamp[MAXU];   /* divisor n */
  int cnt[MAXU];     /* samples to test */
  int first[MAXU];   /* first blocked sample index or INT_MAX */
  int nid[MAXU];     /* node id of the successor after relaxation (for state forwarding) */
  int gbase[MAXU];   /* first granule of the control in gl[] (cost-shaping kernels only: they sum its sample terms in order) */
  double dts[MAXU];  /* sample spacing T/n (em:98), cost-shaping kernels only */
  double cy0, sy0;   /* cos/sin of the node's yaw (yaw controls) */
  unsigned int gl[GCAP];     /* granule: control | first sample k0 << 8 | sample count << 16 ... */
  unsigned short gl_t[GCAP]; /* ... and index of its first sample time in tts */
};

template <int DIM, int ORD, int NB, bool POT = false>
struct PlanSmem {
  static constexpr int NP = DIM * ORD;
  static constexpr int NS = NP + (POT ? 1 : 0);
  static constexpr int MAXU = 32 * NB;
  static constexpr int NBUF = 2; /* expansion records: B1 of the next pop is pipelined into the second one */
  /* granule order of the sample list (b1_warp): wave-major in the plain kernels, so that the sampler can skip the granules
   * behind a control's first blocked sample; control-major in the cost-shaping kernels, which need every sample's term */
  static constexpr bool WAVE_MAJOR = !POT;
  typedef ExpBuf<DIM, ORD, MAXU, POT ? 1 : 0> EB;
  EB eb[NBUF];
  int cur_buf;
  /* heap top (SoA) in shared memory.  |U| <= 32: a fixed MPLB_HCAP entries inside this struct.  |U| > 32: `hcap`
   * entries in the dynamic shared memory behind the struct, sized per launch (1024 when several plans share an SM, many
   * more when the arena size leaves one plan per SM anyway, as in the 1024^3 / |U| = 125 configuration). */
  static constexpr bool DYN_HEAP = (NB > 1);
  static constexpr int HCAP = DYN_HEAP ? 1 : MPLB_HCAP;
  double hf[HCAP], hg[HCAP];
  int hn[HCAP];
  int hcap;
  /* |U| > 32: ancestor cache of the pushes of one pop.  The k-th push of a pop lands on heap position n0 + k, so every
   * ancestor it can meet lies in one short contiguous range per tree level; those ranges are copied from the global part
   * of the heap into shared memory in ONE asynchronous round trip and kept coherent by write-through, instead of one
   * HBM round trip per push (~100 pushes per pop with |U| = 125). */
  static constexpr int ACAP = DYN_HEAP ? 320 : 1;
  alignas(16) HeapEnt ac[ACAP];
  unsigned long long ac_bar; /* mbarrier of the bulk-copy variant (MPLB_BULK_PREFETCH) */
  int ac_lo[32], ac_off[32], ac_cnt[32]; /* per level l >= 1: first cached position, offset in ac[], count */
  int ac_valid;
  /* pushes of one 32-control batch, in control order (block-parallel push, see push_batch_blocks) */
  static constexpr int QCAP = DYN_HEAP ? 32 : 1;
  double q_f[QCAP], q_g[QCAP];
  int q_n[QCAP], q_defer[QCAP];
  /* current node */
  double cur[NS];
  unsigned long long cur_k0, cur_k1; /* packed lattice key of the current node */
  double cur_g;
  unsigned long long cur_kh;
  int cur_node, cur_tag, goal_hit;
  double goal_pos[3], goal_vel[3], goal_acc[3];
  unsigned long long gk0, gk1;
  int goal_key_ok;
  /* per-plan constants */
  double U[MAXU * 3];
  double cost[MAXU];   /* J(u) + w*dt, eb:343-345 */
  double Ut[MAXU * 3]; /* u / ORD! exactly as pr:128-131 divides the leading coefficient */
  double Au[MAXU * 3]; /* top polynomial coefficient of the filtered sampling path, in cells */
  int toff_s[MPLB_NCAP], tcnt_s[MPLB_NCAP];
  /* probe results of warp 0 (staged in shared memory so nothing lives in registers across the barrier) */
  int p_nid[MAXU], p_slot[MAXU];
  double p_g[MAXU], p_pg[MAXU], p_h[MAXU];
  double tts[MPLB_TT_CAP]; /* accumulated sample times (em:98-99), all divisors */
  /* per-sample cost terms of the current expansion, by granule slot: the potential-map term and the yaw term (em:121-128).
   * |U| > 32: (term, yaw term) pairs in the dynamic shared memory behind the heap top, as many as the launch's controls
   * and largest sample divisor need (shaped_terms); a fixed MAXU * 64 here would not fit next to a useful heap top. */
  static constexpr bool DYN_TERMS = POT && DYN_HEAP;
  double terms[(POT && !DYN_TERMS) ? MAXU * 64 : 1];
  double yterms[(POT && !DYN_TERMS) ? MAXU * 64 : 1];
  double Uyaw[POT ? MAXU : 1];        /* yaw rate of each control */
  int n_before;      /* n_nodes before this expansion */
  int n_log;         /* predecessor records written (log mode) */
  int cur_depth, pf_depth; /* RowHdr::depth of the current node / of the prefetched root */
  /* pending sift-down (heap warp) and prefetched root row */
  int sd_pending, sd_n;
  double sd_f, sd_g;
  int pf_node;
  unsigned long long pf_k0, pf_k1;
  double pf_st[NS];
#ifdef MPLB_BULK_ROW
  alignas(16) unsigned char pf_row[(sizeof(RowHdr) + NS * sizeof(double) + 15) & ~15];
  unsigned long long pf_bar; /* mbarrier of the bulk row copy */
  unsigned pf_phase;
#endif
  int n_nodes, n_heap, tsize, pops, n_closed, status, plan_idx;
  long long n_samples, n_valid;
  unsigned long long t_start; /* %globaltimer when this CTA picked the plan up */
  unsigned long long pop_hash, closed_hash;
#ifdef MPLB_PHASE_TIMING
  unsigned long long dbg[8];
#endif
};

/* ---------------------------------------------------------------- heap in shared memory with global spill */
template <class SM>
__device__ __forceinline__ constexpr size_t heap_dyn_offset() { return (sizeof(SM) + 15) & ~(size_t)15; }

/* |U| > 32 cost-shaping kernels: the (term, yaw term) pairs behind the S.hcap heap entries (20 bytes each; the host keeps
 * hcap a multiple of 256, so the pairs start 16-byte aligned) */
template <class SM>
__device__ __forceinline__ double2 *shaped_terms(SM &S) {
  return reinterpret_cast<double2 *>(reinterpret_cast<unsigned char *>(&S) + heap_dyn_offset<SM>() + (size_t)S.hcap * 20);
}

template <class SM>
struct HeapView {
  SM &S;
  HeapEnt *spill; /* global array indexed by heap position (entries >= hcap live here) */
  NodeHot *hot;
  __device__ __forceinline__ int hcap() const { return SM::DYN_HEAP ? S.hcap : SM::HCAP; }
  __device__ __forceinline__ double *hf() const {
    if (SM::DYN_HEAP) return reinterpret_cast<double *>(reinterpret_cast<unsigned char *>(&S) + heap_dyn_offset<SM>());
    return S.hf;
  }
  __device__ __forceinline__ double *hg() const { return SM::DYN_HEAP ? hf() + S.hcap : S.hg; }
  __device__ __forceinline__ int *hn() const { return SM::DYN_HEAP ? reinterpret_cast<int *>(hf() + 2 * (size_t)S.hcap) : S.hn; }
  __device__ __forceinline__ void get(int i, double &f, double &g, int &n) const {
    if (i < hcap()) { f = hf()[i]; g = hg()[i]; n = hn()[i]; }
    else { HeapEnt e = spill[i]; f = e.f; g = e.g; n = e.node; }
  }
  __device__ __forceinline__ void set(int i, double f, double g, int n) const {
    if (i < hcap()) { hf()[i] = f; hg()[i] = g; hn()[i] = n; }
    else { HeapEnt e; e.f = f; e.g = g; e.node = n; e.pad = 0; spill[i] = e; }
    hot[n & 0x7fffffff].heap_pos = i;
  }
  __device__ __forceinline__ int node_at(int i) const { return (i < hcap()) ? hn()[i] : spill[i].node; }
  __device__ __forceinline__ void set_g(int i, double g) const { if (i < hcap()) hg()[i] = g; else spill[i].g = g; }

  /* serial push/increase: sift up while the parent is strictly worse (boost siftup) */
  __device__ __forceinline__ void sift_up(int pos, double f, double g, int n) const {
    while (pos != 0) {
      int par = (pos - 1) >> 1;
      double pf, pg; int pn;
      get(par, pf, pg, pn);
      if (heap_worse(pf, pg, f, g)) { set(pos, pf, pg, pn); pos = par; }
      else break;
    }
    set(pos, f, g, n);
  }
  /* warp-cooperative sift up: lane k examines ancestor k+1; identical result to the serial loop */
  __device__ MPLB_SIFTUP_INLINE void sift_up_warp(int pos, double f, double g, int n, int lane) const {
    int p1 = pos + 1;
    int depth = 31 - __clz(p1);            /* number of ancestors */
    int my = (p1 >> (lane + 1)) - 1;       /* ancestor lane+1 */
    bool have = lane < depth;
    double af = 0.0, ag = 0.0; int an = 0;
    if (have) get(my, af, ag, an);
    bool moves = have && heap_worse(af, ag, f, g);
    unsigned stopm = __ballot_sync(0xffffffffu, !moves); /* first non-moving ancestor (or beyond depth) */
    int stop = __ffs(stopm) - 1;                          /* ancestors 1..stop move down one level */
    if (lane < stop) set((p1 >> lane) - 1, af, ag, an);   /* ancestor lane+1 -> position of ancestor lane (lane 0: pos) */
    if (lane == 0) set((p1 >> stop) - 1, f, g, n);
    __syncwarp();
  }
  /* ---- |U| > 32: ancestor cache (see PlanSmem::ac).  Called by one full warp. */
  /* (forceinline on purpose: a HeapView whose address escapes into a call turns every shared-memory access generic) */
  __device__ __forceinline__ void cache_ancestors(int n0, int K, int lane) const {
    const int hc = hcap();
    int lo = 0, cnt = 0;
    if (lane >= 1) { /* lane l prepares level l: ancestors at distance l of the positions [n0, n0 + K) */
      lo = ((n0 + 1) >> lane) - 1;
      const int hi = ((n0 + K) >> lane) - 1;
      if (lo < hc) lo = hc; /* positions below hcap live in shared memory already */
      lo &= ~1;             /* even start and even count: 16-byte aligned, 48-byte granular ranges of 24-byte entries */
      cnt = hi - lo + 1;
      cnt = cnt > 0 ? ((cnt + 1) & ~1) : 0;
    }
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    const bool fits = total <= SM::ACAP;
    S.ac_lo[lane] = lo; S.ac_off[lane] = incl - cnt; S.ac_cnt[lane] = fits ? cnt : 0;
    __syncwarp();
    if (fits) {
#ifdef MPLB_BULK_PREFETCH
      /* one bulk asynchronous copy (TMA engine, cp.async.bulk) per level, completion on a shared-memory mbarrier */
      const unsigned bar = (unsigned)__cvta_generic_to_shared(&S.ac_bar);
      if (lane == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((unsigned)(total * 24)) : "memory");
      }
      __syncwarp();
      if (cnt > 0) {
        const unsigned dst = (unsigned)__cvta_generic_to_shared(&S.ac[incl - cnt]);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                     "l"(spill + lo), "r"((unsigned)(cnt * 24)), "r"(bar)
                     : "memory");
      }
      unsigned done = 0;
      while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar) : "memory");
      __syncwarp(); /* nobody polls the barrier any more */
      if (lane == 0) asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
#else
      for (int l = 1; l < 32; l++) { /* 8-byte asynchronous copies (LDGSTS), all levels in flight together */
        const int c_l = S.ac_cnt[l], lo_l = S.ac_lo[l], off_l = S.ac_off[l];
        for (int q = lane; q < c_l * 3; q += 32) {
          const unsigned dst = (unsigned)__cvta_generic_to_shared(reinterpret_cast<unsigned long long *>(&S.ac[off_l]) + q);
          const unsigned long long *src = reinterpret_cast<const unsigned long long *>(spill + lo_l) + q;
          asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
        }
      }
      asm volatile("cp.async.wait_all;" ::: "memory");
#endif
    }
    __syncwarp();
    if (lane == 0) S.ac_valid = 1;
    __syncwarp();
  }
  /* entry at position i, which is an ancestor at distance l >= 1 of a position the cache was built for */
  __device__ __forceinline__ void cget(int i, int l, double &f, double &g, int &n) const {
    if (i < hcap()) { f = hf()[i]; g = hg()[i]; n = hn()[i]; return; }
    const int k = i - S.ac_lo[l];
    if (k >= 0 && k < S.ac_cnt[l]) { const HeapEnt &e = S.ac[S.ac_off[l] + k]; f = e.f; g = e.g; n = e.node; }
    else { HeapEnt e = spill[i]; f = e.f; g = e.g; n = e.node; }
  }
  __device__ __forceinline__ void cset(int i, int l, double f, double g, int n) const {
    if (i < hcap()) { hf()[i] = f; hg()[i] = g; hn()[i] = n; }
    else {
      HeapEnt e; e.f = f; e.g = g; e.node = n; e.pad = 0;
      spill[i] = e; /* write-through */
      const int k = i - S.ac_lo[l];
      if (l >= 1 && k >= 0 && k < S.ac_cnt[l]) S.ac[S.ac_off[l] + k] = e;
    }
    hot[n & 0x7fffffff].heap_pos = i;
  }
  /* sift_up_warp for a push at position pos covered by the cache: identical result, ancestors read from shared memory */
  __device__ __forceinline__ void sift_up_warp_cached(int pos, double f, double g, int n, int lane) const {
    int p1 = pos + 1;
    int depth = 31 - __clz(p1);
    int my = (p1 >> (lane + 1)) - 1;
    bool have = lane < depth;
    double af = 0.0, ag = 0.0; int an = 0;
    if (have) cget(my, lane + 1, af, ag, an);
    bool moves = have && heap_worse(af, ag, f, g);
    unsigned stopm = __ballot_sync(0xffffffffu, !moves);
    int stop = __ffs(stopm) - 1;
    if (lane < stop) cset((p1 >> lane) - 1, lane, af, ag, an);
    if (lane == 0) cset((p1 >> stop) - 1, stop, f, g, n);
    __syncwarp();
  }
  /* ---- |U| > 32: R new heap entries (S.q_f/q_g/q_n, control order) pushed at positions n0 .. n0 + R - 1, same result as R
   * sequential pushes, most of them done in parallel.
   * Positions whose (pos + 1) >> G agree form a block: they share their ancestors from distance G upwards, and the
   * ancestors at distances 1 .. G of a block are ancestors of no other block ("private").  A push that comes to rest after
   * examining only private ancestors (it moves up fewer than G levels) commutes with every push of another block, so one
   * lane per block runs its block's pushes one after another while the other lanes do the same for theirs (pass 1).  A push
   * that would have to look beyond distance G, and everything after it in its block, is deferred; pass 2 executes the
   * deferred pushes in control order with the warp-cooperative sift-up.  Measured on the |U| = 125 workload 58 % of the
   * pushes do not move at all and 6 % move 3 levels or more. */
  __device__ __forceinline__ void push_batch_blocks(int n0, int R, int lane) const {
    constexpr int G = 3;
    const int b0 = (n0 + 1) >> G;
    const int bid = b0 + lane;
    int r_lo = (bid << G) - (n0 + 1), r_hi = ((bid + 1) << G) - (n0 + 1);
    if (r_lo < 0) r_lo = 0;
    if (r_hi > R) r_hi = R;
    int defer_from = r_hi;
    for (int r = r_lo; r < r_hi; r++) {
      const int p1 = n0 + r + 1;
      const double f = S.q_f[r], g = S.q_g[r];
      const int n = S.q_n[r];
      double af[G], ag[G];
      int an[G];
      int s = 0;
      bool beyond = false;
#pragma unroll
      for (int d = 1; d <= G; d++) { /* examine the ancestors at distances 1 .. G while they are strictly worse */
        if (s == d - 1 && !beyond) {
          cget((p1 >> d) - 1, d, af[d - 1], ag[d - 1], an[d - 1]);
          if (heap_worse(af[d - 1], ag[d - 1], f, g)) { s = d; if (d == G) beyond = true; }
        }
      }
      if (beyond) { defer_from = r; break; } /* it would have to examine distance G + 1: nothing was written yet */
#pragma unroll
      for (int d = 1; d <= G; d++) /* ancestors 1 .. s move down one level each */
        if (d <= s) cset((p1 >> (d - 1)) - 1, d - 1, af[d - 1], ag[d - 1], an[d - 1]);
      cset((p1 >> s) - 1, s, f, g, n);
    }
    S.q_defer[lane] = defer_from;
    __syncwarp();
    for (int r = 0; r < R; r++) { /* pass 2: the deferred pushes, in control order */
      const int k = ((n0 + r + 1) >> G) - b0;
      if (r >= S.q_defer[k]) sift_up_warp_cached(n0 + r, S.q_f[r], S.q_g[r], S.q_n[r], lane);
    }
    __syncwarp();
  }

  /* pop by one full warp: the levels inside shared memory are walked as before; below them every round fetches the
   * 4-level subtree under the current position (30 entries, one per lane, ONE round trip) and walks it with shuffles.
   * Same comparisons in the same order as sift_down => same heap. */
  __device__ __forceinline__ void sift_down_warp(int n_heap, double f, double g, int n, int lane) const {
    int pos = 0;
    const int hc = hcap();
    bool done = false;
    while (true) { /* shared-memory levels */
      const int c = 2 * pos + 1;
      if (c >= n_heap) { done = true; break; }
      if (c + 1 >= hc) break;
      double cf = hf()[c], cg = hg()[c]; int cn = hn()[c]; int cc = c;
      if (c + 1 < n_heap) {
        const double rf = hf()[c + 1], rg = hg()[c + 1];
        if (heap_worse(cf, cg, rf, rg)) { cc = c + 1; cf = rf; cg = rg; cn = hn()[c + 1]; }
      }
      if (!heap_worse(cf, cg, f, g)) { if (lane == 0) set(pos, cf, cg, cn); pos = cc; }
      else { done = true; break; }
    }
    while (!done) {
      const long long p1 = (long long)pos + 1;
      const int L = 1 + (lane >= 2) + (lane >= 6) + (lane >= 14);
      const long long q = (p1 << L) - 1 + (lane - ((1 << L) - 2));
      const bool valid = lane < 30 && q < (long long)n_heap;
      double ef = 0.0, eg = 0.0; int en = 0;
      if (valid) get((int)q, ef, eg, en);
      int j = 0;
#pragma unroll
      for (int lv = 1; lv <= 4; lv++) {
        const int rl = (1 << lv) - 2 + 2 * j; /* lane holding the left child */
        double cf = __shfl_sync(0xffffffffu, ef, rl), cg = __shfl_sync(0xffffffffu, eg, rl);
        int cn = __shfl_sync(0xffffffffu, en, rl);
        const bool cv = __shfl_sync(0xffffffffu, (int)valid, rl) != 0;
        const double rf = __shfl_sync(0xffffffffu, ef, rl + 1), rg = __shfl_sync(0xffffffffu, eg, rl + 1);
        const int rn = __shfl_sync(0xffffffffu, en, rl + 1);
        const bool rv = __shfl_sync(0xffffffffu, (int)valid, rl + 1) != 0;
        if (!cv) { done = true; break; }
        int right = 0;
        if (rv && heap_worse(cf, cg, rf, rg)) { right = 1; cf = rf; cg = rg; cn = rn; }
        if (!heap_worse(cf, cg, f, g)) { if (lane == 0) set(pos, cf, cg, cn); pos = 2 * pos + 1 + right; j = 2 * j + right; }
        else { done = true; break; }
      }
    }
    if (lane == 0) set(pos, f, g, n);
    __syncwarp();
  }

  /* pop: sift the former last element down from the root; ties still move down (boost siftdown) */
  __device__ __forceinline__ void sift_down(int n_heap, int pos, double f, double g, int n) const {
    while (true) {
      int c = 2 * pos + 1;
      if (c >= n_heap) break;
      double cf, cg; int cn;
      get(c, cf, cg, cn);
      if (c + 1 < n_heap) {
        double rf, rg; int rn;
        get(c + 1, rf, rg, rn);
        if (heap_worse(cf, cg, rf, rg)) { c = c + 1; cf = rf; cg = rg; cn = rn; } /* right child only if strictly better */
      }
      if (!heap_worse(cf, cg, f, g)) { set(pos, cf, cg, cn); pos = c; }
      else break;
    }
    set(pos, f, g, n);
  }
};

/* Arena data (table slots, node records, state rows) is touched once or twice per pop: load it with .cg so that it
 * does not evict the occupancy bricks, which are the only global data with reuse, from L1. */
__device__ __forceinline__ Slot load_slot_cg(const Slot *p) {
  const int4 *q = reinterpret_cast<const int4 *>(p);
  int4 a = __ldcg(q), b = __ldcg(q + 1);
  Slot s;
  s.k0 = ((unsigned long long)(unsigned)a.y << 32) | (unsigned)a.x;
  s.k1lo = (unsigned)a.z; s.node1 = (unsigned)a.w;
  s.g = __hiloint2double(b.y, b.x); s.pg = __hiloint2double(b.w, b.z);
  return s;
}
__device__ __forceinline__ NodeHot load_hot_cg(const NodeHot *p) {
  const int4 *q = reinterpret_cast<const int4 *>(p);
  int4 a = __ldcg(q), b = __ldcg(q + 1);
  NodeHot h;
  h.g = __hiloint2double(a.y, a.x); h.h = __hiloint2double(a.w, a.z); h.pg = __hiloint2double(b.y, b.x);
  h.heap_pos = b.z; h.action = (short)(b.w & 0xffff); h.flags = (unsigned char)((b.w >> 16) & 0xff); h.pad0 = 0;
  return h;
}

/* ---------------------------------------------------------------- hash table */
__device__ __forceinline__ unsigned table_hash(unsigned long long k0, unsigned long long k1) {
  unsigned long long h = (k0 ^ (k1 * 0x9E3779B97F4A7C15ull)) * 0xD6E8FEB86659FD93ull;
  return (unsigned)(h >> 32) ^ (unsigned)h;
}

__device__ __forceinline__ bool slot_matches(const Slot &s, unsigned long long k0, unsigned long long k1, bool wide,
                                             const unsigned char *rows, size_t row_bytes) {
  if (s.k0 != k0 || s.k1lo != (unsigned int)k1) return false;
  if (!wide) return true;
  const RowHdr *h = reinterpret_cast<const RowHdr *>(rows + (size_t)(s.node1 - 1) * row_bytes);
  return h->k1 == k1;
}

/* serial probe from slot i: returns node id or -1; *end_slot = matching slot / first empty slot */
__device__ __forceinline__ int table_find_from(const Slot *table, int tsize, unsigned i, unsigned long long k0,
                                               unsigned long long k1, bool wide, const unsigned char *rows, size_t row_bytes,
                                               int *end_slot, double *g, double *pg) {
  unsigned mask = (unsigned)tsize - 1u;
  i &= mask;
  while (true) {
    Slot s = table[i];
    if (s.node1 == 0u) { *end_slot = (int)i; return -1; }
    if (slot_matches(s, k0, k1, wide, rows, row_bytes)) { *end_slot = (int)i; *g = s.g; *pg = s.pg; return (int)s.node1 - 1; }
    i = (i + 1) & mask;
  }
}

/* rebuild insert (table growth): returns the slot index */
__device__ __forceinline__ int table_insert_atomic(Slot *table, int tsize, unsigned long long k0, unsigned long long k1, int id,
                                                   double g, double pg) {
  unsigned mask = (unsigned)tsize - 1u;
  unsigned i = table_hash(k0, k1) & mask;
  unsigned long long w1 = ((unsigned long long)(unsigned)(id + 1) << 32) | (unsigned long long)(unsigned int)k1;
  unsigned long long *t = reinterpret_cast<unsigned long long *>(table);
  while (atomicCAS(&t[4 * i + 1], 0ull, w1) != 0ull) i = (i + 1) & mask; /* claim by the (k1lo,node1) word */
  t[4 * i] = k0;
  table[i].g = g;
  table[i].pg = pg;
  return (int)i;
}

/* ---------------------------------------------------------------- exact reference arithmetic with cheap filters */
/* Cold exact paths are kept out of line on purpose: the per-pop instruction footprint has to stay well inside the
 * 32 KB L1.5 instruction cache (a first version with everything inlined touched 36 KB per pop and ran several
 * times slower, every line missing). */
__device__ __noinline__ int lattice_int_exact(double x, double q) { return round_int(ddiv(x, q)); }
__device__ __noinline__ int sample_divisor_exact(double mvT, double res) { return __double2int_rz(ceil(ddiv(mvT, res))); }
__device__ __noinline__ double div_exact(double a, double b) { return ddiv(a, b); }

/* lattice int round(x / q) (wp:97-120) with q = 0.01 or 0.1: x*(1/q) decides unless within 1e-6 of a tie. */
__device__ __forceinline__ int lattice_int(double x, double q, double inv_q) {
  double y = dmul(x, inv_q);
  double ym = magic_add(y);
  if (fabs(dsub(y, magic_rint(ym))) < 0.499999 && fabs(y) < 1073741824.0) return magic_int(ym);
  return lattice_int_exact(x, q);
}

/* max(5, (int)ceil(max_v*T/res)) (em:95): the product with 1/res decides unless within 1e-9 of an integer. */
__device__ __forceinline__ int sample_divisor(double max_v, double T, double res, double inv_res) {
  double mvT = dmul(max_v, T);
  double x = dmul(mvT, inv_res);
  double xm = magic_add(x);
  double r = magic_rint(xm);
  int n;
  if (fabs(dsub(x, r)) > 1e-9 && x < 1073741824.0) n = magic_int(xm) + ((x > r) ? 1 : 0); /* ceil(x) */
  else n = sample_divisor_exact(mvT, res);
  return n < 5 ? 5 : n;
}

/* ---------------------------------------------------------------- yaw controls (Control::*xYAW) */
using mplb_ref::heading_dot; /* v.normalized() . (cos yaw, sin yaw), shared with the LPA* core */
/* Lattice ints of a full state row: polynomial part (wp:95-112) and, with yaw controls, round(yaw / 0.1) (wp:114-117);
 * the yaw slot of a non-yaw plan packs as 0. */
template <int DIM, int ORD, int NS>
__device__ __forceinline__ void lattice_ints_x(const DevCfg &c, const double *st, int *ints) {
  lattice_ints<DIM, ORD>(st, ints);
  if (NS > DIM * ORD) ints[DIM * ORD] = c.use_yaw ? round_int(ddiv(st[DIM * ORD], 0.1)) : 0;
}
/* The reference's (int)std::round(x / q) of every key field of a state row is defined: the rounded quotient fits int32. */
template <int DIM, int ORD, int NS>
__device__ __forceinline__ bool lattice_ints_defined(const DevCfg &c, const double *st) {
  bool ok = true;
  for (int f = 0; f < NS; f++) {
    if (f == DIM * ORD && !c.use_yaw) break;
    const double r = mplb_ref::round_haz(ddiv(st[f], f < DIM ? 0.01 : 0.1));
    ok = ok && r >= -2147483648.0 && r <= 2147483647.0;
  }
  return ok;
}
/* The state row of a waypoint (wp:22-58): the polynomial part, then the yaw slot of the cost-shaping / yaw kernels. */
template <int DIM, int ORD, int NS>
__device__ __forceinline__ void waypoint_state(const DevCfg &c, const mplb_waypoint &w, double *s) {
  for (int ax = 0; ax < DIM; ax++) {
    s[ax] = w.pos[ax];
    if (ORD >= 2) s[DIM + ax] = w.vel[ax];
    if (ORD >= 3) s[2 * DIM + ax] = w.acc[ax];
    if (ORD >= 4) s[3 * DIM + ax] = w.jrk[ax];
  }
  if (NS > DIM * ORD) s[DIM * ORD] = c.use_yaw ? w.yaw : 0.0;
}

/* ---------------------------------------------------------------- phase B1: one lane per control (em:155-160,163-165) */
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ void expand_b1(const DevCfg &c, const SM &S, EBT &E, int i) {
  constexpr int NP = DIM * ORD;
  constexpr int NS = EBT::NS;
  const double T = c.dt;
  double es[NS];
  double max_v = 0.0;
  bool dyn_ok = true, same_pos = true;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
    Axis<ORD> A(&E.st[ax], DIM, S.U[i * 3 + ax], S.Ut[i * 3 + ax]);
    es[0 * DIM + ax] = A.p(T);
    if (ORD >= 2) es[1 * DIM + ax] = A.v(T);
    if (ORD >= 3) es[2 * DIM + ax] = A.a(T);
    if (ORD >= 4) es[3 * DIM + ax] = A.j(T);
    double mv = A.max_vel(T);
    if (mv > max_v) max_v = mv; /* em:91-94 */
    /* validate_primitive pr:449-475: only derivatives below the control order, bound <= 0 disables (pr:485) */
    if (ORD >= 2 && c.v_max > 0.0 && mv > c.v_max) dyn_ok = false;
    if (ORD >= 3 && c.a_max > 0.0 && A.max_acc(T) > c.a_max) dyn_ok = false;
    if (ORD >= 4 && c.j_max > 0.0 && A.max_jrk(T) > c.j_max) dyn_ok = false;
    same_pos = same_pos && (E.st[ax] == es[ax]); /* em:163 */
  }
  int ints[NS];
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
#pragma unroll
    for (int d = 0; d < ORD; d++)
      ints[ax * ORD + d] = (d == 0) ? lattice_int(es[ax], 0.01, 100.0) : lattice_int(es[d * DIM + ax], 0.1, 10.0);
  }
  if (NS > NP) { /* yaw slot: pr_yaw_ = Primitive1D(p.yaw, u(Dim)) (pr:36,242-253), evaluated and normalised at t = T (pr:328) */
    double yaw1 = 0.0;
    int yi = 0;
    if (c.use_yaw) {
      yaw1 = normalize_angle(dadd(dmul(S.Uyaw[i], T), E.st[NP]));
      yi = lattice_int(yaw1, 0.1, 10.0);
      if (c.yaw_max > 0.0) { /* validate_yaw (pr:503-525): heading inside the semi-FOV at both ends */
        const double v0x = (ORD >= 2) ? E.st[DIM + 0] : S.U[i * 3 + 0], v0y = (ORD >= 2) ? E.st[DIM + 1] : S.U[i * 3 + 1];
        const double v1x = (ORD >= 2) ? es[DIM + 0] : S.U[i * 3 + 0], v1y = (ORD >= 2) ? es[DIM + 1] : S.U[i * 3 + 1];
        if ((v0x != 0.0 || v0y != 0.0) && heading_dot(v0x, v0y, E.cy0, E.sy0) < c.cos_yaw_max) dyn_ok = false;
        if (v1x != 0.0 || v1y != 0.0) {
          double sn, cs;
          trig::sincos_cr(yaw1, &sn, &cs);
          if (heading_dot(v1x, v1y, cs, sn) < c.cos_yaw_max) dyn_ok = false;
        }
      }
    }
    es[NP] = yaw1;
    ints[NP] = yi;
  }
#pragma unroll
  for (int f = 0; f < NS; f++) E.es[i * NS + f] = es[f];
  unsigned long long k0, k1;
  bool key_ok = pack_key_nohash<DIM, ORD, NS>(c, ints, k0, k1);
  /* tn == curr (em:158, wp:132-135): equal lattice tuples <=> equal packed keys (the packing is injective inside the
   * key range; a tuple outside it is reported through key_bad before it can matter) */
  const bool self = key_ok && (k0 == E.pk0) && (k1 == E.pk1);
  E.k0[i] = k0; E.k1[i] = k1;
  E.first[i] = 0x7fffffff;
  int verdict, n = 0, cnt = 0;
  if (self) verdict = 0;
  else if (!dyn_ok) verdict = 1;
  else if (same_pos) verdict = 4;
  else {
    verdict = 5;
    n = sample_divisor(max_v, T, c.res, c.inv_res);
    cnt = (n < MPLB_NCAP && c.use_fast) ? S.tcnt_s[n] : c.tcnt[n];
  }
  E.nsamp[i] = n;
  E.cnt[i] = cnt;
  if ((verdict >= 3) && !key_ok) E.key_bad = 1;
  E.verdict[i] = verdict;
  E.nid[i] = -1;
}

/* Filtered sampling (see filtered_w), per launch: the top polynomial coefficient u / ORD! of control i, in cells. */
template <int DIM, int ORD, class SM>
__device__ __forceinline__ void filter_top(const DevCfg &c, SM &S, int i) {
  const double fact = (ORD == 1) ? 1.0 : (ORD == 2) ? 2.0 : (ORD == 3) ? 6.0 : 24.0;
  for (int ax = 0; ax < 3; ax++) S.Au[i * 3 + ax] = (ax < DIM) ? c.U[i * 3 + ax] / fact * c.inv_res : 0.0;
}

/* Filtered sampling, per pop: the sampling base of the node in E.st on axis ax (parent cell coordinate and lower
 * polynomial coefficients, in cells). */
template <int DIM, int ORD, class EBT>
__device__ __forceinline__ void filter_base(const DevCfg &c, EBT &E, int ax) {
  E.y0[ax] = dmul(dsub(E.st[ax], c.origin[ax]), c.inv_res);
  if (ORD >= 2) E.Ap[0 * 3 + ax] = dmul(E.st[DIM + ax], c.inv_res);
  if (ORD >= 3) E.Ap[1 * 3 + ax] = dmul(dmul(E.st[2 * DIM + ax], 0.5), c.inv_res);
  if (ORD >= 4) E.Ap[2 * 3 + ax] = dmul(div_exact(E.st[3 * DIM + ax], 6.0), c.inv_res);
}

/* B1 for all controls of one node by ONE warp, plus the flat sample list (granules) and the sampling base.
 * E.st / E.pk0 / E.pk1 must hold the node's state and packed lattice key.
 * Granule q of a control holds its samples 8q .. 8q + 7.  SM::WAVE_MAJOR: the list holds granule 0 of every sampled
 * control, then granule 1 of every control that has one, and so on, so that the sampler reaches a control's later
 * granules after its earlier ones have had the chance to find a blocked sample.  Otherwise: all granules of control 0,
 * then all of control 1, ... (E.gbase[i] is the first granule of control i). */
template <int DIM, int ORD, int NB, class SM, class EBT>
__device__ MPLB_B1_INLINE void b1_warp(const DevCfg &c, const SM &S, EBT &E, int lane, bool fast) {
  if (lane == 0) E.key_bad = 0;
  if (EBT::NS > DIM * ORD && lane == 31 && c.use_yaw && c.yaw_max > 0.0)
    trig::sincos_cr(normalize_angle(E.st[DIM * ORD]), &E.sy0, &E.cy0); /* evaluate(0) normalises the yaw too (pr:328) */
  if (fast && lane < DIM) filter_base<DIM, ORD>(c, E, lane);
  __syncwarp();
  int gbase = 0;
  int ng[NB];
#pragma unroll
  for (int b = 0; b < NB; b++) {
    const int i = b * 32 + lane;
    ng[b] = 0;
    if (i < c.nU) {
      expand_b1<DIM, ORD>(c, S, E, i);
      if (fast && E.verdict[i] == 5) ng[b] = (E.cnt[i] + 7) >> 3;
    }
    if (SM::WAVE_MAJOR) continue;
    int incl = ng[b]; /* warp scan of the granule counts */
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
    int excl = gbase + incl - ng[b];
    if (i < c.nU) { E.gbase[i] = excl; if ((c.pot || c.use_yaw) && E.nsamp[i] > 0) E.dts[i] = ddiv(c.dt, (double)E.nsamp[i]); }
    for (int q = 0; q < ng[b]; q++) {
      E.gl[excl + q] = (unsigned)i | ((unsigned)(q * 8) << 8) | ((unsigned)E.cnt[i] << 16);
      E.gl_t[excl + q] = (unsigned short)(S.toff_s[E.nsamp[i]] + q * 8);
    }
    gbase += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (SM::WAVE_MAJOR) {
    int ngmax = 0;
#pragma unroll
    for (int b = 0; b < NB; b++) ngmax = max(ngmax, ng[b]);
    ngmax = __reduce_max_sync(0xffffffffu, ngmax);
    const unsigned lt = (1u << lane) - 1u;
    for (int q = 0; q < ngmax; q++) {
#pragma unroll
      for (int b = 0; b < NB; b++) {
        const int i = b * 32 + lane;
        const unsigned m = __ballot_sync(0xffffffffu, ng[b] > q);
        if (ng[b] > q) {
          const int g = gbase + __popc(m & lt);
          E.gl[g] = (unsigned)i | ((unsigned)(q * 8) << 8) | ((unsigned)E.cnt[i] << 16);
          E.gl_t[g] = (unsigned short)(S.toff_s[E.nsamp[i]] + q * 8);
        }
        gbase += __popc(m);
      }
    }
  }
  if (lane == 0) E.n_gran = gbase;
  __syncwarp();
}

/* One collision sample, exact (em:100-104,119): true when the sample at time t of control i is outside or occupied. */
template <int DIM, int ORD, class SM>
__device__ __noinline__ bool sample_blocked_exact(const DevCfg &c, const SM &S, const double *st, int i, double t, int *cell_idx) {
#ifdef MPLB_PHASE_TIMING
  atomicAdd(const_cast<unsigned long long *>(&S.dbg[4]), 1ull);
#endif
  int pn[3] = {0, 0, 0};
  bool outside = false;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
    Axis<ORD> A(&st[ax], DIM, S.U[i * 3 + ax], S.Ut[i * 3 + ax]);
    pn[ax] = float_to_cell(A.p(t), c.origin[ax], c.res);
    outside = outside || pn[ax] < 0 || pn[ax] >= c.nd[ax];
  }
  if (outside) { if (cell_idx) *cell_idx = -1; return true; }
  if (cell_idx) *cell_idx = (DIM == 2) ? pn[0] + c.nd[0] * pn[1] : pn[0] + c.nd[0] * pn[1] + c.nd[0] * c.nd[1] * pn[2];
  return brick_occupied<DIM>(c, pn[0], pn[1], pn[2]);
}

/* Filtered cell coordinate of one axis.  The cell coordinate minus one half, w = (p(t) - origin)/res - 0.5, is evaluated
 * as one FP64 Horner chain in cells (parent coordinate y0 and lower coefficients per pop, filter_base; top coefficient
 * per control, filter_top; FMA allowed because the value is only used to decide a rounding).  Its distance from the real
 * value is < 2^-45 * M, M = the host's magnitude bound (build_cfg).  When w is farther than c.fast_delta from a rounding
 * tie (clear_of_tie), round(w) equals the reference's round((p - origin)/res - 0.5) (mu:103-108): c.fast_delta also
 * covers the reference's own rounding of that expression, see build_cfg.  Otherwise the caller evaluates the exact
 * formula. */
template <int ORD, class SM, class EBT>
__device__ __forceinline__ double filtered_w(const SM &S, const EBT &E, int i, int ax, double t) {
  double dy = S.Au[i * 3 + ax];
#pragma unroll
  for (int d = ORD - 2; d >= 0; d--) dy = __fma_rn(dy, t, E.Ap[d * 3 + ax]);
  return __dsub_rn(__fma_rn(dy, t, E.y0[ax]), 0.5);
}
/* wm = magic_add(w): true when round(w) = magic_int(wm) is decided by the filter */
__device__ __forceinline__ bool clear_of_tie(const DevCfg &c, double w, double wm) {
  return fabs(__dsub_rn(w, magic_rint(wm))) < 0.5 - c.fast_delta;
}

/* Filtered sample: the filtered cell on every axis, then the occupancy bit.  *sure is cleared when an axis is too close
 * to a tie (the return value is then meaningless and the caller evaluates sample_blocked_exact). */
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ bool sample_blocked_filtered(const DevCfg &c, const SM &S, const EBT &E, int i, double t, bool *sure) {
  int pn[3] = {0, 0, 0};
  bool ok = true, outside = false;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
    double w = filtered_w<ORD>(S, E, i, ax, t);
    double wm = magic_add(w);
    ok = ok && clear_of_tie(c, w, wm);
    pn[ax] = magic_int(wm);
    outside = outside || pn[ax] < 0 || pn[ax] >= c.nd[ax];
  }
  *sure = ok;
  if (outside || !ok) return outside;
  return brick_occupied<DIM>(c, pn[0], pn[1], pn[2]);
}

/* B2, per-control exact form: warps take controls round-robin, lanes take samples (trace kernel, and the search
 * kernel when the fast tables do not fit). */
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ void expand_b2_percontrol(const DevCfg &c, const SM &S, EBT &E, int warp, int lane, int nwarps) {
  for (int i = warp; i < c.nU; i += nwarps) {
    if (E.verdict[i] != 5) continue;
    int n = E.nsamp[i];
    int cnt = E.cnt[i];
    const double *tt = c.ttab + c.toff[n];
    int first = 0x7fffffff;
    for (int base = 0; base < cnt; base += 32) {
      int k = base + lane;
      bool blocked = false;
      if (k < cnt) blocked = sample_blocked_exact<DIM, ORD>(c, S, E.st, i, __ldg(&tt[k]), nullptr);
      unsigned m = __ballot_sync(0xffffffffu, blocked);
      if (m) { first = base + __ffs(m) - 1; break; }
    }
    if (lane == 0) E.first[i] = first;
  }
}

/* em:25-45 for a state (tolerances, then ray trace mu:117-134); executed by one full warp. */
template <int DIM, int ORD, class SM>
__device__ __noinline__ bool goal_test_warp(const DevCfg &c, const SM &S, const double *st, int lane) {
  double m = 0.0;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) m = fmax(m, fabs(dsub(st[ax], S.goal_pos[ax])));
  bool goaled = m <= c.tol_pos;
  if (goaled && c.tol_vel >= 0.0) {
    m = 0.0;
#pragma unroll
    for (int ax = 0; ax < DIM; ax++) m = fmax(m, fabs(dsub((ORD >= 2) ? st[DIM + ax] : 0.0, S.goal_vel[ax])));
    goaled = m <= c.tol_vel;
  }
  if (goaled && c.tol_acc >= 0.0) {
    m = 0.0;
#pragma unroll
    for (int ax = 0; ax < DIM; ax++) m = fmax(m, fabs(dsub((ORD >= 3) ? st[2 * DIM + ax] : 0.0, S.goal_acc[ax])));
    goaled = m <= c.tol_acc;
  }
  if (!goaled) return false;
  /* rayTrace(state.pos, goal.pos): the points of mplb_ref.h's ray_setup / ray_point, lanes take consecutive points */
  double diff[3] = {0, 0, 0}, s;
  const int max_diff = ray_setup(DIM, c.res, st, S.goal_pos, diff, &s);
  bool hit = false;
  for (int base = 1; base < max_diff; base += 32) {
    int n = base + lane;
    bool outside = false, occ = false;
    if (n < max_diff) {
      int pn[3] = {0, 0, 0};
#pragma unroll
      for (int ax = 0; ax < DIM; ax++) {
        pn[ax] = float_to_cell(ray_point(st[ax], diff[ax], s, n), c.origin[ax], c.res);
        outside = outside || pn[ax] < 0 || pn[ax] >= c.nd[ax];
      }
      if (!outside) occ = brick_occupied<DIM>(c, pn[0], pn[1], pn[2]);
    }
    unsigned mo = __ballot_sync(0xffffffffu, outside);
    unsigned mh = __ballot_sync(0xffffffffu, occ);
    if (mo) { /* break at the first outside cell: only hits before it count */
      unsigned before = (1u << (__ffs(mo) - 1)) - 1u;
      hit = (mh & before) != 0u;
      break;
    }
    if (mh) { hit = true; break; }
  }
  return !hit;
}

/* eb:46-64 (heur_ignore_dynamics_ = true).  With a prior trajectory (eb:49-51) the target is the prior's waypoint at the
 * state's own time, plus the prior's remaining cost: row `depth` of c.prior holds both (the state's time is a function of
 * its depth alone, see RowHdr::depth; rows exist while size_t(t / dt) < prior_traj_.size()). */
template <int DIM, int ORD, class SM>
__device__ __forceinline__ double heuristic(const DevCfg &c, const SM &S, const double *st, unsigned long long k0,
                                            unsigned long long k1, int depth) {
  if (c.eps == 0.0) return 0.0; /* gs:53,87 */
  if (S.goal_key_ok && k0 == S.gk0 && k1 == S.gk1) return 0.0;
  const bool pr = c.prior_n > 0 && depth < c.prior_n;
  const double *P = pr ? c.prior + 4 * depth : S.goal_pos;
  double m = 0.0;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) m = fmax(m, fabs(dsub(st[ax], pr ? __ldg(&P[ax]) : P[ax])));
  double h;
  if (c.v_max > 0.0) h = (c.vmax_rcp_exact != 0.0) ? dmul(dmul(c.w, m), c.vmax_rcp_exact) : div_exact(dmul(c.w, m), c.v_max);
  else h = dmul(c.w, m);
  return pr ? dadd(h, __ldg(&P[3])) : h;
}

/* unpack the lattice ints of a node from its packed key */
template <int NS>
__device__ __forceinline__ void unpack_ints(const DevCfg &c, unsigned long long k0, unsigned long long k1, int *ints) {
#pragma unroll
  for (int f = 0; f < NS; f++) {
    unsigned long long wv = c.kword[f] ? k1 : k0;
    unsigned long long v = (wv >> c.kshift[f]) & ((1ull << c.kbits[f]) - 1ull);
    ints[f] = (int)((long long)v + (long long)c.koff[f]);
  }
}

template <int NS>
__device__ __forceinline__ unsigned long long khash_of_ints(const int *ints, int nkey) {
  unsigned long long h = khash_init();
#pragma unroll
  for (int f = 0; f < NS; f++)
    if (f < nkey) h = khash_step(h, ints[f]); /* the yaw slot of a non-yaw plan is not part of the key (wp:114) */
  return khash_final(h);
}

/* Start set-up (tid 0) of a start in S.cur whose lattice tuple lies outside the packable range: a derivative above its
 * bound or an unwrapped yaw.  The reference plans from such a start.  Its tuple equals no successor's (validated
 * successors lie inside the range), so it is pushed under the reserved key MPLB_KEY_OUT_OF_RANGE; otherwise as the
 * kernel pushes an in-range start.  The pop loop hashes the lattice ints it unpacks from the current node's packed key;
 * the hash seeds set here cancel what it unpacks from the reserved key and add the start's true tuple instead:
 * (h ^ kh_true ^ kh_reserved) ^ kh_reserved = h ^ kh_true, and likewise for the sum.  A start whose (int)std::round of
 * a field is undefined in the reference (the rounded quotient leaves int32) ends the plan with MPLB_PLAN_KEY_RANGE.
 * Out of line: a cold path that must leave the search kernel's register allocation alone. */
template <int DIM, int ORD, class SM>
__device__ __noinline__ void start_out_of_range(const DevCfg &c, const BatchArgs &a, SM &S, int pid, NodeHot *hot, Slot *table,
                                                unsigned char *rows, int *poplog) {
  constexpr int NS = SM::NS;
  if (!lattice_ints_defined<DIM, ORD, NS>(c, S.cur)) { S.status = MPLB_PLAN_KEY_RANGE; return; }
  const int nk = (NS > DIM * ORD) ? c.nkey : NS;
  int ints[NS], ur[NS];
  lattice_ints_x<DIM, ORD, NS>(c, S.cur, ints);
  const unsigned long long k = MPLB_KEY_OUT_OF_RANGE;
  unpack_ints<NS>(c, k, k, ur);
  const unsigned long long kh_true = khash_of_ints<NS>(ints, nk), kh_reserved = khash_of_ints<NS>(ur, nk);
  /* eb:46-64: h = 0 on the goal's tuple, which only a comparison of the tuples shows here (a goal with this tuple is
   * outside the range too); otherwise the heuristic gets a key that differs from the goal's */
  const mplb_waypoint &gl = c.prior_on ? c.prior_goal : a.goals[pid];
  bool at_goal = gl.control == c.control && gl.enable_t == 0;
  if (at_goal) {
    double gs[NS];
    int gi[NS];
    waypoint_state<DIM, ORD, NS>(c, gl, gs);
    lattice_ints_x<DIM, ORD, NS>(c, gs, gi);
    for (int f = 0; f < nk; f++) at_goal = at_goal && gi[f] == ints[f];
  }
  NodeHot n0;
  n0.g = 0.0; n0.h = at_goal ? 0.0 : heuristic<DIM, ORD>(c, S, S.cur, ~S.gk0, S.gk1, 0); n0.pg = 0.0; n0.heap_pos = 0;
  n0.action = -1; n0.flags = 3; n0.pad0 = 0;
  hot[0] = n0;
  int slot = table_insert_atomic(table, S.tsize, k, k, 0, 0.0, 0.0);
  RowHdr *rh = reinterpret_cast<RowHdr *>(rows);
  rh->k0 = k; rh->k1 = k; rh->parent = -1; rh->slot = slot; rh->pred_head = -1; rh->depth = 0;
  double *rs = reinterpret_cast<double *>(rows + sizeof(RowHdr));
  for (int f = 0; f < NS; f++) rs[f] = S.cur[f];
  S.n_nodes = 1; S.n_heap = 0;
  S.cur_node = 0; S.cur_g = 0.0; S.cur_tag = 0;
  S.cur_k0 = k; S.cur_k1 = k;
  S.pop_hash = 0xCBF29CE484222325ull ^ kh_true ^ kh_reserved;
  S.closed_hash = kh_true - kh_reserved;
  if (a.want_poplog) poplog[0] = 0;
  S.pops = 1;
}

/* Generic serial relaxation of successors [i0, i1) in control order (lane 0 of warp 0): re-probes the table in
 * global memory, so it is correct under every hazard (duplicate siblings, slot collisions).  gs:79-143. */
template <int DIM, int ORD, class SM>
__device__ __noinline__ void relax_serial(const DevCfg &c, SM &S, typename SM::EB &E, HeapEnt *spill, Slot *table, NodeHot *hot,
                                          unsigned char *rows, int i0, int i1, bool wide, PredRec *plog) {
  const HeapView<SM> H{S, spill, hot}; /* built here: a view whose address escapes would turn heap accesses generic */
  constexpr int NS = SM::NS;
  constexpr size_t ROWB = (sizeof(RowHdr) + NS * sizeof(double) + 15) & ~(size_t)15; /* 16-byte aligned rows */
  const double kInf = __longlong_as_double(0x7ff0000000000000ll);
  const int cn = S.cur_node;
  const double cg = S.cur_g;
  for (int idx = i0; idx < i1; idx++) {
    int v = E.verdict[idx];
    if (v == 5) v = (E.first[idx] == 0x7fffffff) ? 3 : 2;
    if (v < 3) continue;
    const unsigned long long k0 = E.k0[idx], k1 = E.k1[idx];
    int slot; double gold = kInf, pgold = 0.0;
    int nid = table_find_from(table, S.tsize, table_hash(k0, k1), k0, k1, wide, rows, ROWB, &slot, &gold, &pgold);
    NodeHot hn;
    if (nid < 0) { /* gs:84-88 */
      nid = S.n_nodes++;
      hn.g = kInf; hn.h = heuristic<DIM, ORD>(c, S, &E.es[idx * NS], k0, k1, S.cur_depth + 1); hn.pg = 0.0; hn.heap_pos = -1; hn.action = -1;
      hn.flags = 0; hn.pad0 = 0;
      RowHdr *rh = reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB);
      rh->k0 = k0; rh->k1 = k1; rh->parent = -1; rh->slot = slot; rh->pred_head = -1; rh->depth = S.cur_depth + 1;
      double *rs = reinterpret_cast<double *>(rows + (size_t)nid * ROWB + sizeof(RowHdr));
      for (int f = 0; f < NS; f++) rs[f] = E.es[idx * NS + f];
      Slot sl; sl.k0 = k0; sl.k1lo = (unsigned int)k1; sl.node1 = (unsigned)(nid + 1); sl.g = kInf; sl.pg = 0.0;
      table[slot] = sl;
    } else hn = hot[nid];
    E.nid[idx] = nid;
    S.p_slot[idx] = slot; /* later batches of this pop test their empty slots against it */
    double ecost = S.cost[idx];
    if ((c.pot || c.use_yaw) && v == 3) { /* cost shaping (em:114-115,121-127); only the POT instantiations can have these set */
      double acc = 0.0;
      const int base_t = E.gbase[idx] * 8, cn_t = E.cnt[idx];
      if constexpr (SM::DYN_TERMS) {
        const double2 *T = shaped_terms(S);
        for (int q = 0; q < cn_t; q++) { acc = dadd(acc, T[base_t + q].x); acc = dadd(acc, T[base_t + q].y); }
      } else
      for (int q = 0; q < cn_t; q++) { acc = dadd(acc, S.terms[base_t + q]); acc = dadd(acc, S.yterms[base_t + q]); }
      ecost = dadd(acc, S.cost[idx]);
    }
    if (plog) { /* gs:100-102: every finite-cost edge is recorded, improving or not */
      RowHdr *rh = reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB);
      PredRec r; r.cost = ecost; r.pred = cn; r.next = rh->pred_head; r.action = idx; r.pad = 0;
      const int e = S.n_log++;
      plog[e] = r;
      rh->pred_head = e;
    }
    double tentative = dadd(cg, ecost); /* gs:107 */
    if (tentative < hn.g) { /* gs:109-141 */
      double f = dadd(tentative, dmul(c.eps, hn.h));
      hn.g = tentative; hn.pg = cg; hn.action = (short)idx;
      reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB)->parent = cn;
      table[slot].g = tentative; table[slot].pg = cg;
      int fl = hn.flags;
      if ((fl & 1) && !(fl & 2)) { /* increase(): f lowered, sift up only (gs:131-133) */
        hot[nid] = hn;
        H.sift_up(hn.heap_pos, f, tentative, nid);
      } else {
        int tag = nid;
        if (fl & 2) { /* closed node re-pushed (gs:135-141): refresh g copies of its stale entries */
          for (int q = 0; q < S.n_heap; q++) if ((H.node_at(q) & 0x7fffffff) == nid) H.set_g(q, tentative);
          tag = nid | 0x80000000;
        }
        hn.flags = (unsigned char)(fl | 1);
        hot[nid] = hn;
        H.sift_up(S.n_heap, f, tentative, tag);
        S.n_heap++;
      }
    } else if (tentative == hn.g && cg > hn.pg) { /* recoverTraj tie: larger predecessor g wins (gs:398-403) */
      hn.pg = cg; hn.action = (short)idx;
      hot[nid] = hn;
      table[slot].pg = cg;
      reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB)->parent = cn;
    }
  }
}

/* B2, flat form, plain kernels: thread `t` of `nthreads` sampling threads takes sample (t & 7) of granule
 * (t >> 3) + j * (nthreads / 8) of the wave-major list.  (Handing the granules to octets through a shared counter instead
 * measured no faster than not skipping at all.)
 * A sample whose index k is >= E.first[u] at the time the thread reaches it is skipped and issues no brick load.  This is
 * exact: E.first[u] only ever holds the index of a sample that was evaluated and found blocked, so a skipped sample has a
 * larger index than some blocked sample and cannot be the first one.  Every value E.first[u] takes is >= the first blocked
 * index k*, so k* is skipped only once E.first[u] == k*, i.e. once it is recorded.  The final atomicMin value is the true
 * first blocked index, and first == INT_MAX still means that no sample is blocked (nothing is skipped then). */
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ void sample_granules(const DevCfg &c, const SM &S, EBT &E, int t, int nthreads) {
  const int sub = t & 7;
  const volatile int *first = E.first; /* lowered by the other octets while this one works */
  for (int g = t >> 3; g < E.n_gran; g += nthreads >> 3) {
    const unsigned info = E.gl[g];
    const int u = (int)(info & 0xffu);
    const int k = (int)((info >> 8) & 0xffu) + sub;
    if (k >= (int)(info >> 16) || k >= first[u]) continue;
#ifdef MPLB_PHASE_TIMING
    if (sub == 0) atomicAdd(const_cast<unsigned long long *>(&S.dbg[2]), 1ull); /* granules evaluated */
#endif
    const double ts = S.tts[(int)E.gl_t[g] + sub];
    bool sure = true;
    bool blk = sample_blocked_filtered<DIM, ORD>(c, S, E, u, ts, &sure);
    if (!sure) blk = sample_blocked_exact<DIM, ORD>(c, S, E.st, u, ts, nullptr);
    if (blk) atomicMin(&E.first[u], k);
  }
}

/* ---------------------------------------------------------------- cost shaping (em:104-128): search region + potential map
 * Separate code path, compiled only into the POT instantiations so that the plain-map kernel keeps its size. */
template <int DIM, int ORD, class SM>
__device__ __noinline__ bool cell_exact(const DevCfg &c, const SM &S, const double *st, int i, double t, int *pn) {
  bool outside = false;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
    Axis<ORD> A(&st[ax], DIM, S.U[i * 3 + ax], S.Ut[i * 3 + ax]);
    pn[ax] = float_to_cell(A.p(t), c.origin[ax], c.res);
    outside = outside || pn[ax] < 0 || pn[ax] >= c.nd[ax];
  }
  return outside;
}
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ bool cell_filtered(const DevCfg &c, const SM &S, const EBT &E, int i, double t, int *pn, bool *sure) {
  bool ok = true, outside = false;
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
    double w = filtered_w<ORD>(S, E, i, ax, t);
    double wm = magic_add(w);
    ok = ok && clear_of_tie(c, w, wm);
    pn[ax] = magic_int(wm);
    outside = outside || pn[ax] < 0 || pn[ax] >= c.nd[ax];
  }
  *sure = ok;
  return outside;
}
/* One sample with cost shaping: returns blocked (em:104-106,116-120) and the cost term of em:114-115 (0 when none). */
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ bool sample_shaped(const DevCfg &c, const SM &S, const EBT &E, int i, double t, double *term,
                                              double *yterm) {
  int pn[3] = {0, 0, 0};
  bool sure;
  bool outside = cell_filtered<DIM, ORD>(c, S, E, i, t, pn, &sure);
  if (!sure) outside = cell_exact<DIM, ORD>(c, S, E.st, i, t, pn);
  *term = 0.0;
  *yterm = 0.0;
  if (outside) return true;
  const size_t idx = (DIM == 2) ? (size_t)pn[0] + (size_t)c.nd[0] * pn[1]
                                : (size_t)pn[0] + (size_t)c.nd[0] * pn[1] + (size_t)c.nd[0] * c.nd[1] * pn[2];
  if (c.region && !((c.region[idx >> 5] >> (idx & 31)) & 1u)) return true; /* not in the search region */
  if (c.pot) {
    const int p = (int)c.pot[idx];
    if (p >= 100) return true;
    if (p > 0) {
      double vn = 0.0;
      if (c.grad_w != 0.0) { /* pt.vel.norm() = sqrt of the left-to-right sum of squares */
        double ss = 0.0;
#pragma unroll
        for (int ax = 0; ax < DIM; ax++) {
          Axis<ORD> A(&E.st[ax], DIM, S.U[i * 3 + ax], S.Ut[i * 3 + ax]);
          double v = A.v(t);
          ss = (ax == 0) ? dmul(v, v) : dadd(ss, dmul(v, v));
        }
        vn = sqrt(ss);
      }
      *term = dmul(E.dts[i], dadd(dmul(c.pot_w, (double)p), dmul(c.grad_w, vn)));
    }
  } else if (brick_occupied<DIM>(c, pn[0], pn[1], pn[2])) return true;
  if (c.use_yaw && c.wyaw > 0.0) { /* em:121-128: (1 - heading . velocity direction) * wyaw * dt_s */
    Axis<ORD> Ax(&E.st[0], DIM, S.U[i * 3 + 0], S.Ut[i * 3 + 0]);
    Axis<ORD> Ay(&E.st[1], DIM, S.U[i * 3 + 1], S.Ut[i * 3 + 1]);
    const double vx = Ax.v(t), vy = Ay.v(t);
    const double nrm = sqrt(dadd(dmul(vx, vx), dmul(vy, vy)));
    if (nrm > 1e-5) {
      double sn, cs;
      trig::sincos_cr(normalize_angle(dadd(dmul(S.Uyaw[i], t), E.st[DIM * ORD])), &sn, &cs);
      const double v_value = dsub(1.0, heading_dot(vx, vy, cs, sn));
      *yterm = dmul(dmul(c.wyaw, v_value), E.dts[i]);
    }
  }
  return false;
}
template <int DIM, int ORD, class SM, class EBT>
__device__ __forceinline__ void sample_granules_shaped(const DevCfg &c, SM &S, EBT &E, int t, int nthreads) {
  const int gstep = nthreads >> 3;
  const int sub = t & 7;
  for (int g = t >> 3; g < E.n_gran; g += gstep) {
    const unsigned info = E.gl[g];
    const int u = (int)(info & 0xffu);
    const int k = (int)((info >> 8) & 0xffu) + sub;
    if (k < (int)(info >> 16)) {
      double term, yterm;
      const bool blk = sample_shaped<DIM, ORD>(c, S, E, u, S.tts[(int)E.gl_t[g] + sub], &term, &yterm);
      if constexpr (SM::DYN_TERMS) shaped_terms(S)[g * 8 + sub] = make_double2(term, yterm);
      else { S.terms[g * 8 + sub] = term; S.yterms[g * 8 + sub] = yterm; }
      if (blk) atomicMin(&E.first[u], k);
    }
  }
}

/* ---------------------------------------------------------------- the kernel */
template <int DIM, int ORD, int NB, bool POT>
__global__ void __launch_bounds__(MPLB_NT, (NB == 1 && !POT) ? MPLB_MIN_CTAS : 2) /* the other instantiations are shared-memory bound at 2 per SM */
astar_batch_kernel(const __grid_constant__ DevCfg c, const __grid_constant__ BatchArgs a) {
  constexpr int NP = DIM * ORD;
  constexpr int NS = NP + (POT ? 1 : 0); /* cost-shaping / yaw instantiations carry a yaw slot after the polynomial state */
  constexpr int NW = MPLB_NT / 32;
  using SM = PlanSmem<DIM, ORD, NB, POT>;
  constexpr size_t ROWB = (sizeof(RowHdr) + NS * sizeof(double) + 15) & ~(size_t)15; /* 16-byte aligned rows */
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SM &S = *reinterpret_cast<SM *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const double kInf = __longlong_as_double(0x7ff0000000000000ll);
  const unsigned lt_mask = (1u << lane) - 1u;

  unsigned char *base = a.arena + (size_t)blockIdx.x * a.stride;
  NodeHot *hot = reinterpret_cast<NodeHot *>(base);
  unsigned char *rows = base + a.off_rows;
  HeapEnt *spill = reinterpret_cast<HeapEnt *>(base + a.off_heap);
  Slot *table = reinterpret_cast<Slot *>(base + a.off_table);
  int *poplog = reinterpret_cast<int *>(base + a.off_poplog);
  PredRec *plog = a.log_cap > 0 ? reinterpret_cast<PredRec *>(base + a.off_log) : nullptr; /* log mode: see PredRec */
  const bool wide = c.key_wide != 0;
  const bool fast = c.use_fast != 0;
  HeapView<SM> H{S, spill, hot};

  /* ---------------- per-launch constants */
  if (tid == 0) S.hcap = SM::DYN_HEAP ? a.hcap : SM::HCAP;
#ifdef MPLB_BULK_ROW
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((unsigned)__cvta_generic_to_shared(&S.pf_bar)) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    S.pf_phase = 0;
  }
#endif
  for (int i = tid; i < c.nU * 3; i += MPLB_NT) { S.U[i] = c.U[i]; S.Ut[i] = Axis<ORD>::top_of(c.U[i]); }
  if (POT) for (int i = tid; i < c.nU; i += MPLB_NT) S.Uyaw[i] = (c.use_yaw && c.Uyaw) ? c.Uyaw[i] : 0.0;
  for (int i = tid; i < c.nU; i += MPLB_NT) {
    double J = 0.0;
    for (int ax = 0; ax < DIM; ax++) { double u = c.U[i * 3 + ax]; J = dadd(J, dmul(dmul(u, u), c.dt)); } /* pr:92-122,403-407 */
    S.cost[i] = dadd(J, dmul(c.w, c.dt));                                                                /* eb:343-345 */
    filter_top<DIM, ORD>(c, S, i);
  }
  if (fast) {
    for (int i = tid; i < MPLB_NCAP; i += MPLB_NT) { S.toff_s[i] = (i <= c.n_hi) ? c.toff[i] : 0; S.tcnt_s[i] = (i <= c.n_hi) ? c.tcnt[i] : 0; }
    for (int i = tid; i < c.tt_total; i += MPLB_NT) S.tts[i] = c.ttab[i];
  }

  while (true) {
    __syncthreads();
    if (tid == 0) { S.plan_idx = atomicAdd(a.work_counter, 1); S.t_start = global_timer_ns(); }
    __syncthreads();
    const int w = S.plan_idx;
    if (w >= a.n_work) break;
    const int pid = a.work ? a.work[w] : w;
    if (a.slot_of_plan && tid == 0) a.slot_of_plan[pid] = blockIdx.x;

    /* ---------------- per-plan init (pb:275-306, gs:44-60) */
    {
      unsigned long long *t64 = reinterpret_cast<unsigned long long *>(table);
      for (int i = tid; i < 4 * MPLB_TINIT; i += MPLB_NT) t64[i] = 0ull;
    }
    if (tid == 0) {
      const mplb_waypoint &st = a.starts[pid];
      S.tsize = MPLB_TINIT; S.n_nodes = 0; S.n_heap = 0; S.pops = 0; S.n_closed = 0; S.status = -1;
      S.n_samples = 0; S.n_valid = 0; S.n_before = 0; S.sd_pending = 0; S.pf_node = -1;
      S.n_log = 0; S.cur_depth = 0; S.pf_depth = 0;
      S.cur_buf = 0;
      for (int q = 0; q < SM::NBUF; q++) { S.eb[q].ready = 0; S.eb[q].node = -1; S.eb[q].key_bad = 0; }
      S.pop_hash = 0ull; S.closed_hash = 0ull; S.goal_hit = 0;
      /* eb:295-298, em:224: with a prior trajectory installed the requested goal is ignored, the goal stays the prior's end */
      const mplb_waypoint &gq = a.goals[pid];
      const mplb_waypoint &gl = c.prior_on ? c.prior_goal : gq;
      for (int ax = 0; ax < 3; ax++) { S.goal_pos[ax] = gl.pos[ax]; S.goal_vel[ax] = gl.vel[ax]; S.goal_acc[ax] = gl.acc[ax]; }
      double s0[NS];
      waypoint_state<DIM, ORD, NS>(c, st, s0);
      for (int f = 0; f < NS; f++) S.cur[f] = s0[f];
      /* goal lattice key: comparable only when the goal carries the same control flags (wp:92-125) */
      S.goal_key_ok = 0;
      if (gl.control == c.control && gl.enable_t == 0) {
        double gs[NS];
        waypoint_state<DIM, ORD, NS>(c, gl, gs);
        int gi[NS];
        lattice_ints_x<DIM, ORD, NS>(c, gs, gi);
        S.goal_key_ok = pack_key_nohash<DIM, ORD, NS>(c, gi, S.gk0, S.gk1) ? 1 : 0;
      }
      if (st.control != c.control || st.enable_t != 0) S.status = MPLB_INTERNAL_BADCTRL;
      else {
        /* pb:283: ENV_->is_free(start.pos) -> mu:44,57-62 on the int8 grid */
        int pn[3] = {0, 0, 0};
        bool outside = false;
        for (int ax = 0; ax < DIM; ax++) {
          pn[ax] = float_to_cell(s0[ax], c.origin[ax], c.res);
          outside = outside || pn[ax] < 0 || pn[ax] >= c.nd[ax];
        }
        bool is_free = false;
        if (!outside) {
          size_t idx = (DIM == 2) ? (size_t)pn[0] + (size_t)c.nd[0] * pn[1]
                                  : (size_t)pn[0] + (size_t)c.nd[0] * pn[1] + (size_t)c.nd[0] * c.nd[1] * pn[2];
          int8_t v = c.grid[idx];
          is_free = v < 100 && v >= 0;
        }
        if (!is_free) S.status = MPLB_PLAN_START_NOT_FREE;
      }
    }
    __syncthreads();
    if (S.status < 0 && warp == 0) { /* gs:44: is_goal(start) */
      bool g0 = goal_test_warp<DIM, ORD>(c, S, S.cur, lane);
      if (lane == 0 && g0) S.status = MPLB_PLAN_START_IS_GOAL;
    }
    __syncthreads();
    if (S.status < 0 && tid == 0) { /* gs:47-60: the start node is pushed and is necessarily the first pop (gs:64-68) */
      int ints[NS];
      lattice_ints_x<DIM, ORD, NS>(c, S.cur, ints);
      unsigned long long k0, k1;
      if (!pack_key_nohash<DIM, ORD, NS>(c, ints, k0, k1)) start_out_of_range<DIM, ORD>(c, a, S, pid, hot, table, rows, poplog);
      else {
        NodeHot n0;
        n0.g = 0.0; n0.h = heuristic<DIM, ORD>(c, S, S.cur, k0, k1, 0); n0.pg = 0.0; n0.heap_pos = 0; n0.action = -1;
        n0.flags = 3; n0.pad0 = 0;
        hot[0] = n0;
        int slot = table_insert_atomic(table, S.tsize, k0, k1, 0, 0.0, 0.0);
        RowHdr *rh = reinterpret_cast<RowHdr *>(rows);
        rh->k0 = k0; rh->k1 = k1; rh->parent = -1; rh->slot = slot; rh->pred_head = -1; rh->depth = 0;
        double *rs = reinterpret_cast<double *>(rows + sizeof(RowHdr));
        for (int f = 0; f < NS; f++) rs[f] = S.cur[f];
        S.n_nodes = 1; S.n_heap = 0;
        S.cur_node = 0; S.cur_g = 0.0; S.cur_tag = 0;
        S.cur_k0 = k0; S.cur_k1 = k1;
        S.pop_hash = 0xCBF29CE484222325ull;
        if (a.want_poplog) poplog[0] = 0;
        S.pops = 1;
      }
    }
    __syncthreads();

#ifdef MPLB_PHASE_TIMING
    long long ph[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long long tlast = clock64();
    if (tid < 8) S.dbg[tid] = 0;
#endif
    /* ---------------- main loop (gs:63-162): S.cur* always holds the node popped last */
    while (S.status < 0) {
      MPLB_TICK(7);
      /* capacity: this expansion can add at most nU nodes / heap entries */
      if (S.n_nodes + c.nU > a.cap || S.n_heap + c.nU + 1 > a.cap || (plog && S.n_log + c.nU > a.log_cap)) {
        __syncthreads();
        if (tid == 0) S.status = MPLB_INTERNAL_OVERFLOW;
        __syncthreads();
        break;
      }
      if ((long long)(S.n_nodes + c.nU) * a.load_inv > S.tsize) { /* keep the load factor <= 1/load_inv: grow in place and re-insert every node */
        long long nt = S.tsize;
        while ((long long)(S.n_nodes + c.nU) * a.load_inv > nt) nt <<= 1;
        __syncthreads();
        if (nt > a.tsize_max) { if (tid == 0) S.status = MPLB_INTERNAL_OVERFLOW; __syncthreads(); break; }
        unsigned long long *t64 = reinterpret_cast<unsigned long long *>(table);
        for (size_t i = tid; i < 4 * (size_t)nt; i += MPLB_NT) t64[i] = 0ull;
        __syncthreads();
        for (int i = tid; i < S.n_nodes; i += MPLB_NT) {
          RowHdr *rh = reinterpret_cast<RowHdr *>(rows + (size_t)i * ROWB);
          rh->slot = table_insert_atomic(table, (int)nt, rh->k0, rh->k1, i, hot[i].g, hot[i].pg);
        }
        if (tid == 0) S.tsize = (int)nt;
        __syncthreads();
      }

      /* ================= P1/P2 ================= */
      const int cb = S.cur_buf; /* read once per iteration: the search warp flips it at the pop */
      typename SM::EB &E = S.eb[cb];
      const bool hit = (SM::NBUF > 1) && E.ready && (E.node == S.cur_node); /* B1 of this node was done one pop ahead */
      if (!hit) { /* ---- P1 on the critical path: the search warp runs B1 for the current node */
        if (warp == 0) {
          if (lane < NS) E.st[lane] = S.cur[lane];
          if (lane == 0) { E.pk0 = S.cur_k0; E.pk1 = S.cur_k1; }
          __syncwarp();
          b1_warp<DIM, ORD, NB>(c, S, E, lane, fast);
        }
        if (warp != NW - 1) asm volatile("bar.sync 1, %0;" ::"n"(MPLB_NT - 32) : "memory"); /* B1 outputs visible to the sampling warps */
        /* E.node / E.ready are deliberately left alone: every warp evaluates `hit` from them right after the loop-end
         * barrier, and a write here could reach a late warp before it has done so.  The record is rewritten by the
         * heap warp before it is consulted again (the next pop uses the other record). */
      }
      MPLB_TICK(0);
      if (warp == NW - 1) {
        /* ---- heap warp: finish the previous pop's sift-down, prefetch the new root's state row ... */
        if (SM::DYN_HEAP) { /* |U| > 32: the heap is deep and mostly in global memory -> cooperative sift-down */
          if (S.sd_pending) H.sift_down_warp(S.n_heap, S.sd_f, S.sd_g, S.sd_n, lane);
          __syncwarp();
        }
        if (lane == 0) {
          if (!SM::DYN_HEAP && S.sd_pending) H.sift_down(S.n_heap, 0, S.sd_f, S.sd_g, S.sd_n);
          S.sd_pending = 0;
          int pf = -1;
          if (S.n_heap > 0) {
            pf = H.hn()[0] & 0x7fffffff;
            const RowHdr *rh = reinterpret_cast<const RowHdr *>(rows + (size_t)pf * ROWB);
#ifdef MPLB_BULK_ROW
            /* A/B variant (slower, not the default): the whole state row (header + state, ROWB contiguous 16-byte aligned
             * bytes) arrives with ONE bulk asynchronous copy (TMA engine, cp.async.bulk) completing on an mbarrier, instead
             * of 3 + NS scalar loads. */
            {
              const unsigned bar = (unsigned)__cvta_generic_to_shared(&S.pf_bar);
              const unsigned dst = (unsigned)__cvta_generic_to_shared(S.pf_row);
              asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((unsigned)ROWB) : "memory");
              asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(rh),
                           "r"((unsigned)ROWB), "r"(bar)
                           : "memory");
              unsigned done = 0;
              while (!done)
                asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                             : "=r"(done) : "r"(bar), "r"(S.pf_phase) : "memory");
              S.pf_phase ^= 1u;
              const RowHdr *sh = reinterpret_cast<const RowHdr *>(S.pf_row);
              S.pf_k0 = sh->k0; S.pf_k1 = sh->k1; S.pf_depth = sh->depth;
              const double *ss = reinterpret_cast<const double *>(S.pf_row + sizeof(RowHdr));
#pragma unroll
              for (int f = 0; f < NS; f++) S.pf_st[f] = ss[f];
            }
#else
            S.pf_k0 = __ldcg(&rh->k0); S.pf_k1 = __ldcg(&rh->k1); S.pf_depth = __ldcg(&rh->depth);
            const double *rs = reinterpret_cast<const double *>(rows + (size_t)pf * ROWB + sizeof(RowHdr));
#pragma unroll
            for (int f = 0; f < NS; f++) S.pf_st[f] = __ldcg(&rs[f]);
#endif
          }
          S.pf_node = pf;
        }
        __syncwarp();
        asm volatile("bar.arrive 3, 64;" ::: "memory"); /* heap and prefetched row are ready for the search warp's P3 */
        /* ---- ... and run B1 for that node into the other expansion record while the others work on the current one */
        if (SM::NBUF > 1) {
          typename SM::EB &E2 = S.eb[(cb ^ 1) & (SM::NBUF - 1)];
          const int pf = S.pf_node;
          if (pf >= 0) {
            if (lane == 0) {
#pragma unroll
              for (int f = 0; f < NS; f++) E2.st[f] = S.pf_st[f];
              E2.pk0 = S.pf_k0; E2.pk1 = S.pf_k1;
            }
            __syncwarp();
            b1_warp<DIM, ORD, NB>(c, S, E2, lane, fast);
          }
          if (lane == 0) { E2.node = pf; E2.ready = (pf >= 0) ? 1 : 0; }
        }
      } else {
        if (NB > 1 || warp == 0) {
          /* issue the table probes — WIN consecutive 32-byte slots per candidate, one HBM round trip in all but a
           * few per cent of the cases at load factor <= 1/4 — and compute h while they fly.  |U| > 32: the 32-control
           * batches are dealt to the search and sampling warps (batch b -> warp b mod (NW - 1)), whose round trips then
           * overlap instead of following each other on the search warp; the sampling warps sample afterwards (sampling is
           * the short phase of this shape). */
          constexpr int WIN = (NB == 1) ? MPLB_WIN : 2;
#pragma unroll
          for (int b = 0; b < NB; b++) {
            if (NB > 1 && (b % (NW - 1)) != warp) continue;
            const int i = b * 32 + lane;
            const bool probing = (i < c.nU) && (E.verdict[i] >= 4);
            const unsigned long long k0 = probing ? E.k0[i] : 0ull, k1 = probing ? E.k1[i] : 0ull;
            const unsigned mask = (unsigned)S.tsize - 1u;
            const unsigned h0 = table_hash(k0, k1) & mask;
            Slot sw[WIN];
            if (probing) {
#pragma unroll
              for (int q = 0; q < WIN; q++) sw[q] = load_slot_cg(&table[(h0 + q) & mask]);
            }
            double hv = 0.0;
            if (probing) hv = heuristic<DIM, ORD>(c, S, &E.es[i * NS], k0, k1, S.cur_depth + 1);
            int nid = -1, slot = -1;
            double g = kInf, pg = 0.0;
            if (probing) {
              bool done = false;
#pragma unroll
              for (int q = 0; q < WIN; q++) {
                if (!done) {
                  if (sw[q].node1 == 0u) { slot = (int)((h0 + q) & mask); done = true; }
                  else if (slot_matches(sw[q], k0, k1, wide, rows, ROWB)) {
                    nid = (int)sw[q].node1 - 1; slot = (int)((h0 + q) & mask); g = sw[q].g; pg = sw[q].pg; done = true;
                  }
                }
              }
              if (!done) nid = table_find_from(table, S.tsize, h0 + WIN, k0, k1, wide, rows, ROWB, &slot, &g, &pg);
            }
            if (i < c.nU) { S.p_nid[i] = nid; S.p_slot[i] = slot; S.p_g[i] = g; S.p_pg[i] = pg; S.p_h[i] = hv; }
          }
          MPLB_TICK(1);
        }
        if (warp != 0) {
          if (warp == 1) { /* ---- goal test (gs:146) and parity hash of the current node (needed only in P3) */
            bool gh = goal_test_warp<DIM, ORD>(c, S, S.cur, lane);
            if (lane == 0) { /* parity hash of the lattice ints (off the serial chain) */
              int ints[NS];
              unpack_ints<NS>(c, S.cur_k0, S.cur_k1, ints);
              S.goal_hit = gh ? 1 : 0; S.cur_kh = khash_of_ints<NS>(ints, (NS > DIM * ORD) ? c.nkey : NS);
            }
          }
          /* ---- B2: all collision samples of all controls, flat over 8-sample granules (warps 1..NW-2) */
          if (POT) sample_granules_shaped<DIM, ORD>(c, S, E, tid - 32, MPLB_NT - 64); /* host guarantees the fast tables */
          else if (fast) sample_granules<DIM, ORD>(c, S, E, tid - 32, MPLB_NT - 64);
          else expand_b2_percontrol<DIM, ORD>(c, S, E, warp - 1, lane, NW - 2);
        }
        MPLB_TICK(2);
        asm volatile("bar.sync 2, %0;" ::"n"(MPLB_NT - 32) : "memory"); /* probes + collision outcomes visible to the search warp */
        MPLB_TICK(3);
      }

      /* ================= P3 (warp 0): relax (gs:79-143), terminate (gs:146-161), take the next node (gs:64-68) */
      if (warp == 0) {
        asm volatile("bar.sync 3, 64;" ::: "memory"); /* the heap warp has finished the sift-down and the root prefetch */
        const int cn = S.cur_node;
        const double cg = S.cur_g;
        if (lane == 0) { /* bookkeeping of the current pop */
          S.n_before = S.n_nodes;
          unsigned long long kh = S.cur_kh;
          S.pop_hash = (S.pop_hash ^ kh) * 0x100000001B3ull;
          if (!S.cur_tag) { S.n_closed++; S.closed_hash += kh; }
        }
        int ns_acc = 0, nv_acc = 0;
        if (SM::DYN_HEAP) { if (lane == 0) S.ac_valid = 0; __syncwarp(); }
#pragma unroll
        for (int b = 0; b < NB; b++) {
          const int i = b * 32 + lane;
          int v = (i < c.nU) ? E.verdict[i] : 0;
          if (v == 5) {
            int first = E.first[i];
            v = (first == 0x7fffffff) ? 3 : 2;
            ns_acc += (v == 3) ? E.cnt[i] : first + 1;
          }
          const bool valid = v >= 3;
          const int r_nid_b = (i < c.nU) ? S.p_nid[i] : -1;
          const int r_slot_b = (i < c.nU) ? S.p_slot[i] : -1;
          const double r_g_b = (i < c.nU) ? S.p_g[i] : kInf;
          const double r_pg_b = (i < c.nU) ? S.p_pg[i] : 0.0;
          const double r_h_b = (i < c.nU) ? S.p_h[i] : 0.0;
          const unsigned long long rk0_b = (i < c.nU) ? E.k0[i] : 0ull, rk1_b = (i < c.nU) ? E.k1[i] : 0ull;
          const unsigned vmask = __ballot_sync(0xffffffffu, valid);
          nv_acc += __popc(vmask);
          if (vmask == 0u) continue;
          const bool found = valid && r_nid_b >= 0;
          const bool isnew = valid && r_nid_b < 0;
          /* hazards: two successors -> one node or one table slot; later batches vs nodes created earlier in this pop */
          bool hazard = false;
#ifdef MPLB_PHASE_TIMING
          long long td0 = clock64();
#endif
          {
            unsigned newm = __ballot_sync(0xffffffffu, isnew);
            unsigned fndm = __ballot_sync(0xffffffffu, found);
            if (isnew) {
              unsigned m1 = __match_any_sync(newm, rk0_b ^ (rk1_b * 0x9E3779B97F4A7C15ull));
              unsigned m2 = __match_any_sync(newm, r_slot_b);
              hazard = (__popc(m1) > 1) || (__popc(m2) > 1);
            }
            if (found) { unsigned m3 = __match_any_sync(fndm, r_nid_b); hazard = hazard || (__popc(m3) > 1); }
            if (NB > 1 && b > 0) { /* the probes predate everything earlier batches of this pop did */
              if (found) /* an earlier batch may already have relaxed the same node */
                for (int q = 0; q < b * 32; q++) hazard = hazard || (E.nid[q] == r_nid_b);
              if (isnew) /* an earlier batch may have created this key, or taken this empty slot: both show as the same slot
                            (equal keys share the probe sequence, hence its first empty slot) */
                for (int q = 0; q < b * 32; q++) hazard = hazard || (E.nid[q] >= S.n_before && S.p_slot[q] == r_slot_b);
            }
            hazard = __any_sync(0xffffffffu, hazard) || (plog != nullptr); /* log mode relaxes serially: the records live there */
          }
#ifdef MPLB_PHASE_TIMING
          long long td1 = clock64();
          if (lane == 0) MPLB_COUNT(0, td1 - td0);
#endif
          if (hazard) {
            if (lane == 0) {
              MPLB_COUNT(3, 1);
              relax_serial<DIM, ORD>(c, S, E, spill, table, hot, rows, b * 32, min(c.nU, b * 32 + 32), wide, plog);
              if (SM::DYN_HEAP) S.ac_valid = 0; /* the serial routine moved heap entries behind the ancestor cache's back */
            }
            __syncwarp();
            continue;
          }
          double ecost = valid ? S.cost[i] : 0.0;
          if (POT && (c.pot || c.use_yaw) && v == 3 && valid) { /* em:114-115,121-127: accumulate the sample terms in sample order, then eb:343-345 */
            double acc = 0.0;
            const int base_t = E.gbase[i] * 8, cn_t = E.cnt[i];
            if constexpr (SM::DYN_TERMS) {
              const double2 *T = shaped_terms(S);
              for (int q = 0; q < cn_t; q++) { acc = dadd(acc, T[base_t + q].x); acc = dadd(acc, T[base_t + q].y); }
            } else
            for (int q = 0; q < cn_t; q++) { acc = dadd(acc, S.terms[base_t + q]); acc = dadd(acc, S.yterms[base_t + q]); }
            ecost = dadd(acc, S.cost[i]);
          }
          const double tentative = dadd(cg, ecost); /* gs:107 */
          const bool improve = found && tentative < r_g_b;
          const bool tie = found && tentative == r_g_b && cg > r_pg_b; /* recoverTraj tie rule (gs:398-403) */
          const unsigned newm = __ballot_sync(0xffffffffu, isnew);
          int nid = r_nid_b;
          if (isnew) nid = S.n_nodes + __popc(newm & lt_mask);
          const int n_new = __popc(newm);
          if (valid) E.nid[i] = nid;
          double hval = r_h_b;
          int fl = 0, hpos = -1;
          if (improve) { const NodeHot hn = load_hot_cg(&hot[nid]); hval = hn.h; fl = hn.flags; hpos = hn.heap_pos; } /* rare dependent load */
          const double f = dadd(tentative, dmul(c.eps, hval));
          /* lane-parallel stores */
          if (isnew) { /* gs:84-88: the node's coord is this (first) discoverer's state */
            RowHdr *rh = reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB);
            rh->k0 = rk0_b; rh->k1 = rk1_b; rh->parent = cn; rh->slot = r_slot_b; rh->pred_head = -1; rh->depth = S.cur_depth + 1;
            double *rs = reinterpret_cast<double *>(rows + (size_t)nid * ROWB + sizeof(RowHdr));
#pragma unroll
            for (int q = 0; q < NS; q++) rs[q] = E.es[i * NS + q];
            Slot sl; sl.k0 = rk0_b; sl.k1lo = (unsigned int)rk1_b; sl.node1 = (unsigned)(nid + 1); sl.g = tentative; sl.pg = cg;
            table[r_slot_b] = sl;
            NodeHot hn; hn.g = tentative; hn.h = hval; hn.pg = cg; hn.heap_pos = -1; hn.action = (short)i; hn.flags = 1; hn.pad0 = 0;
            hot[nid] = hn;
          } else if (improve) {
            NodeHot hn; hn.g = tentative; hn.h = hval; hn.pg = cg; hn.heap_pos = hpos; hn.action = (short)i;
            hn.flags = (unsigned char)(fl | 1); hn.pad0 = 0;
            hot[nid] = hn;
            table[r_slot_b].g = tentative; table[r_slot_b].pg = cg;
            reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB)->parent = cn;
          } else if (tie) {
            hot[nid].pg = cg; hot[nid].action = (short)i;
            table[r_slot_b].pg = cg;
            reinterpret_cast<RowHdr *>(rows + (size_t)nid * ROWB)->parent = cn;
          }
          if (lane == 0) S.n_nodes += n_new;
#ifdef MPLB_PHASE_TIMING
          if (lane == 0) MPLB_COUNT(1, clock64() - td1);
#endif
          MPLB_TICK(4);
          /* heap operations in control order (gs:129-141) */
          unsigned hm = __ballot_sync(0xffffffffu, isnew || improve);
          if (SM::DYN_HEAP && hm != 0u && hm == newm && S.n_heap >= H.hcap()) {
            /* deep heap and nothing but first-time pushes in this batch: block-parallel (see push_batch_blocks) */
            const int n0 = S.n_heap, R = __popc(hm);
            if (isnew) { const int r = __popc(newm & lt_mask); S.q_f[r] = f; S.q_g[r] = tentative; S.q_n[r] = nid; }
            __syncwarp();
            if (!S.ac_valid) H.cache_ancestors(n0, c.nU, lane);
            H.push_batch_blocks(n0, R, lane);
            if (lane == 0) S.n_heap = n0 + R;
            __syncwarp();
            hm = 0u;
          }
          while (hm) {
            const int j = __ffs(hm) - 1;
            hm &= hm - 1;
            const double jf = __shfl_sync(0xffffffffu, f, j), jg = __shfl_sync(0xffffffffu, tentative, j);
            const int jn = __shfl_sync(0xffffffffu, nid, j), jfl = __shfl_sync(0xffffffffu, fl, j);
            int jpos = __shfl_sync(0xffffffffu, hpos, j);
            const bool jnew = (newm >> j) & 1u;
            if (!jnew && (jfl & 1) && !(jfl & 2)) { /* increase(): f lowered, sift up only (gs:131-133) */
              if (jpos < 0 || jpos >= S.n_heap || (H.node_at(jpos) & 0x7fffffff) != jn) jpos = hot[jn].heap_pos; /* moved by an earlier sift of this pop */
              H.sift_up_warp(jpos, jf, jg, jn, lane);
              if (SM::DYN_HEAP) { if (lane == 0) S.ac_valid = 0; __syncwarp(); } /* arbitrary position: not through the cache */
            } else {
              int tag = jn;
              if (!jnew && (jfl & 2)) { /* closed node re-pushed (gs:135-141): refresh g copies of its stale entries */
                for (int q = lane; q < S.n_heap; q += 32) if ((H.node_at(q) & 0x7fffffff) == jn) H.set_g(q, jg);
                tag = jn | 0x80000000;
                __syncwarp();
                if (SM::DYN_HEAP) { if (lane == 0) S.ac_valid = 0; __syncwarp(); }
              }
              const int np = S.n_heap;
              __syncwarp();
              if (SM::DYN_HEAP && np >= H.hcap()) { /* deep heap: ancestors of this pop's pushes come from the shared-memory cache */
#ifdef MPLB_PHASE_TIMING
                long long tq0 = clock64();
#endif
                if (!S.ac_valid) H.cache_ancestors(np, c.nU, lane);
#ifdef MPLB_PHASE_TIMING
                long long tq1 = clock64();
#endif
                H.sift_up_warp_cached(np, jf, jg, tag, lane);
#ifdef MPLB_PHASE_TIMING
                if (lane == 0) { MPLB_COUNT(5, tq1 - tq0); MPLB_COUNT(6, clock64() - tq1); MPLB_COUNT(7, 1); }
#endif
              } else
              H.sift_up_warp(np, jf, jg, tag, lane);
              if (lane == 0) S.n_heap = np + 1;
              __syncwarp();
            }
          }
        }
        MPLB_TICK(5);
        /* ---- termination and the next pop */
        ns_acc = __reduce_add_sync(0xffffffffu, ns_acc);
        if (lane == 0) {
          S.n_samples += ns_acc;
          S.n_valid += nv_acc;
          int status = -1;
          if (E.key_bad) status = MPLB_PLAN_KEY_RANGE;
          else if (S.goal_hit) status = MPLB_PLAN_OK;
          else if (c.max_num > 0 && S.pops >= c.max_num) status = MPLB_PLAN_MAX_EXPAND;
          else if (S.n_heap == 0) status = MPLB_PLAN_QUEUE_EMPTY;
          if (status >= 0) S.status = status;
          else {
            const int tagged = H.hn()[0];
            const double topg = H.hg()[0];
            const int n = S.n_heap - 1;
            if (n > 0) { H.get(n, S.sd_f, S.sd_g, S.sd_n); S.sd_pending = 1; } /* sift-down deferred to the heap warp */
            S.n_heap = n;
            const int nx = tagged & 0x7fffffff;
            unsigned long long k0, k1;
            int ndepth;
            if (nx >= S.n_before) { /* created in this expansion: forward its state from shared memory */
              int j = 0;
              for (int q = 0; q < c.nU; q++) if (E.nid[q] == nx) { j = q; break; }
              k0 = E.k0[j]; k1 = E.k1[j];
              ndepth = S.cur_depth + 1;
#pragma unroll
              for (int f = 0; f < NS; f++) S.cur[f] = E.es[j * NS + f];
            } else if (nx == S.pf_node) {
              k0 = S.pf_k0; k1 = S.pf_k1;
              ndepth = S.pf_depth;
#pragma unroll
              for (int f = 0; f < NS; f++) S.cur[f] = S.pf_st[f];
            } else {
              const RowHdr *rh = reinterpret_cast<const RowHdr *>(rows + (size_t)nx * ROWB);
              k0 = rh->k0; k1 = rh->k1;
              ndepth = rh->depth;
              const double *rs = reinterpret_cast<const double *>(rows + (size_t)nx * ROWB + sizeof(RowHdr));
#pragma unroll
              for (int f = 0; f < NS; f++) S.cur[f] = rs[f];
            }
            S.cur_depth = ndepth;
            S.cur_k0 = k0; S.cur_k1 = k1;
            S.cur_node = nx;
            S.cur_g = topg;
            S.cur_tag = (tagged & 0x80000000) ? 1 : 0;
            hot[nx].flags = 3; /* iterationclosed = true (gs:68); a popped node is always opened */
            if (a.want_poplog && S.pops < a.cap) poplog[S.pops] = nx;
            S.pops++;
            if (SM::NBUF > 1) S.cur_buf = cb ^ 1; /* the next pop's expansion record is the one the heap warp filled */
          }
        }
        MPLB_TICK(6);
      }
      __syncthreads();
    }
#ifdef MPLB_PHASE_TIMING
    if (tid == 0 && a.phase_cycles) for (int k = 0; k < 8; k++) { a.phase_cycles[(size_t)pid * 16 + k] = ph[k]; a.phase_cycles[(size_t)pid * 16 + 8 + k] = (long long)S.dbg[k]; }
#endif

    /* ---------------- results + recoverTraj (gs:369-455) */
    if (tid == 0) {
      mplb_result r;
      r.status = S.status; r.n_seg = 0; r.cost = kInf;
      r.pops = S.pops; r.n_nodes = S.n_nodes; r.n_open = S.n_heap; r.n_closed = S.n_closed;
      r.n_prims = (long long)S.pops * c.nU; r.n_samples = S.n_samples; r.n_valid = S.n_valid;
      r.pop_hash = S.pop_hash; r.closed_hash = S.closed_hash;
      if (S.status == MPLB_PLAN_START_IS_GOAL) r.cost = 0.0;
      int *acts = a.actions ? a.actions + (size_t)pid * a.max_seg : nullptr;
      if (acts) for (int k = 0; k < a.max_seg; k++) acts[k] = -1;
      if (S.status == MPLB_PLAN_OK) {
        int n = 0, cnode = S.cur_node;
        bool ok = true;
        if (plog) {
          /* log mode, gs:386-437 verbatim: among the node's predecessor records take the smallest g_pred + cost with the
           * predecessors' FINAL g, ties -> larger g_pred, then the earliest record; the choice is written back into the
           * node (parent / action) so that the second pass below and the node getters read it. */
          while (true) {
            RowHdr *rh = reinterpret_cast<RowHdr *>(rows + (size_t)cnode * ROWB);
            int e = rh->pred_head, best = -1;
            double min_rhs = kInf, min_g = kInf;
            for (; e >= 0; e = plog[e].next) { /* newest -> oldest: on a full tie the older record replaces the newer one */
              const double gp = hot[plog[e].pred].g;
              const double rhs = dadd(gp, plog[e].cost);
              if (rhs < min_rhs || (rhs == min_rhs && gp >= min_g)) { min_rhs = rhs; min_g = gp; best = e; }
            }
            if (best < 0 || n > S.n_nodes) { ok = false; break; }
            rh->parent = plog[best].pred;
            hot[cnode].action = (short)plog[best].action;
            n++; cnode = plog[best].pred;
            if (cnode == 0) break; /* gs:433: reached the start key */
          }
        } else
        while (cnode != 0) {
          int p = reinterpret_cast<const RowHdr *>(rows + (size_t)cnode * ROWB)->parent;
          if (p < 0 || n > S.n_nodes) { ok = false; break; }
          n++; cnode = p;
        }
        if (!ok) r.status = MPLB_PLAN_TRACEBACK_FAILED;
        else {
          r.n_seg = n;
          r.cost = hot[S.cur_node].g; /* gs:179 */
          cnode = S.cur_node;
          for (int k = n - 1; k >= 0; k--) {
            int p = reinterpret_cast<const RowHdr *>(rows + (size_t)cnode * ROWB)->parent;
            if (k < a.max_seg) {
              if (acts) acts[k] = hot[cnode].action;
              if (a.seg_states) {
                double *row = a.seg_states + ((size_t)pid * a.max_seg + k) * 13;
                const double *ps = reinterpret_cast<const double *>(rows + (size_t)p * ROWB + sizeof(RowHdr));
                for (int q = 0; q < 13; q++) row[q] = 0.0;
                for (int d = 0; d < ORD; d++)
                  for (int ax = 0; ax < DIM; ax++) row[d * 3 + ax] = ps[d * DIM + ax];
                if (NS > NP && c.use_yaw) row[12] = ps[NP];
              }
            }
            cnode = p;
          }
        }
      }
      r.device_ms = (double)(global_timer_ns() - S.t_start) * 1e-6;
      a.results[pid] = r;
      if (r.status == MPLB_INTERNAL_OVERFLOW) a.overflow_list[atomicAdd(a.overflow_count, 1)] = pid;
    }
    if (a.want_poplog) { /* retained plan: expose the shared-memory part of the heap to the host getters */
      __syncthreads();
      if (tid == 0 && S.sd_pending) { H.sift_down(S.n_heap, 0, S.sd_f, S.sd_g, S.sd_n); S.sd_pending = 0; }
      __syncthreads();
      for (int i = tid; i < S.n_heap && i < H.hcap(); i += MPLB_NT) {
        HeapEnt e; e.f = H.hf()[i]; e.g = H.hg()[i]; e.node = H.hn()[i]; e.pad = 0;
        spill[i] = e;
      }
    }
  }
}

/* ---------------------------------------------------------------- get_succ for arbitrary states (parity artefact) */
template <int DIM, int ORD, int NB>
__global__ void __launch_bounds__(MPLB_NT) expand_trace_kernel(const __grid_constant__ DevCfg c, const mplb_waypoint *states, int n_states,
                                                               mplb_prim_trace *rows) {
  constexpr int NS = DIM * ORD;
  constexpr int NW = MPLB_NT / 32;
  using SM = PlanSmem<DIM, ORD, NB>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SM &S = *reinterpret_cast<SM *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < c.nU * 3; i += MPLB_NT) { S.U[i] = c.U[i]; S.Ut[i] = Axis<ORD>::top_of(c.U[i]); }
  for (int i = tid; i < c.nU; i += MPLB_NT) {
    double J = 0.0;
    for (int ax = 0; ax < DIM; ax++) { double u = c.U[i * 3 + ax]; J = dadd(J, dmul(dmul(u, u), c.dt)); }
    S.cost[i] = dadd(J, dmul(c.w, c.dt));
  }
  if (c.use_fast) for (int i = tid; i < MPLB_NCAP; i += MPLB_NT) S.tcnt_s[i] = (i <= c.n_hi) ? c.tcnt[i] : 0;
  typename SM::EB &E = S.eb[0];
  for (int s = blockIdx.x; s < n_states; s += gridDim.x) {
    __syncthreads();
    if (tid == 0) {
      const mplb_waypoint &st = states[s];
      for (int ax = 0; ax < DIM; ax++) {
        E.st[ax] = st.pos[ax];
        if (ORD >= 2) E.st[DIM + ax] = st.vel[ax];
        if (ORD >= 3) E.st[2 * DIM + ax] = st.acc[ax];
        if (ORD >= 4) E.st[3 * DIM + ax] = st.jrk[ax];
      }
      int ints0[NS];
      lattice_ints<DIM, ORD>(E.st, ints0);
      if (!pack_key_nohash<DIM, ORD>(c, ints0, E.pk0, E.pk1)) { E.pk0 = E.pk1 = MPLB_KEY_OUT_OF_RANGE; } /* out-of-range state: nothing is its self-loop */
      E.key_bad = 0;
    }
    __syncthreads();
    for (int i = tid; i < c.nU; i += MPLB_NT) expand_b1<DIM, ORD>(c, S, E, i);
    __syncthreads();
    expand_b2_percontrol<DIM, ORD>(c, S, E, warp, lane, NW);
    __syncthreads();
    for (int i = tid; i < c.nU; i += MPLB_NT) {
      mplb_prim_trace r;
      int v = E.verdict[i];
      if (v == 5) v = (E.first[i] == 0x7fffffff) ? 3 : 2;
      r.verdict = v;
      r.n = (v == 2 || v == 3) ? E.nsamp[i] : 0;
      r.n_tested = (v == 3) ? E.cnt[i] : (v == 2 ? E.first[i] + 1 : 0);
      r.block_idx = -1;
      if (v == 2) {
        int cell = -1;
        sample_blocked_exact<DIM, ORD>(c, S, E.st, i, c.ttab[c.toff[E.nsamp[i]] + E.first[i]], &cell);
        r.block_idx = cell;
      }
      r.cost = (v >= 3) ? S.cost[i] : (v == 2 ? __longlong_as_double(0x7ff0000000000000ll) : 0.0);
      for (int q = 0; q < 13; q++) r.succ[q] = 0.0;
      for (int ax = 0; ax < DIM; ax++) { /* tn carries every derivative (pr:321-331) */
        Axis<ORD> A(&E.st[ax], DIM, S.U[i * 3 + ax]);
        r.succ[ax] = A.p(c.dt); r.succ[3 + ax] = A.v(c.dt); r.succ[6 + ax] = A.a(c.dt); r.succ[9 + ax] = A.j(c.dt);
      }
      int ints[NS];
      lattice_ints<DIM, ORD>(&E.es[i * NS], ints);
      for (int q = 0; q < 16; q++) r.key[q] = 0;
      for (int f = 0; f < NS; f++) r.key[f] = ints[f];
      r.key[15] = NS;
      rows[(size_t)s * c.nU + i] = r;
    }
  }
}

/* ---------------------------------------------------------------- the filtered sampler on arbitrary states (parity artefact)
 * B1 as the search runs it, then, for every control whose primitive needs sampling (verdict 5), every sample time of its
 * divisor: the filtered cell (filtered_w, clear_of_tie, with the search's per-launch and per-pop set-up) next to the exact one
 * (cell_exact).  Rows are appended in no particular order through *count; only the first `cap` are stored. */
template <int DIM, int ORD, int NB>
__global__ void __launch_bounds__(MPLB_NT) probe_samples_kernel(const __grid_constant__ DevCfg c, const mplb_waypoint *states,
                                                                int n_states, mplb_sample_probe *rows, int cap, int *count) {
  constexpr int NW = MPLB_NT / 32;
  using SM = PlanSmem<DIM, ORD, NB>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SM &S = *reinterpret_cast<SM *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < c.nU * 3; i += MPLB_NT) { S.U[i] = c.U[i]; S.Ut[i] = Axis<ORD>::top_of(c.U[i]); }
  for (int i = tid; i < c.nU; i += MPLB_NT) filter_top<DIM, ORD>(c, S, i);
  if (c.use_fast) for (int i = tid; i < MPLB_NCAP; i += MPLB_NT) S.tcnt_s[i] = (i <= c.n_hi) ? c.tcnt[i] : 0;
  typename SM::EB &E = S.eb[0];
  for (int s = blockIdx.x; s < n_states; s += gridDim.x) {
    __syncthreads();
    if (tid == 0) {
      const mplb_waypoint &st = states[s];
      for (int ax = 0; ax < DIM; ax++) {
        E.st[ax] = st.pos[ax];
        if (ORD >= 2) E.st[DIM + ax] = st.vel[ax];
        if (ORD >= 3) E.st[2 * DIM + ax] = st.acc[ax];
        if (ORD >= 4) E.st[3 * DIM + ax] = st.jrk[ax];
      }
      int ints0[DIM * ORD];
      lattice_ints<DIM, ORD>(E.st, ints0);
      if (!pack_key_nohash<DIM, ORD>(c, ints0, E.pk0, E.pk1)) { E.pk0 = E.pk1 = MPLB_KEY_OUT_OF_RANGE; }
    }
    __syncthreads();
    for (int i = tid; i < c.nU; i += MPLB_NT) expand_b1<DIM, ORD>(c, S, E, i);
    if (tid < DIM) filter_base<DIM, ORD>(c, E, tid);
    __syncthreads();
    for (int i = warp; i < c.nU; i += NW) {
      if (E.verdict[i] != 5) continue;
      const double *tt = c.ttab + c.toff[E.nsamp[i]];
      for (int k = lane; k < E.cnt[i]; k += 32) {
        mplb_sample_probe r;
        r.state = s; r.control = i; r.k = k;
        r.t = tt[k];
        bool sure = true;
        int pe[3] = {0, 0, 0};
        cell_exact<DIM, ORD>(c, S, E.st, i, r.t, pe);
        for (int ax = 0; ax < 3; ax++) {
          r.w[ax] = 0.0; r.cell_fast[ax] = 0; r.cell_exact[ax] = pe[ax];
          if (ax < DIM) {
            const double w = filtered_w<ORD>(S, E, i, ax, r.t), wm = magic_add(w);
            sure = sure && clear_of_tie(c, w, wm);
            r.w[ax] = w;
            r.cell_fast[ax] = magic_int(wm);
          }
        }
        r.sure = sure ? 1 : 0;
        const int slot = atomicAdd(count, 1);
        if (slot < cap) rows[slot] = r;
      }
    }
  }
}

}  // namespace mplb
