/*
 * mplb_device.cuh — device-side arithmetic of the lattice planner (sm_90a).
 *
 * Every floating-point operation that the reference performs on the hot path is written here with
 * explicit round-to-nearest intrinsics (__dadd_rn / __dmul_rn / __ddiv_rn never contract to FMA), in the
 * reference's own left-to-right order, so that voxel indices, lattice keys and costs are bit-identical to
 * the CPU planner.  Terms the reference multiplies by a structurally-zero coefficient are dropped: adding an
 * exact zero changes at most the sign of a zero result, which no consumer (round, compare, abs) observes.
 *
 * Reference files (under motion_primitive_library/include/):
 *   primitive.h (pr)  waypoint.h (wp)  math.h (mt)  map_util.h (mu)  env_map.h (em)  env_base.h (eb)
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/mplb.h"
#include "mplb_ref.h"

namespace mplb {

#ifndef MPLB_NT
#define MPLB_NT 160   /* threads per CTA: one CTA owns one plan (warp 0 search, warps 1..NW-2 sampling, last warp heap) */
#endif
#define MPLB_MAXU 128 /* max |U| */
#ifndef MPLB_MIN_CTAS
#define MPLB_MIN_CTAS 6 /* resident CTAs per SM the plain |U| <= 32 search kernel is compiled for (64 registers per thread of the
                           64 K an SM has).  A sweep of threads x CTAs/SM on the 65 536-query bench list (256x3, 224x4, 192x5,
                           256x4, 160x6, 128x8) put 160x6 first: more, smaller plans per SM hide the per-pop latency chain better
                           than more sampling warps per plan once the batch is deep enough to keep every slot busy (a 1024-query
                           batch is tail bound and prefers 256x3). */
#endif

/* exact reference arithmetic shared with the rest of the library (mplb_ref.h) */
using mplb_ref::dadd;
using mplb_ref::dsub;
using mplb_ref::dmul;
using mplb_ref::ddiv;
using mplb_ref::round_int;
using mplb_ref::float_to_cell;
using mplb_ref::normalize_angle;
using mplb_ref::ray_setup;
using mplb_ref::ray_point;
using mplb_ref::khash_init;
using mplb_ref::khash_step;
using mplb_ref::khash_final;

/* Rounding without the XU pipe.  Every FP64 conversion / rounding instruction (F2I, I2F, FRND, MUFU.RCP64H)
 * issues to the low-rate XU pipe and has a long latency on the serial chain of a pop; adding and subtracting
 * 1.5 * 2^52 rounds to nearest-even on the FP64 pipe instead and leaves the integer in the low mantissa word.
 * Valid for |x| < 2^31; used only inside filters that defer to the exact formula near ties. */
#define MPLB_MAGIC 6755399441055744.0
__device__ __forceinline__ double magic_add(double x) { return __dadd_rn(x, MPLB_MAGIC); }
__device__ __forceinline__ double magic_rint(double xm) { return __dsub_rn(xm, MPLB_MAGIC); }
__device__ __forceinline__ int magic_int(double xm) { return __double2loint(xm); }

/* Device view of planner + map configuration (kernel parameter, by value). */
struct DevCfg {
  int dim, ord, control, nU, ns; /* ns = dim*ord doubles of state per node */
  int max_num;
  double dt, w, eps, v_max, a_max, j_max, tol_pos, tol_vel, tol_acc;
  /* map (mu:20-314) */
  int nd[3];
  int bd[3]; /* brick-grid dims */
  double origin[3];
  double res;
  const int8_t *grid;               /* int8 cells, x fastest (mu:33-41) */
  const unsigned long long *bricks; /* occupancy bit-bricks: 4x4x4 voxels (3D) or 8x8 cells (2D) per 64-bit word */
  /* control set and sample-time tables */
  const double *U;    /* nU rows of 3 */
  const double *ttab; /* accumulated sample times for every divisor n (em:98-99), concatenated */
  const int *toff;    /* offset of divisor n's row in ttab */
  const int *tcnt;    /* number of samples for divisor n (n or n+1) */
  int n_hi;           /* largest tabulated divisor */
  /* lattice-key packing: field f = axis*ord + derivative (wp:92-125 order) */
  int koff[13]; /* 12 polynomial fields + yaw (wp:114-117) */
  unsigned char kshift[13], kbits[13], kword[13];
  int key_wide; /* 1 when word 1 of the key needs more than 32 bits (table slots then also compare the row header) */
  /* filtered collision sampling (FP64 Horner in cell units with a guard band): see sample_blocked_filtered */
  double inv_res;   /* 1/res, used only inside filters whose doubtful cases fall back to the exact division */
  int use_fast;     /* tables fit in shared memory and every dynamic bound is known */
  int tt_total;     /* number of entries of ttab */
  double fast_delta; /* guard band around rounding ties of the filtered sampler, in cells */
  double vmax_rcp_exact; /* 1/v_max when v_max is a power of two (x / v_max == x * this, bit for bit), else 0 */
  /* cost shaping of env_map (em:104-118): optional potential map (int8 per cell) and search-region bitmask */
  const int8_t *pot;
  const unsigned int *region;
  double pot_w, grad_w;
  /* yaw controls (Control::*xYAW, pr:236-253): extra state double + key field, FOV check pr:503-525, cost em:121-128 */
  int use_yaw;          /* the control flag carries use_yaw: state rows hold yaw after the polynomial part */
  int nkey;             /* number of lattice-key fields = dim*ord + use_yaw */
  double yaw_max, wyaw; /* eb:388 (<= 0 disables the FOV check), eb:372 */
  double cos_yaw_max;   /* correctly rounded cos(yaw_max), prepared on the host */
  const double *Uyaw;   /* yaw rate of every control (column Dim of U), or null */
  /* prior trajectory (eb:46-53,249-256, em:187-225): row d = (pos of the prior at the time of a depth-d state, remaining
   * cost), d < prior_n; the prior's end point replaces every requested goal (em:224, eb:295-298) */
  const double *prior;
  int prior_n;  /* rows of the table (0 when even a depth-0 state falls behind the prior's end) */
  int prior_on; /* a prior trajectory is installed: prior_goal replaces the goals */
  mplb_waypoint prior_goal;
};

/* ------------------------------------------------------------------------------------------------
 * Polynomial primitive on one axis (pr:21-198), specialised per control order: the literal six-coefficient form is
 * mplb_ref.h's Prim1; this one drops its structurally-zero terms.  Coefficients c1..c5 (c0 is 0 for every control
 * constructor pr:35-52).  For control order ORD the leading non-zero coefficient is c[5-ORD] = u.
 *   ORD 1 (VEL): c4 = u, c5 = p          ORD 2 (ACC): c3 = u, c4 = v, c5 = p
 *   ORD 3 (JRK): c2 = u, c3 = a, ...     ORD 4 (SNP): c1 = u, c2 = j, ...
 * st[] holds (p, v, a, j) of the parent on this axis (only the first ORD entries are meaningful).      */
template <int ORD>
struct Axis {
  double c1, c2, c3, c4, c5;
  double top; /* leading coefficient divided by its factorial exactly as pr:128-131 does (u/2, u/6, u/24): per-control
                 constant, computed once per launch with a true division (x/2 is the exact scaling x*0.5) */
  __device__ __forceinline__ static double top_of(double u) {
    return (ORD == 1) ? u : (ORD == 2) ? __dmul_rn(u, 0.5) : (ORD == 3) ? __ddiv_rn(u, 6.0) : __ddiv_rn(u, 24.0);
  }
  __device__ __forceinline__ Axis(const double *st, int stride, double u, double top_) {
    c1 = c2 = c3 = c4 = 0.0;
    c5 = st[0];
    top = top_;
    if (ORD == 1) { c4 = u; }
    if (ORD == 2) { c3 = u; c4 = st[stride]; }
    if (ORD == 3) { c2 = u; c3 = st[2 * stride]; c4 = st[stride]; }
    if (ORD == 4) { c1 = u; c2 = st[3 * stride]; c3 = st[2 * stride]; c4 = st[stride]; }
  }
  __device__ __forceinline__ Axis(const double *st, int stride, double u) : Axis(st, stride, u, top_of(u)) {}
  /* pr:128-131   c0/120 t^5 + c1/24 t^4 + c2/6 t^3 + c3/2 t t + c4 t + c5 */
  __device__ __forceinline__ double p(double t) const {
    double s = 0.0;
    if (ORD >= 4) s = dmul(top, dmul(dmul(dmul(t, t), t), t));
    if (ORD >= 3) { double x = dmul((ORD == 3) ? top : ddiv(c2, 6.0), dmul(dmul(t, t), t)); s = (ORD >= 4) ? dadd(s, x) : x; }
    if (ORD >= 2) { double x = dmul(dmul((ORD == 2) ? top : dmul(c3, 0.5), t), t); s = (ORD >= 3) ? dadd(s, x) : x; }
    { double x = dmul(c4, t); s = (ORD >= 2) ? dadd(s, x) : x; }
    return dadd(s, c5);
  }
  /* pr:134-137   c0/24 t^4 + c1/6 t^3 + c2/2 t t + c3 t + c4 */
  __device__ __forceinline__ double v(double t) const {
    if (ORD == 1) return c4;
    double s = 0.0;
    if (ORD >= 4) s = dmul(ddiv(c1, 6.0), dmul(dmul(t, t), t));
    if (ORD >= 3) { double x = dmul(dmul(dmul(c2, 0.5), t), t); s = (ORD >= 4) ? dadd(s, x) : x; }
    { double x = dmul(c3, t); s = (ORD >= 3) ? dadd(s, x) : x; }
    return dadd(s, c4);
  }
  /* pr:140-142   c0/6 t^3 + c1/2 t t + c2 t + c3 */
  __device__ __forceinline__ double a(double t) const {
    if (ORD <= 2) return c3;
    double s = 0.0;
    if (ORD >= 4) s = dmul(dmul(dmul(c1, 0.5), t), t);
    { double x = dmul(c2, t); s = (ORD >= 4) ? dadd(s, x) : x; }
    return dadd(s, c3);
  }
  /* pr:145   c0/2 t t + c1 t + c2 */
  __device__ __forceinline__ double j(double t) const {
    if (ORD <= 3) return c2;
    return dadd(dmul(c1, t), c2);
  }
  /* pr:353-363 with extrema_v pr:152-162 -> solve(0, c0/6, c1/2, c2, c3) (mt:117-131) */
  __device__ __forceinline__ double max_vel(double T) const {
    double m = fmax(fabs(v(0.0)), fabs(v(T)));
    if (ORD == 3) {
      if (c2 != 0.0) { /* linear: -e/d */
        double r = ddiv(-c3, c2);
        if (r > 0.0 && r < T) { double x = fabs(v(r)); m = x > m ? x : m; }
      }
    }
    if (ORD == 4) {
      double qc = dmul(c1, 0.5);
      if (qc != 0.0) { /* quad(b=qc, c=c2, d=c3), mt:22-33 */
        double disc = dsub(dmul(c2, c2), dmul(dmul(4.0, qc), c3));
        if (!(disc < 0.0)) {
          double sq = sqrt(disc); /* IEEE correctly rounded */
          double den = dmul(2.0, qc);
          double r1 = ddiv(dsub(-c2, sq), den), r2 = ddiv(dadd(-c2, sq), den);
          bool stop = false; /* pr:155-160: roots visited in order, break at the first root >= T */
          if (r1 > 0.0 && r1 < T) { double x = fabs(v(r1)); m = x > m ? x : m; } else if (r1 >= T) stop = true;
          if (!stop && r2 > 0.0 && r2 < T) { double x = fabs(v(r2)); m = x > m ? x : m; }
        }
      } else if (c2 != 0.0) {
        double r = ddiv(-c3, c2);
        if (r > 0.0 && r < T) { double x = fabs(v(r)); m = x > m ? x : m; }
      }
    }
    return m;
  }
  /* pr:369-379 with extrema_a pr:169-179 -> solve(0, 0, c0/2, c1, c2) */
  __device__ __forceinline__ double max_acc(double T) const {
    double m = fmax(fabs(a(0.0)), fabs(a(T)));
    if (ORD == 4 && c1 != 0.0) {
      double r = ddiv(-c2, c1);
      if (r > 0.0 && r < T) { double x = fabs(a(r)); m = x > m ? x : m; }
    }
    return m;
  }
  /* pr:384-394: extrema_j needs c0 != 0 -> never */
  __device__ __forceinline__ double max_jrk(double T) const { return fmax(fabs(j(0.0)), fabs(j(T))); }
  /* pr:92-122 with the structurally-zero coefficients removed: J = u*u*T for every control order */
  __device__ __forceinline__ double J(double T) const {
    double u = (ORD == 1) ? c4 : (ORD == 2) ? c3 : (ORD == 3) ? c2 : c1;
    return dmul(dmul(u, u), T);
  }
};

/* Occupancy test of an inside cell through the bit-bricks (value == 100, mu:48). */
template <int DIM>
__device__ __forceinline__ bool brick_occupied(const DevCfg &c, int x, int y, int z) {
  if (DIM == 3) {
    size_t b = (size_t)(x >> 2) + (size_t)c.bd[0] * ((size_t)(y >> 2) + (size_t)c.bd[1] * (size_t)(z >> 2));
    unsigned bit = (x & 3) | ((y & 3) << 2) | ((z & 3) << 4);
    return (__ldg(&c.bricks[b]) >> bit) & 1ull;
  } else {
    size_t b = (size_t)(x >> 3) + (size_t)c.bd[0] * (size_t)(y >> 3);
    unsigned bit = (x & 7) | ((y & 7) << 3);
    return (__ldg(&c.bricks[b]) >> bit) & 1ull;
  }
}

/* Lattice ints of a state (wp:92-125): pos/0.01, derivatives/0.1, axis-major order. st[d*DIM + axis]. */
template <int DIM, int ORD>
__device__ __forceinline__ void lattice_ints(const double *st, int *ints) {
#pragma unroll
  for (int ax = 0; ax < DIM; ax++) {
#pragma unroll
    for (int d = 0; d < ORD; d++) {
      double x = st[d * DIM + ax];
      ints[ax * ORD + d] = round_int(ddiv(x, d == 0 ? 0.01 : 0.1));
    }
  }
}

/* Both words of the key of a state outside the packable range (an out-of-range start, a probed state).  No successor
 * that the search probes packs to it, because the all-ones value of a field decodes to at least the field's upper end
 * (koff + 2^kbits - 1 >= hi, build_cfg), and every such successor keeps one field below that end: its velocity, within
 * v_max by validation (pr:449-475; control order >= 2 needs v_max > 0), or, for VEL controls, its positions, within
 * 2 |u| dt of the map (a popped state has no valid successor unless its own position is inside the map, em:104). */
#define MPLB_KEY_OUT_OF_RANGE (~0ull)

/* Pack ints into the 128-bit node key (no parity hash); false when a field leaves its packable range. */
template <int DIM, int ORD, int NF = DIM * ORD>
__device__ __forceinline__ bool pack_key_nohash(const DevCfg &c, const int *ints, unsigned long long &k0, unsigned long long &k1) {
  k0 = 0; k1 = 0;
  bool ok = true;
#pragma unroll
  for (int f = 0; f < NF; f++) {
    long long v = (long long)ints[f] - (long long)c.koff[f];
    if (v < 0 || v >= (1ll << c.kbits[f])) ok = false;
    unsigned long long uv = (unsigned long long)v << c.kshift[f];
    if (c.kword[f]) k1 |= uv; else k0 |= uv;
  }
  return ok;
}

/* Pack ints into the 128-bit node key; returns false when a field leaves its packable range. */
template <int DIM, int ORD>
__device__ __forceinline__ bool pack_key(const DevCfg &c, const int *ints, unsigned long long &k0, unsigned long long &k1,
                                         unsigned long long &kh) {
  k0 = 0; k1 = 0;
  unsigned long long h = khash_init();
  bool ok = true;
#pragma unroll
  for (int f = 0; f < DIM * ORD; f++) {
    h = khash_step(h, ints[f]);
    long long v = (long long)ints[f] - (long long)c.koff[f];
    if (v < 0 || v >= (1ll << c.kbits[f])) ok = false;
    unsigned long long uv = (unsigned long long)v << c.kshift[f];
    if (c.kword[f]) k1 |= uv; else k0 |= uv;
  }
  kh = khash_final(h);
  return ok;
}

}  // namespace mplb
