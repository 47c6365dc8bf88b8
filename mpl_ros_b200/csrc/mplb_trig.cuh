/*
 * mplb_trig.cuh — correctly rounded sin/cos for the yaw branch (pr:503-525 validate_yaw, em:121-128 yaw cost).
 *
 * The reference calls libm cos()/sin(), whose last bit is unspecified (glibc 2.39 is one ulp off the correctly
 * rounded value on ~0.14 % of arguments; CUDA's libdevice on more).  The product defines the yaw branch with the
 * correctly rounded functions instead: double-double argument reduction by pi/2 (three-part constant) and a
 * double-double Taylor/Horner evaluation on |r| <= pi/4 up to r^31, accurate to ~2^-100, rounded once.  The same
 * definition is what the oracle evaluates in trig_mode 1; tests/test_oracle_yaw.py checks it against mpmath.
 * Usable from host code too (cos(yaw_max) is prepared on the host).  Constants: tools/gen_trig_tables.py.
 */
#pragma once
#include <cmath>
#if defined(__CUDACC__)
#include <cuda_runtime.h>
#else /* a plain host compiler (the host build of the LPA* core, tests/cpp/lpa_emul.cpp): the qualifiers mean host code */
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif
#endif

namespace mplb {
namespace trig {

#define MPLB_TRIG_CONST static constexpr
MPLB_TRIG_CONST double PIO2_1 = 0x1.921fb54442d18p+0, PIO2_2 = 0x1.1a62633145c07p-54, PIO2_3 = -0x1.f1976b7ed8fbcp-110;
MPLB_TRIG_CONST double TWO_OVER_PI = 0x1.45f306dc9c883p-1;
/* 1/n! as double-double (hi, lo), n = 2..31 */
#define MPLB_INV_FACT_INIT { \
  {0x1.0000000000000p-1, 0x0.0p+0}, /* 1/2! */ \
  {0x1.5555555555555p-3, 0x1.5555555555555p-57}, /* 1/3! */ \
  {0x1.5555555555555p-5, 0x1.5555555555555p-59}, /* 1/4! */ \
  {0x1.1111111111111p-7, 0x1.1111111111111p-63}, /* 1/5! */ \
  {0x1.6c16c16c16c17p-10, -0x1.f49f49f49f49fp-65}, /* 1/6! */ \
  {0x1.a01a01a01a01ap-13, 0x1.a01a01a01a01ap-73}, /* 1/7! */ \
  {0x1.a01a01a01a01ap-16, 0x1.a01a01a01a01ap-76}, /* 1/8! */ \
  {0x1.71de3a556c734p-19, -0x1.c154f8ddc6c00p-73}, /* 1/9! */ \
  {0x1.27e4fb7789f5cp-22, 0x1.cbbc05b4fa99ap-76}, /* 1/10! */ \
  {0x1.ae64567f544e4p-26, -0x1.c062e06d1f209p-80}, /* 1/11! */ \
  {0x1.1eed8eff8d898p-29, -0x1.2aec959e14c06p-83}, /* 1/12! */ \
  {0x1.6124613a86d09p-33, 0x1.f28e0cc748ebep-87}, /* 1/13! */ \
  {0x1.93974a8c07c9dp-37, 0x1.05d6f8a2efd1fp-92}, /* 1/14! */ \
  {0x1.ae7f3e733b81fp-41, 0x1.1d8656b0ee8cbp-97}, /* 1/15! */ \
  {0x1.ae7f3e733b81fp-45, 0x1.1d8656b0ee8cbp-101}, /* 1/16! */ \
  {0x1.952c77030ad4ap-49, 0x1.ac981465ddc6cp-103}, /* 1/17! */ \
  {0x1.6827863b97d97p-53, 0x1.eec01221a8b0bp-107}, /* 1/18! */ \
  {0x1.2f49b46814157p-57, 0x1.2650f61dbdcb4p-112}, /* 1/19! */ \
  {0x1.e542ba4020225p-62, 0x1.ea72b4afe3c2fp-120}, /* 1/20! */ \
  {0x1.71b8ef6dcf572p-66, -0x1.d043ae40c4647p-120}, /* 1/21! */ \
  {0x1.0ce396db7f853p-70, -0x1.aebcdbd20331cp-124}, /* 1/22! */ \
  {0x1.761b41316381ap-75, -0x1.3423c7d91404fp-130}, /* 1/23! */ \
  {0x1.f2cf01972f578p-80, -0x1.9ada5fcc1ab14p-135}, /* 1/24! */ \
  {0x1.3f3ccdd165fa9p-84, -0x1.58ddadf344487p-139}, /* 1/25! */ \
  {0x1.88e85fc6a4e5ap-89, -0x1.71c37ebd16540p-143}, /* 1/26! */ \
  {0x1.d1ab1c2dccea3p-94, 0x1.054d0c78aea14p-149}, /* 1/27! */ \
  {0x1.0a18a2635085dp-98, 0x1.b9e2e28e1aa54p-153}, /* 1/28! */ \
  {0x1.259f98b4358adp-103, 0x1.eaf8c39dd9bc5p-157}, /* 1/29! */ \
  {0x1.3932c5047d60ep-108, 0x1.832b7b530a627p-162}, /* 1/30! */ \
  {0x1.434d2e783f5bcp-113, 0x1.0b87b91be9affp-167}, /* 1/31! */ \
}

struct DD { double hi, lo; };
#ifdef __CUDA_ARCH__
__device__ __forceinline__ double t_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double t_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double t_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double t_fma(double a, double b, double c) { return __fma_rn(a, b, c); }
#else
inline double t_add(double a, double b) { return a + b; }
inline double t_sub(double a, double b) { return a - b; }
inline double t_mul(double a, double b) { return a * b; }
inline double t_fma(double a, double b, double c) { return std::fma(a, b, c); }
#endif
__host__ __device__ inline DD two_sum(double a, double b) {
  double s = t_add(a, b), bb = t_sub(s, a);
  return {s, t_add(t_sub(a, t_sub(s, bb)), t_sub(b, bb))};
}
__host__ __device__ inline DD quick_two_sum(double a, double b) { double s = t_add(a, b); return {s, t_sub(b, t_sub(s, a))}; }
__host__ __device__ inline DD two_prod(double a, double b) { double p = t_mul(a, b); return {p, t_fma(a, b, -p)}; }
__host__ __device__ inline DD dd_add(DD x, DD y) {
  DD s = two_sum(x.hi, y.hi), t = two_sum(x.lo, y.lo);
  s.lo = t_add(s.lo, t.hi);
  s = quick_two_sum(s.hi, s.lo);
  s.lo = t_add(s.lo, t.lo);
  return quick_two_sum(s.hi, s.lo);
}
__host__ __device__ inline DD dd_mul(DD x, DD y) {
  DD p = two_prod(x.hi, y.hi);
  p.lo = t_add(p.lo, t_add(t_mul(x.hi, y.lo), t_mul(x.lo, y.hi)));
  return quick_two_sum(p.hi, p.lo);
}
__host__ __device__ inline DD dd_neg(DD x) { return {-x.hi, -x.lo}; }

/* Reference-quality path: everything in double-double, ~2^-100 accurate.  About 1.5k instructions; taken only when the
 * quick path below cannot decide the rounding (about one call in 16 000). */
__host__ __device__ __noinline__ inline void sincos_cr_slow(double x, double *sn, double *cs) {
  const double INV_FACT[30][2] = MPLB_INV_FACT_INIT; /* folded into immediates by the unrolled loops */
  const double kd = rint(t_mul(x, TWO_OVER_PI));
  const int k = (int)kd;
  DD a = two_prod(kd, PIO2_1), b = two_prod(kd, PIO2_2), c = two_prod(kd, PIO2_3);
  DD r = two_sum(x, -a.hi);
  r = dd_add(r, DD{-a.lo, 0.0});
  r = dd_add(r, dd_neg(b));
  r = dd_add(r, dd_neg(c));
  const DD r2 = dd_mul(r, r);
  DD ps = {INV_FACT[29][0], INV_FACT[29][1]}; /* 1/31! */
#pragma unroll
  for (int n = 29; n >= 3; n -= 2) {
    ps = dd_mul(ps, r2);
    ps = dd_add(DD{INV_FACT[n - 2][0], INV_FACT[n - 2][1]}, dd_neg(ps));
  }
  ps = dd_mul(ps, r2);
  ps = dd_add(DD{1.0, 0.0}, dd_neg(ps));
  const DD s = dd_mul(ps, r);
  DD pc = {INV_FACT[28][0], INV_FACT[28][1]}; /* 1/30! */
#pragma unroll
  for (int n = 28; n >= 2; n -= 2) {
    pc = dd_mul(pc, r2);
    pc = dd_add(DD{INV_FACT[n - 2][0], INV_FACT[n - 2][1]}, dd_neg(pc));
  }
  pc = dd_mul(pc, r2);
  const DD cq = dd_add(DD{1.0, 0.0}, dd_neg(pc));
  DD so, co;
  switch (((k % 4) + 4) % 4) {
    case 0: so = s; co = cq; break;
    case 1: so = cq; co = dd_neg(s); break;
    case 2: so = dd_neg(s); co = dd_neg(cq); break;
    default: so = dd_neg(cq); co = s; break;
  }
  *sn = t_add(so.hi, so.lo);
  *cs = t_add(co.hi, co.lo);
}

/* sin(x) and cos(x), each rounded to nearest, |x| < 2^20 (Ziv's two-step scheme).
 * Quick path: the same double-double argument reduction, the leading terms of the series in double-double
 * (sin: r, r^3/3!, r^5/5!, r^7/7!; cos: 1, r^2/2!, ..., r^8/8!) and the remaining tail (below 2^-21 of the result) in
 * plain double, for a total error under 2^-70 of the result.  The rounding of hi + lo is accepted when it is the same
 * for lo +- 2^-68 |hi|; otherwise the slow path decides.  Both paths return the correctly rounded value, so which one
 * ran is unobservable. */
__host__ __device__ __noinline__ inline void sincos_cr(double x, double *sn, double *cs) {
  const double F[30][2] = MPLB_INV_FACT_INIT; /* only constant indices are used: folded into immediates */
  const double kd = rint(t_mul(x, TWO_OVER_PI));
  const int k = (int)kd;
  DD a = two_prod(kd, PIO2_1), b = two_prod(kd, PIO2_2), c = two_prod(kd, PIO2_3);
  DD r = two_sum(x, -a.hi);
  r = dd_add(r, DD{-a.lo, 0.0});
  r = dd_add(r, dd_neg(b));
  r = dd_add(r, dd_neg(c));
  const DD r2 = dd_mul(r, r);
  const double z = r2.hi;
  const double z2 = t_mul(z, z);
  /* sin */
  const DD r3 = dd_mul(r2, r), r5 = dd_mul(r3, r2), r7 = dd_mul(r5, r2);
  double ps = F[19][0];                                   /* 1/21! */
  ps = t_sub(F[17][0], t_mul(z, ps));                      /* 1/19! */
  ps = t_sub(F[15][0], t_mul(z, ps));
  ps = t_sub(F[13][0], t_mul(z, ps));
  ps = t_sub(F[11][0], t_mul(z, ps));
  ps = t_sub(F[9][0], t_mul(z, ps));
  ps = t_sub(F[7][0], t_mul(z, ps));                       /* 1/9! */
  const double tail_s = t_mul(t_mul(r.hi, t_mul(z2, z2)), ps);
  DD s = dd_add(dd_mul(r5, DD{F[3][0], F[3][1]}), dd_neg(dd_mul(r7, DD{F[5][0], F[5][1]})));
  s = dd_add(s, DD{tail_s, 0.0});
  s = dd_add(dd_neg(dd_mul(r3, DD{F[1][0], F[1][1]})), s);
  s = dd_add(r, s);
  /* cos */
  const DD r4 = dd_mul(r2, r2), r6 = dd_mul(r4, r2), r8 = dd_mul(r4, r4);
  double pc = F[20][0];                                   /* 1/22! */
  pc = t_sub(F[18][0], t_mul(z, pc));
  pc = t_sub(F[16][0], t_mul(z, pc));
  pc = t_sub(F[14][0], t_mul(z, pc));
  pc = t_sub(F[12][0], t_mul(z, pc));
  pc = t_sub(F[10][0], t_mul(z, pc));
  pc = t_sub(F[8][0], t_mul(z, pc));                       /* 1/10! */
  const double tail_c = -t_mul(t_mul(t_mul(z2, z2), z), pc);
  DD cq = dd_add(dd_neg(dd_mul(r6, DD{F[4][0], F[4][1]})), dd_mul(r8, DD{F[6][0], F[6][1]}));
  cq = dd_add(cq, DD{tail_c, 0.0});
  cq = dd_add(dd_mul(r4, DD{F[2][0], F[2][1]}), cq);
  cq = dd_add(DD{-t_mul(r2.hi, 0.5), -t_mul(r2.lo, 0.5)}, cq);
  cq = dd_add(DD{1.0, 0.0}, cq);
  DD so, co;
  switch (((k % 4) + 4) % 4) {
    case 0: so = s; co = cq; break;
    case 1: so = cq; co = dd_neg(s); break;
    case 2: so = dd_neg(s); co = dd_neg(cq); break;
    default: so = dd_neg(cq); co = s; break;
  }
  const double es = t_mul(fabs(so.hi), 0x1p-68), ec = t_mul(fabs(co.hi), 0x1p-68);
  const double s1 = t_add(so.hi, t_add(so.lo, es)), s2 = t_add(so.hi, t_sub(so.lo, es));
  const double c1 = t_add(co.hi, t_add(co.lo, ec)), c2 = t_add(co.hi, t_sub(co.lo, ec));
  if (s1 == s2 && c1 == c2) { *sn = s1; *cs = c1; return; }
#if defined(MPLB_TRIG_STATS) && !defined(__CUDA_ARCH__)
  mplb_trig_slow_calls++;
#endif
  sincos_cr_slow(x, sn, cs);
}

}  // namespace trig
}  // namespace mplb
