// physics.cuh -- per-pair / per-term arithmetic of the torchmd force field,
// shared by every kernel.  Pure functions on scalars; compiled for the device
// by nvcc and (for unit tests only, tests/hostcheck) for the host by g++.
//
// Two kinds of arithmetic live here:
//  * the DECISION arithmetic (minimum image, squared distance, cutoff test) is
//    written with explicitly rounded single operations so that a pair is inside
//    the cutoff here exactly when the reference's fp32 torch path says so
//    (forces.py:360-372, 76-81): sub, div, round-half-even, mul, sub, then
//    sqrt_rn(fma(z,z,fma(y,y,x*x))) <= fl32(cutoff)   [measured, see
//    tests/golden/PROVENANCE.txt];
//  * the VALUE arithmetic (energies, force coefficients) is ordinary fp32 with
//    FMA contraction allowed; it only has to meet the 1e-4 kcal/mol/A tolerance.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define TMD_HD __host__ __device__ __forceinline__
#else
#define TMD_HD inline
#endif

namespace tmd {

// ---- exactly rounded primitives ------------------------------------------------
TMD_HD float mul_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  volatile float r = a * b;
  return r;
#endif
}
TMD_HD float add_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  volatile float r = a + b;
  return r;
#endif
}
TMD_HD float sub_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  volatile float r = a - b;
  return r;
#endif
}
TMD_HD float div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  volatile float r = a / b;
  return r;
#endif
}
TMD_HD float fma_rn(float a, float b, float c) {
#if defined(__CUDA_ARCH__)
  return __fmaf_rn(a, b, c);
#else
  return fmaf(a, b, c);
#endif
}
TMD_HD float sqrt_rn(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  volatile float r = sqrtf(a);
  return r;
#endif
}
TMD_HD float rsqrt_fast(float a) {
#if defined(__CUDA_ARCH__)
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
#else
  return 1.0f / sqrtf(a);
#endif
}

// 1/sqrt(a) to ~1 ulp: hardware approximation (2 ulp) + one Newton step.  The r^-12
// wall amplifies the relative error of 1/r thirteen-fold, so the raw approximation
// alone would cost ~5e-5 kcal/mol/A on a close O-O pair.
TMD_HD float rsqrt_refined(float a) {
  float y = rsqrt_fast(a);
  float t = a * y;
  return fmaf(y, fmaf(-0.5f * t, y, 0.5f), y);
}

// ---- minimum image, one component -----------------------------------------------
// Reference: w = d - L * round(d / L), four separately rounded ops, round half to
// even (forces.py:364).  The quotient is first estimated with a multiply and
// rounded with the 1.5*2^23 trick; whenever that estimate is further than 0.05
// from a rounding boundary (and small enough for the trick) it provably equals
// rint(div_rn(d, L)), because |d*fl(1/L) - div_rn(d,L)| < 2^-22 |q| < 1e-3 for
// |q| < 4096.  Otherwise the true IEEE division is taken.  L*r and the final
// subtraction are single rounded ops like torch's.  `r` returns the image count.
TMD_HD float min_image_exact(float d, float L, float invL, float& r) {
  const float magic = 12582912.0f;  // 1.5 * 2^23
  float q = d * invL;
  r = sub_rn(add_rn(q, magic), magic);
  if (!(fabsf(q - r) < 0.45f) || !(fabsf(q) < 4096.0f)) r = rintf(div_rn(d, L));
  return sub_rn(d, mul_rn(L, r));
}
// Same result without the guard, valid when the caller guarantees |w| < 0.45 L and
// |d| < 4096 L for every pair it sees: the host checks  cutoff + 2*skin < 0.45 * min(L)
// (listed pairs cannot be further apart) and k_prepare flags positions beyond 2000 L.
TMD_HD float min_image_fast(float d, float L, float invL, float& r) {
  const float magic = 12582912.0f;
  r = sub_rn(add_rn(d * invL, magic), magic);
  return sub_rn(d, mul_rn(L, r));
}
TMD_HD float min_image(float d, float L, float invL) {
  float r;
  return min_image_exact(d, L, invL, r);
}

// Exact rounding error of d = fl(a - b)  (Knuth TwoSum on a + (-b)): a - b == d + err.
// Across the periodic boundary a - b is ~L and loses up to ulp(L)/2 (4e-6 A for
// L ~ 100 A); with a force gradient of ~40 kcal/mol/A^2 on a hydrogen bond that alone
// is 1.5e-4 kcal/mol/A -- the dominant error of the reference's own fp32 path.  The
// cutoff DECISION keeps the reference's rounded value; the force VALUES add err back.
TMD_HD float sub_err(float a, float b, float d) {
  float a1 = add_rn(d, b);
  float c1 = sub_rn(d, a1);
  float da = sub_rn(a, a1);
  return sub_rn(da, add_rn(b, c1));
}

// Separation of a pair that straddles the box, for the force VALUES: one fused multiply-add  fl(d - L * n)  on the
// unrounded product (the decision path's fl(d - fl(L * n)) carries the rounding of L * n, up to ulp(L * n) / 2, for the
// image counts 3, 5, 6, 7 ...; for 0, +-1, +-2, +-4 both are the same bits), plus the bits fl(a - b) dropped.
TMD_HD float straddle_value(float a, float b, float d, float L, float n) { return add_rn(fmaf(-L, n, d), sub_err(a, b, d)); }

TMD_HD float rcp_refined(float a) {
#if defined(__CUDA_ARCH__)
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(a));
  return fmaf(y, fmaf(-a, y, 1.0f), y);  // one Newton step: ~0.5 ulp, no slow path
#else
  return 1.0f / a;
#endif
}

// Largest fp32 s with sqrt_rn(s) <= rc: turns the reference's `dist <= cutoff` into a
// comparison on the squared distance without changing a single decision (host only).
inline float squared_threshold(float rc) {
  float s = rc * rc;
  while (sqrtf(s) > rc) s = nextafterf(s, 0.0f);
  for (;;) {
    float up = nextafterf(s, INFINITY);
    if (sqrtf(up) <= rc) s = up;
    else break;
  }
  return s;
}

// Squared length in the rounding order of torch.norm(dim=1) on (P,3) fp32.
TMD_HD float norm2_ref(float x, float y, float z) {
  return fma_rn(z, z, fma_rn(y, y, mul_rn(x, x)));
}

// The reference's cutoff decision for one pair of a periodic box, from the original fp32
// positions (guarded minimum image: valid for any separation).
TMD_HD bool ref_inside(float xi, float yi, float zi, float xj, float yj, float zj,
                       float Lx, float Ly, float Lz, float iLx, float iLy, float iLz, float s_max) {
  const float wx = min_image(sub_rn(xi, xj), Lx, iLx);
  const float wy = min_image(sub_rn(yi, yj), Ly, iLy);
  const float wz = min_image(sub_rn(zi, zj), Lz, iLz);
  return norm2_ref(wx, wy, wz) <= s_max;
}

// ---- fp64 decision arithmetic ("precision: double") -------------------------------------
// The reference's fp64 path makes the same decision with the same rounded operations in
// double: w = d - L * rint(d / L) (four separately rounded ops), s = fma(z,z,fma(y,y,x*x))
// (torch.norm(dim=1) on (P,3) fp64, bit-identical on x86-64), inside iff sqrt_rn(s) <= cutoff.
// The overloads keep nvcc from contracting any of it.
TMD_HD double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);
#else
  volatile double r = a * b;
  return r;
#endif
}
TMD_HD double add_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dadd_rn(a, b);
#else
  volatile double r = a + b;
  return r;
#endif
}
TMD_HD double sub_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dsub_rn(a, b);
#else
  volatile double r = a - b;
  return r;
#endif
}
TMD_HD double div_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __ddiv_rn(a, b);
#else
  volatile double r = a / b;
  return r;
#endif
}
TMD_HD double fma_rn(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}
TMD_HD double sqrt_rn(double a) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(a);
#else
  volatile double r = sqrt(a);
  return r;
#endif
}
// Minimum image of one fp64 component, the reference's rounding for any separation.
TMD_HD double min_image64(double d, double L) { return sub_rn(d, mul_rn(L, rint(div_rn(d, L)))); }
TMD_HD double norm2_ref(double x, double y, double z) { return fma_rn(z, z, fma_rn(y, y, mul_rn(x, x))); }
// Largest double s with sqrt_rn(s) <= rc (host only): the fp64 decision on the squared distance.
inline double squared_threshold64(double rc) {
  double s = rc * rc;
  while (sqrt(s) > rc) s = nextafter(s, 0.0);
  for (;;) {
    const double up = nextafter(s, INFINITY);
    if (sqrt(up) <= rc) s = up;
    else break;
  }
  return s;
}

// ---- Wrapper.wrap (wrapper.py:24-27): image offset of a group from its coordinate sum ----
//   com = sum / len ;  offset = floor(com / box) * box        (three rounded fp32 operations)
TMD_HD float wrap_offset(float coord_sum, int len, float box) {
  return mul_rn(floorf(div_rn(div_rn(coord_sum, (float)len), box)), box);
}
TMD_HD double wrap_offset(double coord_sum, int len, double box) {
  return mul_rn(floor(div_rn(div_rn(coord_sum, (double)len), box)), box);
}

// ---- fixed-point periodic coordinates ---------------------------------------------------
// For the pair kernel of a periodic box a coordinate x along a dimension of length L is
// also kept as the 32-bit integer  X = round(x * 2^32 / L) mod 2^32  (computed in fp64 from
// the caller's fp32 position, once per atom and step).  The two's-complement difference
// X_i - X_j then IS the minimum-image separation in units of L / 2^32 (2.3e-8 A for
// L = 100 A): exact, no image search, no loss of low bits across the boundary or for atoms
// that drifted several boxes away -- the VALUES get better than the reference's own fp32
// path.  The cutoff DECISION must still be the reference's; the squared distance s_fx
// computed this way differs from the reference's rounded s_ref by at most
//     m = c0 + c1 * P,      P = largest |coordinate| in the system
// (fx_margin below), so  s_fx < s_max - m  =>  inside,  s_fx > s_max + m  =>  outside, and only
// the ~1e-4 of the pairs in between re-do the reference's arithmetic on the original
// positions (ref_inside).
TMD_HD int32_t fx_encode(float x, double inv_unit) {
#if defined(__CUDA_ARCH__)
  return (int32_t)(uint32_t)(unsigned long long)__double2ll_rn((double)x * inv_unit);  // saturating, NaN -> 0
#else
  const double v = (double)x * inv_unit;
  if (!(fabs(v) < 9.0e18)) return 0;
  return (int32_t)(uint32_t)(unsigned long long)llrint(v);
#endif
}
TMD_HD float fx_delta(int32_t a, int32_t b, float unit) {
  return (float)(int32_t)((uint32_t)a - (uint32_t)b) * unit;
}

// Bound on |s_fx - s_ref| for every pair whose true minimum-image distance is <= rmax
// (host only; u = 2^-24 is the relative error of one rounded fp32 operation).
//   reference (forces.py:360-372): d = fl(p_i - p_j), |d| <= 2P, error <= 2uP;
//   m = fl(L * n), |L n| <= 2P + L/2, error <= u (2P + L);  w = fl(d - m), error <= u L / 2
//   (n = round(fl(d / L)) is the true image count for these pairs);  so each component of
//   w_ref is within  e_ref = u (4P + 1.5 L)  of the exact separation.
//   fixed point: quantisation <= L 2^-32, then int->float, *unit (itself rounded): 3u |w|.
//   s = x*x + y*y + z*z: at most 3 roundings of a sum of positive terms on either side.
// |s_a - s_b| <= 2 rmax sqrt(3) (e_ref + e_fx) + 6u rmax^2, doubled for second-order terms.
inline void fx_margin(double rmax, double Lmax, double* c0, double* c1) {
  const double u = 1.0 / 16777216.0, q = 1.7320508075688772;
  const double e_fix = Lmax / 4294967296.0 + 3.0 * u * rmax;
  *c0 = 2.0 * (2.0 * rmax * q * (1.5 * u * Lmax + e_fix) + 6.0 * u * rmax * rmax);
  *c1 = 2.0 * (2.0 * rmax * q * 4.0 * u);
}

// ---- pair parameters (uniform per launch) -----------------------------------------
struct PairParams {
  uint32_t terms;     // TMD_TERM(...) mask of pair terms
  int periodic;       // 0: no wrapping (box all zero)
  int has_cutoff;     // 0: every listed pair interacts
  int has_switch;     // LJ switching on (needs cutoff)
  int rfa;            // reaction-field electrostatics (needs cutoff)
  float s_max;        // largest fp32 s with sqrt_rn(s) <= fl32(cutoff); +inf if no cutoff
  float cutoff;       // fl32(cutoff)
  float switch_dist;  // fl32(switch_dist)
  float inv_sw_width; // 1 / (cutoff - switch_dist)
  // reaction-field constants (forces.py:466-468); with particle-mesh Ewald, which excludes the reaction field, the same
  // words hold the Ewald splitting parameter alpha and 2 alpha / sqrt(pi)
  union { float krf; float ew_alpha; };
  union { float crf; float ew_beta; };
  float two_krf;
  int true_gradient;  // 1: switched-LJ force is the exact d(E*s)/dr (the reference's autograd path, forces.py:328-336);
                      // 0: the reference's explicit formula with its extra 1/r (forces.py:410-412)
};

enum : uint32_t {
  T_ELEC = 1u << 5,
  T_LJ = 1u << 6,
  T_REP = 1u << 7,
  T_REPCG = 1u << 8,
};

// Energy and dE/dr of one in-cutoff pair at squared distance s.
//   qq   : coulomb_constant * q_i * q_j
//   A, B : LJ table entries of the type pair
// Returns dE/dr summed over the enabled terms; energies are ADDED to e_lj / e_el /
// e_rep / e_repcg.  Follows forces.py:381-491 including the reference's switched
// LJ force  s*dE/dr + E*s'/r  (the extra 1/r is the reference's, forces.py:410-412).
// MODE 0: terms chosen at run time from pp;  MODE 1: LJ with switch + reaction-field
// electrostatics (the production water/protein set-up) resolved at compile time;  MODE 2: terms
// chosen at run time, electrostatics as the real-space part of particle-mesh Ewald,
// qq erfc(alpha r) / r with no shift or switch.  erfcf and expf are the CUDA library functions
// (at most 4 and 2 ulp: CUDA C Programming Guide, "Mathematical Functions"), so a pair's energy and
// force coefficient are within about 1e-6 relative of their exact values.
template <int MODE>
TMD_HD float pair_terms(const PairParams& pp, float s, float qq, float A, float B,
                        float& e_el, float& e_lj, float& e_rep, float& e_repcg,
                        float& rinv_out) {
  const bool do_lj = MODE == 1 ? true : (pp.terms & T_LJ) != 0;
  const bool do_el = MODE == 1 ? true : (pp.terms & T_ELEC) != 0;
  const bool do_rep = MODE == 1 ? false : (pp.terms & T_REP) != 0;
  const bool do_cg = MODE == 1 ? false : (pp.terms & T_REPCG) != 0;
  const bool sw_on = MODE == 1 ? true : pp.has_switch != 0;
  const bool rf_on = MODE == 1 ? true : pp.rfa != 0;
  float rinv = rsqrt_refined(s);
  float r = s * rinv;
  float rinv2 = rcp_refined(s);  // ~0.5 ulp: the high powers below inherit 3x, not 6x, its error
  float rinv6 = rinv2 * rinv2 * rinv2;
  float dedr = 0.0f;
  rinv_out = rinv;
  if (do_lj) {
    float a12 = A * rinv6 * rinv6;
    float b6 = B * rinv6;
    float e = a12 - b6;
    float f = (6.0f * b6 - 12.0f * a12) * rinv;
    if (sw_on) {
      // branch-free: t = 0 below the switch distance gives sw = 1, dsw = 0
      float t = fmaxf((r - pp.switch_dist) * pp.inv_sw_width, 0.0f);
      float sw = 1.0f + t * t * t * (-10.0f + t * (15.0f - t * 6.0f));
      float dsw = t * t * (-30.0f + t * (60.0f - t * 30.0f)) * pp.inv_sw_width;
      // explicit path: s*dE/dr + E*s'/r (sic, forces.py:410-412); autograd path: the true derivative
      const bool exact = MODE == 1 ? false : pp.true_gradient != 0;
      f = sw * f + e * dsw * (exact ? 1.0f : rinv);
      e = e * sw;
    }
    e_lj += e;
    dedr += f;
  }
  if (do_el) {
    if (MODE == 2) {
      const float ar = pp.ew_alpha * r;
      const float e = qq * erfcf(ar) * rinv;
      e_el += e;
      dedr -= (e + qq * pp.ew_beta * expf(-ar * ar)) * rinv;
    } else if (rf_on) {
      e_el += qq * (rinv + pp.krf * s - pp.crf);
      dedr += qq * (pp.two_krf * r - rinv2);
    } else {
      float e = qq * rinv;
      e_el += e;
      dedr -= e * rinv;
    }
  }
  if (do_rep) {
    float a12 = A * rinv6 * rinv6;
    e_rep += a12;
    dedr -= 12.0f * a12 * rinv;
  }
  if (do_cg) {
    float b6 = B * rinv6;
    e_repcg += b6;
    dedr -= 6.0f * b6 * rinv;
  }
  return dedr;
}

// ---- two partners at once: fp32x2 arithmetic ------------------------------------------------
// The pair kernel evaluates the partners a lane handles two at a time.  Hopper (sm_90) has no
// packed single-precision instructions, so each F2 operation is two scalar, correctly rounded
// operations that the compiler may not contract or reassociate (__fmaf_rn / __fmul_rn /
// __fadd_rn); the two independent chains also give the scheduler instruction-level parallelism.
// The host build (fmaf per half) reproduces the device results exactly apart from the two
// hardware approximations that seed the Newton steps.
struct F2 {
  float x, y;
};
TMD_HD F2 f2(float a, float b) { return F2{a, b}; }
TMD_HD F2 f2(float a) { return F2{a, a}; }
TMD_HD F2 f2_fma(F2 a, F2 b, F2 c) { return F2{fma_rn(a.x, b.x, c.x), fma_rn(a.y, b.y, c.y)}; }
TMD_HD F2 f2_mul(F2 a, F2 b) { return F2{mul_rn(a.x, b.x), mul_rn(a.y, b.y)}; }
TMD_HD F2 f2_add(F2 a, F2 b) { return F2{add_rn(a.x, b.x), add_rn(a.y, b.y)}; }
// hardware seeds of the Newton steps: 1/sqrt(s) and -1/s (the sign saves every negation below)
TMD_HD float rsqrt_seed(float s) { return rsqrt_fast(s); }
TMD_HD float neg_rcp_seed(float s) {
#if defined(__CUDA_ARCH__)
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(-s));
  return y;
#else
  return -1.0f / s;
#endif
}

// Uniform constants of pair_coef2 (host-built once per PairParams).
struct SwitchConsts {
  float neg_switch_dist, inv_sw_width;
  float d1, d2, d3;  // -ds/dr polynomial: t^2 (d3 + t (d2 + t d1)),  d = (30, -60, 30) / (cutoff - switch_dist)
  float two_krf, krf, neg_crf;  // reaction field; the Ewald variants (EW) read 2 alpha / sqrt(pi) and alpha from the
                                // first two (the reaction field and PME exclude each other; make_switch_consts_ewald)
};
// Also covers the term sets without switching (t stays 0: sw = 1, ds/dr = 0) and without a reaction field
// (k_rf = c_rf = 0: plain Coulomb), so pair_coef2 serves every combination of "lj" and "electrostatics".
inline SwitchConsts make_switch_consts(const PairParams& pp) {
  SwitchConsts c;
  if (pp.has_switch) {
    c.neg_switch_dist = -pp.switch_dist;
    c.inv_sw_width = pp.inv_sw_width;
    c.d1 = 30.0f * pp.inv_sw_width;
    c.d2 = -60.0f * pp.inv_sw_width;
    c.d3 = 30.0f * pp.inv_sw_width;
  } else {
    c.neg_switch_dist = -1.0e30f;  // (r - 1e30) * 1 < 0 for every r: t = 0
    c.inv_sw_width = 1.0f;
    c.d1 = c.d2 = c.d3 = 0.0f;
  }
  c.two_krf = pp.rfa ? pp.two_krf : 0.0f;
  c.krf = pp.rfa ? pp.krf : 0.0f;
  c.neg_crf = pp.rfa ? -pp.crf : 0.0f;
  return c;
}
// The Ewald instantiations (EW) of pair_coef2 and the cluster kernel's coefficient read alpha and 2 alpha / sqrt(pi).
inline SwitchConsts make_switch_consts_ewald(const PairParams& pp) {
  SwitchConsts c = make_switch_consts(pp);
  c.two_krf = pp.ew_beta;
  c.krf = pp.ew_alpha;
  c.neg_crf = 0.0f;
  return c;
}

// Real-space Ewald electrostatics of two partners for the packed coefficients: MINUS dE/dr and MINUS the energy,
//   -dE/dr = nqq (erfc(alpha r) (-1/r^2) - beta exp(-alpha^2 r^2) / r),   -E = nqq erfc(alpha r) / r
// with nqq = -(k qi qj) and nr2 = -1/r^2 (erfcf / expf per half, within 4 / 2 ulp).
TMD_HD F2 ewald_ndedr2(const SwitchConsts& c, F2 nqq, F2 r, F2 rinv, F2 nr2, F2& erfc_ar) {
  const F2 ar = f2_mul(r, f2(c.krf));  // alpha
  erfc_ar = f2(erfcf(ar.x), erfcf(ar.y));
  const F2 ex = f2(expf(-ar.x * ar.x), expf(-ar.y * ar.y));
  const F2 nb = f2_mul(f2_mul(ex, rinv), f2(-c.two_krf));  // -2 alpha / sqrt(pi) exp(-alpha^2 r^2) / r
  return f2_mul(nqq, f2_fma(erfc_ar, nr2, nb));
}

// MINUS the force coefficient (dE/dr)/r of two partners for LJ with switch + reaction-field
// Coulomb in the explicit-force convention (pair_terms<1> restated with packed operations and
// signs arranged so that no negation is ever needed):
//   s    squared distances          nqq  -(k_e q_i q_j)             A, B  LJ table entries
//   y    rsqrt_seed(s)              nz   neg_rcp_seed(s)
// The force on atom i is then  F_i += w * result.  ENERGY: also the switched LJ energy and MINUS the
// reaction-field Coulomb energy of each partner (forces.py:389-415, 466-478).
// EW: real-space Ewald electrostatics (ewald_ndedr2) in place of the reaction field.
template <bool ENERGY, bool EW = false>
TMD_HD F2 pair_coef2(const SwitchConsts& c, F2 s, F2 nqq, F2 A, F2 B, F2 y, F2 nz, F2& e_lj, F2& ne_el) {
  // 1/r to ~1 ulp and r
  const F2 t = f2_mul(s, y);
  const F2 u = f2_fma(f2_mul(t, f2(-0.5f)), y, f2(0.5f));
  const F2 rinv = f2_fma(y, u, y);
  const F2 r = f2_mul(s, rinv);
  // -1/r^2 to ~0.5 ulp:  nz (1 + (1 + s nz))
  const F2 e1 = f2_fma(s, nz, f2(1.0f));
  const F2 nr2 = f2_fma(nz, e1, nz);
  const F2 nr6 = f2_mul(f2_mul(nr2, nr2), nr2);  // -1/r^6
  const F2 a12 = f2_mul(f2_mul(A, nr6), nr6);    //  A/r^12
  const F2 nb6 = f2_mul(B, nr6);                 // -B/r^6
  const F2 e = f2_add(a12, nb6);                 //  E_lj
  // -(dE/dr) of the unswitched LJ: (12 a12 - 6 b6) / r
  const F2 nf = f2_mul(f2_fma(nb6, f2(6.0f), f2_mul(a12, f2(12.0f))), rinv);
  // switch: t = max((r - r_s) / (r_c - r_s), 0), sw = 1 + t^3 (-10 + t (15 - 6 t)), -ds/dr
  F2 tt = f2_mul(f2_add(r, f2(c.neg_switch_dist)), f2(c.inv_sw_width));
  tt = f2(fmaxf(tt.x, 0.0f), fmaxf(tt.y, 0.0f));
  const F2 t2 = f2_mul(tt, tt);
  const F2 sw = f2_fma(f2_mul(t2, tt), f2_fma(tt, f2_fma(tt, f2(-6.0f), f2(15.0f)), f2(-10.0f)), f2(1.0f));
  const F2 ndsw = f2_mul(t2, f2_fma(tt, f2_fma(tt, f2(c.d1), f2(c.d2)), f2(c.d3)));
  // -(s dE/dr + E s'/r)   (the reference's explicit formula, forces.py:410-412)
  const F2 nfsw = f2_fma(sw, nf, f2_mul(f2_mul(e, ndsw), rinv));
  // reaction field: dE/dr = qq (2 k_rf r - 1/r^2)
  if constexpr (EW) {
    F2 ec;
    const F2 ndedr = f2_add(ewald_ndedr2(c, nqq, r, rinv, nr2, ec), nfsw);
    if (ENERGY) {
      e_lj = f2_mul(e, sw);
      ne_el = f2_mul(f2_mul(nqq, ec), rinv);  // -qq erfc(alpha r) / r
    }
    return f2_mul(ndedr, rinv);
  }
  const F2 ndedr = f2_fma(nqq, f2_fma(f2(c.two_krf), r, nr2), nfsw);
  if (ENERGY) {
    e_lj = f2_mul(e, sw);
    ne_el = f2_mul(nqq, f2_add(f2_fma(f2(c.krf), s, rinv), f2(c.neg_crf)));  // -qq (1/r + k_rf r^2 - c_rf)
  }
  return f2_mul(ndedr, rinv);
}
TMD_HD F2 pair_coef2(const SwitchConsts& c, F2 s, F2 nqq, F2 A, F2 B, F2 y, F2 nz) {
  F2 a, b;
  return pair_coef2<false>(c, s, nqq, A, B, y, nz, a, b);
}

// ---- bonded terms --------------------------------------------------------------------
// Templated on the real type: the bonded kernel evaluates them in fp64 (they are O(N),
// a few percent of the pair work, and a stiff bond turns the 6e-8 A rounding of an fp32
// bond length into a 5e-5 kcal/mol/A force error: 2k = 900 kcal/mol/A^2 for O-H),
// the host unit tests also in fp32.
template <typename T>
struct Vec3T {
  T x, y, z;
};
using Vec3 = Vec3T<float>;
using Vec3d = Vec3T<double>;
template <typename T> TMD_HD Vec3T<T> operator+(Vec3T<T> a, Vec3T<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T> TMD_HD Vec3T<T> operator-(Vec3T<T> a, Vec3T<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> TMD_HD Vec3T<T> operator*(T s, Vec3T<T> a) { return {s * a.x, s * a.y, s * a.z}; }
template <typename T> TMD_HD T dot(Vec3T<T> a, Vec3T<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> TMD_HD Vec3T<T> cross(Vec3T<T> a, Vec3T<T> b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <typename T> TMD_HD T norm(Vec3T<T> a) { return sqrt(dot(a, a)); }

// Minimum-image difference of two positions, reference rounding (decisions).
TMD_HD Vec3 delta_ref(Vec3 a, Vec3 b, int periodic, Vec3 L, Vec3 invL) {
  Vec3 d = {sub_rn(a.x, b.x), sub_rn(a.y, b.y), sub_rn(a.z, b.z)};
  if (periodic) {
    d.x = min_image(d.x, L.x, invL.x);
    d.y = min_image(d.y, L.y, invL.y);
    d.z = min_image(d.z, L.z, invL.z);
  }
  return d;
}

// The same difference for VALUE arithmetic in fp64: exact subtraction of the fp32
// inputs, minimum image with the fp32 box length.
TMD_HD Vec3d delta_f64(Vec3 a, Vec3 b, int periodic, Vec3 L) {
  Vec3d d = {(double)a.x - (double)b.x, (double)a.y - (double)b.y, (double)a.z - (double)b.z};
  if (periodic) {
    d.x -= (double)L.x * rint(d.x / (double)L.x);
    d.y -= (double)L.y * rint(d.y / (double)L.y);
    d.z -= (double)L.z * rint(d.z / (double)L.z);
  }
  return d;
}

// Harmonic bond (forces.py:494-503): E = k (r-r0)^2, dE/dr = 2k (r-r0).
template <typename T>
TMD_HD void bond_term(T r, T k, T r0, T& e, T& dedr) {
  T x = r - r0;
  e = k * x * x;
  dedr = T(2) * k * x;
}

// Harmonic angle (forces.py:506-539).  r21 = p0-p1, r23 = p2-p1.
template <typename T>
TMD_HD T angle_term(Vec3T<T> r21, Vec3T<T> r23, T k, T theta0, Vec3T<T>& f0, Vec3T<T>& f1, Vec3T<T>& f2) {
  T inv21 = T(1) / norm(r21);
  T inv23 = T(1) / norm(r23);
  T c = dot(r23, r21) * inv21 * inv23;
  c = c < T(-1) ? T(-1) : (c > T(1) ? T(1) : c);
  T dth = acos(c) - theta0;
  T sn = sqrt(T(1) - c * c);
  T coef = (sn != T(0)) ? (T(-2) * k * dth / sn) : T(0);  // zero force at sin==0
  f0 = (coef * inv21) * ((c * inv21) * r21 - inv23 * r23);
  f2 = (coef * inv23) * ((c * inv23) * r23 - inv21 * r21);
  f1 = T(-1) * (f0 + f2);
  return k * dth * dth;
}

// Torsion angle phi = -atan2(sin, cos) (forces.py:544-553) and the geometric
// factors the force projection needs.
template <typename T>
struct TorsionGeom {
  Vec3T<T> cA, cB;
  T nA2, nB2, n23, g1, g2, phi;
};
template <typename T>
TMD_HD TorsionGeom<T> torsion_geom(Vec3T<T> r12, Vec3T<T> r23, Vec3T<T> r34) {
  TorsionGeom<T> g;
  g.cA = cross(r12, r23);
  g.cB = cross(r23, r34);
  Vec3T<T> cC = cross(r23, g.cA);
  T nA = norm(g.cA), nB = norm(g.cB), nC = norm(cC);
  Vec3T<T> uB = (T(1) / nB) * g.cB;
  T cosphi = dot(g.cA, uB) / nA;
  T sinphi = dot(cC, uB) / nC;
  g.phi = -atan2(sinphi, cosphi);
  g.nA2 = nA * nA;
  g.nB2 = nB * nB;
  T n23sq = dot(r23, r23);
  g.n23 = sqrt(n23sq);
  g.g1 = dot(r12, r23) / n23sq;
  g.g2 = dot(r34, r23) / n23sq;
  return g;
}
// One torsion term: energy and dE/dphi-like coefficient (forces.py:566-579).
template <typename T>
TMD_HD void torsion_term(T phi, T k, T phi0, T per, int amber_form, T& e, T& coef) {
  if (amber_form) {
    T a = per * phi - phi0;
    e += k * (T(1) + cos(a));
    coef += -per * k * sin(a);
  } else {
    const T pi = T(3.14159265358979323846);
    T a = phi - phi0;
    if (a < -pi) a += T(2) * pi;
    else if (a > pi) a -= T(2) * pi;
    e += k * a * a;
    coef += T(2) * k * a;
  }
}
// Force projection (forces.py:584-603).
template <typename T>
TMD_HD void torsion_forces(const TorsionGeom<T>& g, T coef, Vec3T<T>& f0, Vec3T<T>& f1, Vec3T<T>& f2,
                           Vec3T<T>& f3) {
  T ff0 = (-coef * g.n23) / g.nA2;
  T ff3 = (coef * g.n23) / g.nB2;
  Vec3T<T> v0 = ff0 * g.cA;
  Vec3T<T> v3 = ff3 * g.cB;
  Vec3T<T> s = g.g1 * v0 - g.g2 * v3;
  f0 = T(-1) * v0;
  f1 = v0 + s;
  f2 = v3 - s;
  f3 = T(-1) * v3;
}

}  // namespace tmd
