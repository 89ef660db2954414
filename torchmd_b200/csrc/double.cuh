// double.cuh -- the "precision: double" path (tmd_set_precision(ctx, 64)): fp64 positions,
// velocities, forces and parameters, the reference's fp64 decisions bit for bit.
//
// Full Verlet rows only.  The cell list and the list build are the fp32 kernels of
// neighbor.cuh, run on an fp32 shadow of the positions that k_prepare_f64 writes: the list
// only has to be a superset of the pairs inside the cutoff and never decides anything, so the
// list radius carries the shadow's rounding (bound next to `margin` in tmd_b200.cu, finalize).
//
//   k_prepare_f64   every call: shadow positions, displacement trigger, far-position flag,
//                   refresh of the sorted fp64 records (sentinel record N stays NaN)
//   k_pack_f64      after a rebuild (gated like the rebuild kernels): the sorted records in the
//                   new order
//   k_pair_f64      one warp per atom over its full row, the reference's fp64 predicate, fp64
//                   values, shuffle reduction, one store per atom: no atomics on forces
//
// The bonded terms and the integrator are the <double> instantiations of the kernels of bonded.cuh
// and integrate.cuh.
#pragma once
#include "context.cuh"
#include "neighbor.cuh"
#include "pair.cuh"

namespace tmd {

__global__ void k_prepare_f64(DeviceState S, DeviceState64 D, const double* __restrict__ pos) {
  const int parity = (int)(S.counters[0] & 1ull);
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) S.flags[r * F_COUNT + F_REBUILD0 + (parity ^ 1)] = 0;
  if (i >= S.natoms) return;
  int* fl = S.flags + r * F_COUNT;
  const size_t a = (size_t)r * S.natoms + i;
  const double x = pos[a * 3 + 0], y = pos[a * 3 + 1], z = pos[a * 3 + 2];
  const float sx = (float)x, sy = (float)y, sz = (float)z;
  D.shadow[a * 3 + 0] = sx;
  D.shadow[a * 3 + 1] = sy;
  D.shadow[a * 3 + 2] = sz;
  const float4 ref = S.pos_ref[a];  // shadow positions of the last build
  const float dx = sx - ref.x, dy = sy - ref.y, dz = sz - ref.z;
  if (!(dx * dx + dy * dy + dz * dz <= S.trigger2)) fl[F_REBUILD0 + parity] = 1;  // also for NaN (no list yet)
  if (!(fabs(x) < D.pos_limit) || !(fabs(y) < D.pos_limit) || !(fabs(z) < D.pos_limit)) fl[F_FARPOS] = 1;
  D.xq_s[(size_t)r * (S.natoms + 1) + S.inv[a]] = Rec64{x, y, z, D.q[i]};
}

__global__ void k_pack_f64(DeviceState S, DeviceState64 D, const double* __restrict__ pos) {
  TMD_GATE
  const int r = blockIdx.y;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= S.natoms) return;
  const size_t base = (size_t)r * S.natoms;
  const int i = S.perm[base + k];
  const double* p = pos + (base + i) * 3;
  D.xq_s[(size_t)r * (S.natoms + 1) + k] = Rec64{p[0], p[1], p[2], D.q[i]};
}

// The reference's decision for one pair: rounded difference, minimum image, squared norm.
template <bool PERIODIC>
__device__ __forceinline__ double pair_s64(const Rec64& a, const Rec64& b, double Lx, double Ly, double Lz, double& wx,
                                           double& wy, double& wz) {
  wx = sub_rn(a.x, b.x);
  wy = sub_rn(a.y, b.y);
  wz = sub_rn(a.z, b.z);
  if (PERIODIC) {
    wx = min_image64(wx, Lx);
    wy = min_image64(wy, Ly);
    wz = min_image64(wz, Lz);
  }
  return norm2_ref(wx, wy, wz);
}

// dE/dr of one in-cutoff pair summed over the enabled terms (forces.py:381-491 in fp64); the
// per-term energies are ADDED to e_*.  EWALD: electrostatics as the real-space part of particle-mesh
// Ewald, qq erfc(alpha r) / r.
template <bool EWALD>
__device__ __forceinline__ double pair_terms64(const PairParams64& pp, double s, double qq, double A, double B, double& e_el,
                                               double& e_lj, double& e_rep, double& e_cg, double& rinv) {
  const double r = sqrt_rn(s);
#if defined(__CUDA_ARCH__)
  rinv = __drcp_rn(r);  // correctly rounded like 1.0 / r, without the division's slow-path call in the loop
#else
  rinv = 1.0 / r;
#endif
  const double rinv2 = rinv * rinv;
  const double rinv6 = rinv2 * rinv2 * rinv2;
  const double rinv12 = rinv6 * rinv6;
  double dedr = 0.0;
  if (pp.terms & T_LJ) {
    double e = A * rinv12 - B * rinv6;
    double f = (-12.0 * A * rinv12 + 6.0 * B * rinv6) * rinv;
    if (pp.has_switch && r > pp.switch_dist) {
      const double t = (r - pp.switch_dist) * pp.inv_sw_width;
      const double sw = 1.0 + t * t * t * (-10.0 + t * (15.0 - t * 6.0));
      const double dsw = t * t * (-30.0 + t * (60.0 - t * 30.0)) * pp.inv_sw_width;
      // explicit path: s*dE/dr + E*s'/r (sic, forces.py:410-412); autograd path: the true derivative
      f = sw * f + (pp.true_gradient ? e * dsw : e * dsw * rinv);
      e *= sw;
    }
    e_lj += e;
    dedr += f;
  }
  if (pp.terms & T_ELEC) {
    if (EWALD) {
      const double ar = pp.ew_alpha * r;
      const double e = qq * erfc(ar) * rinv;
      e_el += e;
      dedr -= (e + qq * pp.ew_beta * exp(-ar * ar)) * rinv;
    } else if (pp.rfa) {
      e_el += qq * (rinv + pp.krf * s - pp.crf);
      dedr += qq * (2.0 * pp.krf * r - rinv2);
    } else {
      const double e = qq * rinv;
      e_el += e;
      dedr -= e * rinv;
    }
  }
  if (pp.terms & T_REP) {
    e_rep += A * rinv12;
    dedr -= 12.0 * A * rinv12 * rinv;
  }
  if (pp.terms & T_REPCG) {
    e_cg += B * rinv6;
    dedr -= 6.0 * B * rinv6 * rinv;
  }
  return dedr;
}

template <bool ENERGY, bool PERIODIC, bool EWALD>
__device__ __forceinline__ void pair_f64_body(const DeviceState& S, const DeviceState64& D, double* __restrict__ forces,
                                              double* __restrict__ energies) {
  const int r = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * PAIR_WARPS + (threadIdx.x >> 5);
  const int N = S.natoms;
  const size_t base = (size_t)r * N;
  const PairParams64& pp = D.pp;
  double e_el = 0., e_lj = 0., e_rep = 0., e_cg = 0.;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[0] += 1;  // next call: other flag
  if (k < N) {
    const Rec64* __restrict__ xq = D.xq_s + (size_t)r * (N + 1);
    const int* __restrict__ row = S.nbr + (base + k) * (size_t)S.row_cap;
    const int n = S.nnbr[base + k];
    const Rec64 pi = xq[k];
    const int ti = S.type_s[base + k] * S.ntypes;
    const bool need_ab = (pp.terms & (T_LJ | T_REP | T_REPCG)) != 0;
    double Lx = 0., Ly = 0., Lz = 0.;
    if (PERIODIC) {
      Lx = D.L[3 * r];
      Ly = D.L[3 * r + 1];
      Lz = D.L[3 * r + 2];
    }
    double fx = 0., fy = 0., fz = 0.;
    for (int e = lane; e < n; e += 32) {
      const int entry = __ldcs(row + e);
      if (entry < 0) continue;
      const Rec64 pj = xq[entry & 0xffffff];
      double wx, wy, wz;
      const double s = pair_s64<PERIODIC>(pi, pj, Lx, Ly, Lz, wx, wy, wz);
      if (!(s <= pp.s_max)) continue;  // the reference's decision (NaN sentinel: outside)
      double A = 0., B = 0.;
      if (need_ab) {
        const int t = 2 * (ti + (entry >> 24));
        A = D.AB[t];
        B = D.AB[t + 1];
      }
      double rinv;
      const double dedr = pair_terms64<EWALD>(pp, s, pi.q * pj.q, A, B, e_el, e_lj, e_rep, e_cg, rinv);
      const double c = dedr * rinv;
      fx -= wx * c;
      fy -= wy * c;
      fz -= wz * c;
    }
    fx = warp_sum(fx);
    fy = warp_sum(fy);
    fz = warp_sum(fz);
    if (lane == 0) {
      double* f = forces + (base + S.perm[base + k]) * 3;
      f[0] = fx;
      f[1] = fy;
      f[2] = fz;
    }
  }
  if (ENERGY) {
    __shared__ double red[PAIR_WARPS];
    double* E = energies + (size_t)r * TMD_NUM_ENERGIES;
    if (pp.terms & T_ELEC) block_accumulate<PAIR_WARPS>(0.5 * e_el, E + TMD_E_ELECTROSTATICS, red);
    if (pp.terms & T_LJ) block_accumulate<PAIR_WARPS>(0.5 * e_lj, E + TMD_E_LJ, red);
    if (pp.terms & T_REP) block_accumulate<PAIR_WARPS>(0.5 * e_rep, E + TMD_E_REPULSION, red);
    if (pp.terms & T_REPCG) block_accumulate<PAIR_WARPS>(0.5 * e_cg, E + TMD_E_REPULSIONCG, red);
  }
}
template <bool ENERGY, bool PERIODIC>
__global__ void __launch_bounds__(PAIR_WARPS * 32)
k_pair_f64(DeviceState S, DeviceState64 D, double* __restrict__ forces, double* __restrict__ energies) {
  pair_f64_body<ENERGY, PERIODIC, false>(S, D, forces, energies);
}
// particle-mesh Ewald contexts (periodic only): the same rows with the real-space Ewald electrostatics
template <bool ENERGY>
__global__ void __launch_bounds__(PAIR_WARPS * 32)
k_ewpair64(DeviceState S, DeviceState64 D, double* __restrict__ forces, double* __restrict__ energies) {
  pair_f64_body<ENERGY, true, true>(S, D, forces, energies);
}

// k_export_pairs with the fp64 decision.
__global__ void k_export_pairs_f64(DeviceState S, DeviceState64 D, int r, int* __restrict__ out, long long capacity,
                                   unsigned long long* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (k >= S.natoms) return;
  const int periodic = S.grid[r].periodic;
  const size_t base = (size_t)r * S.natoms;
  const Rec64* xq = D.xq_s + (size_t)r * (S.natoms + 1);
  const int* perm = S.perm + base;
  const int* row = S.nbr + (base + k) * (size_t)S.row_cap;
  const int n = S.nnbr[base + k];
  const Rec64 pi = xq[k];
  const int oi = perm[k];
  const double Lx = D.L[3 * r], Ly = D.L[3 * r + 1], Lz = D.L[3 * r + 2];
  const unsigned lt = (1u << lane) - 1u;
  for (int e0 = 0; e0 < n; e0 += 32) {
    const int e = e0 + lane;
    bool ok = false;
    int oj = 0;
    if (e < n) {
      const int j = row[e] & 0xffffff;
      double wx, wy, wz;
      const double s = periodic ? pair_s64<true>(pi, xq[j], Lx, Ly, Lz, wx, wy, wz)
                                : pair_s64<false>(pi, xq[j], Lx, Ly, Lz, wx, wy, wz);
      oj = perm[j];
      ok = s <= D.pp.s_max && oi < oj;
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    unsigned long long b = 0;
    if (lane == 0 && m) b = atomicAdd(count, (unsigned long long)__popc(m));
    b = __shfl_sync(0xffffffffu, b, 0);
    if (ok) {
      const unsigned long long slot = b + __popc(m & lt);
      if ((long long)slot < capacity) {
        out[slot * 2 + 0] = oi;
        out[slot * 2 + 1] = oj;
      }
    }
  }
}

}  // namespace tmd
