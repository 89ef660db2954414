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
//   k_bonded_terms_f64 / k_bonded_sum_f64   bonded.cuh's two passes on fp64 rows
//   k_vv_first_f64 / k_vv_second_f64 / k_kinetic_f64   integrate.cuh in fp64
#pragma once
#include "bonded.cuh"
#include "context.cuh"
#include "integrate.cuh"
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

// ---- bonded terms: bonded.cuh's layout and fixed-order sum on fp64 positions and rows -------------
struct BondedTables64 {
  const int* atom_ptr;
  const int* entries;
  BondedSetT<double> bonds, angles, torsions[2], pairs14;
  CmapSet cmap;
  BondedSetT<double> ub;
};

__device__ __forceinline__ Vec3d load3d(const double* p, size_t atom) {
  return {p[atom * 3 + 0], p[atom * 3 + 1], p[atom * 3 + 2]};
}
// Minimum-image difference with the reference's fp64 rounding (decisions and values alike).
__device__ __forceinline__ Vec3d delta64(Vec3d a, Vec3d b, int periodic, const double* L) {
  Vec3d d = {sub_rn(a.x, b.x), sub_rn(a.y, b.y), sub_rn(a.z, b.z)};
  if (periodic) {
    d.x = min_image64(d.x, L[0]);
    d.y = min_image64(d.y, L[1]);
    d.z = min_image64(d.z, L[2]);
  }
  return d;
}

__device__ __forceinline__ bool bonded_term_f64(const DeviceState& S, const DeviceState64& D, const BondedTables64& T,
                                                const double* __restrict__ pos, int r, int kind, int t, TermForces& o) {
  const size_t base = (size_t)r * S.natoms;
  const int periodic = S.grid[r].periodic;
  const double* L = D.L + 3 * r;
  if (kind == BK_BOND || kind == BK_UREY_BRADLEY) {  // Urey-Bradley: k_ub (r13 - s0)^2, no cutoff filter (bonded.cuh)
    const BondedSetT<double>& B = kind == BK_BOND ? T.bonds : T.ub;
    const int i = B.idx[2 * t], j = B.idx[2 * t + 1];
    o.n = 2, o.atom[0] = i, o.atom[1] = j;
    const Vec3d d = delta64(load3d(pos, base + i), load3d(pos, base + j), periodic, L);
    const double dist = sqrt_rn(norm2_ref(d.x, d.y, d.z));
    if (kind == BK_BOND && D.pp.has_cutoff && !(dist <= D.pp.cutoff)) return false;  // forces.py:128-136, the fp64 decision
    double dedr;
    bond_term<double>(dist, B.prm[2 * t], B.prm[2 * t + 1], o.e, dedr);
    const Vec3d fv = (dedr / dist) * d;
    o.f[0] = {-fv.x, -fv.y, -fv.z};
    o.f[1] = fv;
    return true;
  }
  if (kind == BK_ANGLE) {
    const int a0 = T.angles.idx[3 * t], a1 = T.angles.idx[3 * t + 1], a2 = T.angles.idx[3 * t + 2];
    o.n = 3, o.atom[0] = a0, o.atom[1] = a1, o.atom[2] = a2;
    const Vec3d p1 = load3d(pos, base + a1);
    const Vec3d r21 = delta64(load3d(pos, base + a0), p1, periodic, L);
    const Vec3d r23 = delta64(load3d(pos, base + a2), p1, periodic, L);
    o.e = angle_term<double>(r21, r23, T.angles.prm[2 * t], T.angles.prm[2 * t + 1], o.f[0], o.f[1], o.f[2]);
    return true;
  }
  if (kind == BK_DIHEDRAL || kind == BK_IMPROPER) {
    const BondedSetT<double>& B = T.torsions[kind == BK_IMPROPER];
    o.n = 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) o.atom[k] = B.idx[4 * t + k];
    const Vec3d p0 = load3d(pos, base + o.atom[0]), p1 = load3d(pos, base + o.atom[1]);
    const Vec3d p2 = load3d(pos, base + o.atom[2]), p3 = load3d(pos, base + o.atom[3]);
    const TorsionGeom<double> g = torsion_geom(delta64(p0, p1, periodic, L), delta64(p1, p2, periodic, L), delta64(p2, p3, periodic, L));
    double e = 0., coef = 0.;
    for (int m = B.term_ptr[t]; m < B.term_ptr[t + 1]; ++m)
      torsion_term<double>(g.phi, B.terms[3 * m], B.terms[3 * m + 1], B.terms[3 * m + 2], B.amber, e, coef);
    torsion_forces(g, coef, o.f[0], o.f[1], o.f[2], o.f[3]);
    o.e = e;
    return true;
  }
  if (kind == BK_CMAP) {
    o.n = 5;
#pragma unroll
    for (int k = 0; k < 5; ++k) o.atom[k] = T.cmap.idx[5 * t + k];
    const Vec3d p0 = load3d(pos, base + o.atom[0]), p1 = load3d(pos, base + o.atom[1]), p2 = load3d(pos, base + o.atom[2]);
    const Vec3d p3 = load3d(pos, base + o.atom[3]), p4 = load3d(pos, base + o.atom[4]);
    o.e = cmap_term(T.cmap, t, delta64(p0, p1, periodic, L), delta64(p1, p2, periodic, L), delta64(p2, p3, periodic, L),
                    delta64(p3, p4, periodic, L), o.f);
    return true;
  }
  // BK_PAIR14 (forces.py:185-236): LJ/scnb with no cutoff or switch, Coulomb/scee, never RF
  const int i = T.pairs14.idx[2 * t], j = T.pairs14.idx[2 * t + 1];
  o.n = 2, o.atom[0] = i, o.atom[1] = j;
  const Vec3d d = delta64(load3d(pos, base + i), load3d(pos, base + j), periodic, L);
  const double dist = sqrt_rn(norm2_ref(d.x, d.y, d.z));
  const double rinv = 1.0 / dist;
  const double* prm = T.pairs14.prm + 4 * t;  // A, B, scnb, scee
  double dedr = 0.;
  if (D.pp.terms & T_LJ) {
    const double r2 = rinv * rinv, r6 = r2 * r2 * r2;
    const double a12 = prm[0] * r6 * r6, b6 = prm[1] * r6;
    o.e = (a12 - b6) / prm[2];
    dedr += (6.0 * b6 - 12.0 * a12) * rinv / prm[2];
  }
  if (D.pp.terms & T_ELEC) {
    const double e = D.q[i] * D.q[j] * rinv / prm[3];
    o.e2 = e;
    dedr -= e * rinv;
  }
  const Vec3d fv = (dedr * rinv) * d;
  o.f[0] = {-fv.x, -fv.y, -fv.z};
  o.f[1] = fv;
  return true;
}

__device__ __forceinline__ void bonded_energy_reduce64(const DeviceState64& D, const BondedTables64& T, int r,
                                                       const BondedEnergies& E, double* __restrict__ energies, double* red) {
  double* Eo = energies + (size_t)r * TMD_NUM_ENERGIES;
  if (T.bonds.n) block_accumulate<BONDED_THREADS / 32>(E.bond, Eo + TMD_E_BONDS, red);
  if (T.angles.n || T.ub.n) block_accumulate<BONDED_THREADS / 32>(E.angle, Eo + TMD_E_ANGLES, red);
  if (T.torsions[0].n || T.cmap.n) block_accumulate<BONDED_THREADS / 32>(E.dih, Eo + TMD_E_DIHEDRALS, red);
  if (T.torsions[1].n) block_accumulate<BONDED_THREADS / 32>(E.imp, Eo + TMD_E_IMPROPERS, red);
  if (T.pairs14.n) {
    if (D.pp.terms & T_LJ) block_accumulate<BONDED_THREADS / 32>(E.lj, Eo + TMD_E_LJ, red);
    if (D.pp.terms & T_ELEC) block_accumulate<BONDED_THREADS / 32>(E.el, Eo + TMD_E_ELECTROSTATICS, red);
  }
}

__global__ void __launch_bounds__(BONDED_THREADS)
k_bonded_terms_f64(DeviceState S, DeviceState64 D, BondedTables64 T, TermLayout lay, const double* __restrict__ pos,
                   double* __restrict__ energies, double* __restrict__ term_f) {
  const int r = blockIdx.y;
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  BondedEnergies E;
  if (g < lay.nterms) {
    int kind = BK_KINDS - 1;
#pragma unroll
    for (int k = BK_KINDS - 2; k >= 0; --k)
      if (g < lay.first[k + 1]) kind = k;
    const int t = g - lay.first[kind];
    TermForces o;
    const bool acts = bonded_term_f64(S, D, T, pos, r, kind, t, o);
    double* out = term_f + ((size_t)r * lay.nslots + lay.slot0[kind] + (size_t)t * o.n) * 3;
#pragma unroll
    for (int k = 0; k < 5; ++k)
      if (k < o.n) {
        out[3 * k + 0] = acts ? o.f[k].x : 0.0;
        out[3 * k + 1] = acts ? o.f[k].y : 0.0;
        out[3 * k + 2] = acts ? o.f[k].z : 0.0;
      }
    if (acts) book_energy(E, kind, o);
  }
  if (energies) {
    __shared__ double red[BONDED_THREADS / 32];
    bonded_energy_reduce64(D, T, r, E, energies, red);
  }
}

// forces += the atom's term forces in the order of its list (after the pair kernel's plain store)
__global__ void __launch_bounds__(BONDED_THREADS)
k_bonded_sum_f64(DeviceState S, BondedTables64 T, TermLayout lay, const double* __restrict__ term_f, double* __restrict__ forces) {
  const int r = blockIdx.y;
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= S.natoms) return;
  const double* tf = term_f + (size_t)r * lay.nslots * 3;
  const int p1 = T.atom_ptr[a + 1];
  if (p1 == T.atom_ptr[a]) return;
  Vec3d f = {0., 0., 0.};
  for (int p = T.atom_ptr[a]; p < p1; ++p) {
    int kind, slot, t;
    bonded_unpack((unsigned)T.entries[p], kind, slot, t);
    const double* v = tf + ((size_t)lay.slot0[kind] + (size_t)t * term_arity(kind) + slot) * 3;
    f.x += v[0];
    f.y += v[1];
    f.z += v[2];
  }
  double* out = forces + ((size_t)r * S.natoms + a) * 3;
  out[0] += f.x;
  out[1] += f.y;
  out[2] += f.z;
}

// ---- integrator (integrator.py:61-74), the reference's operation order in fp64 ---------------------
// pos += vel*dt + ((0.5*a)*dt)*dt ;  vel += (0.5*dt)*a ;  a = F/m
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_first_f64(int natoms, unsigned long long* counters, double* __restrict__ pos, double* __restrict__ vel,
               const double* __restrict__ forces, const double* __restrict__ masses, double dt, double hdt) {
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) counters[1] += 1;  // Philox position of this step
  if (i >= natoms) return;
  const double m = masses[i];
  const size_t a = ((size_t)r * natoms + i) * 3;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double acc = div_rn(forces[a + d], m);
    const double v = vel[a + d];
    const double drift = add_rn(mul_rn(v, dt), mul_rn(mul_rn(mul_rn(0.5, acc), dt), dt));
    pos[a + d] = add_rn(pos[a + d], drift);
    vel[a + d] = add_rn(v, mul_rn(hdt, acc));
  }
}

// three fp64 N(0,1) draws for (atom slot, step): two Philox4x32-10 blocks of the same stream as normal3
// (the second with the top counter bit set), 53-bit uniforms, Box-Muller in fp64
__device__ __forceinline__ double u53(unsigned hi, unsigned lo) {
  return ((double)(((unsigned long long)(hi >> 5) << 26) | (lo >> 6)) + 0.5) * (1.0 / 9007199254740992.0);
}
__device__ __forceinline__ void normal3_f64(uint64_t seed, uint64_t step, uint64_t slot, double out[3]) {
  const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
  const uint4 u = philox4x32_10(make_uint4((unsigned)slot, (unsigned)(slot >> 32), (unsigned)step, (unsigned)(step >> 32)), key);
  const uint4 w = philox4x32_10(make_uint4((unsigned)slot, (unsigned)(slot >> 32) | 0x80000000u, (unsigned)step, (unsigned)(step >> 32)), key);
  const double two_pi = 6.283185307179586;
  const double r0 = sqrt(-2.0 * log(u53(u.x, u.y))), r1 = sqrt(-2.0 * log(u53(w.x, w.y)));
  double s, c;
  sincos(two_pi * u53(u.z, u.w), &s, &c);
  out[0] = r0 * c;
  out[1] = r0 * s;
  out[2] = r1 * cos(two_pi * u53(w.z, w.w));
}

// [vel += ((-gamma*vel)*dt + xi*vcoeff)]  then  vel += (0.5*dt)*(F/m)  (integrator.py:72-74, 67-69)
template <bool THERMOSTAT, bool KINETIC>
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_second_f64(int natoms, const unsigned long long* __restrict__ counters, double* __restrict__ vel,
                const double* __restrict__ forces, const double* __restrict__ masses, double dt, double hdt, double neg_gamma,
                const double* __restrict__ vcoeff, const double* __restrict__ noise, uint64_t seed, uint64_t step_offset,
                double* __restrict__ ke) {
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double ek = 0.0;
  if (i < natoms) {
    const double m = masses[i];
    const size_t slot = (size_t)r * natoms + i;
    const size_t a = slot * 3;
    double xi[3] = {0., 0., 0.};
    double vc = 0.;
    if (THERMOSTAT) {
      vc = vcoeff[i];
      if (noise) {
        xi[0] = noise[a];
        xi[1] = noise[a + 1];
        xi[2] = noise[a + 2];
      } else {
        normal3_f64(seed, step_offset + counters[1], slot, xi);
      }
    }
    double v2 = 0.;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      double v = vel[a + d];
      if (THERMOSTAT) v = add_rn(v, add_rn(mul_rn(mul_rn(neg_gamma, v), dt), mul_rn(xi[d], vc)));
      v = add_rn(v, mul_rn(hdt, div_rn(forces[a + d], m)));
      vel[a + d] = v;
      v2 += v * v;
    }
    if (KINETIC) ek = 0.5 * m * v2;
  }
  if (KINETIC) {
    __shared__ double red[INTEG_THREADS / 32];
    block_accumulate<INTEG_THREADS / 32>(ek, ke + r, red);
  }
}

__global__ void __launch_bounds__(INTEG_THREADS)
k_kinetic_f64(int natoms, const double* __restrict__ vel, const double* __restrict__ masses, double* __restrict__ ke) {
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double ek = 0.0;
  if (i < natoms) {
    const size_t a = ((size_t)r * natoms + i) * 3;
    const double vx = vel[a], vy = vel[a + 1], vz = vel[a + 2];
    ek = 0.5 * masses[i] * (vx * vx + vy * vy + vz * vz);
  }
  __shared__ double red[INTEG_THREADS / 32];
  block_accumulate<INTEG_THREADS / 32>(ek, ke + r, red);
}

}  // namespace tmd
