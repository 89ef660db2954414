// bonded.cuh -- bonded terms (K4): bonds, angles, proper/improper torsions, 1-4, CMAP correction maps, Urey-Bradley.
//
// Replaces forces.py:122-258 (+ evaluate_bonds/angles/torsion, forces.py:494-605).
//
// Two passes, deterministic: k_bonded_terms evaluates every term ONCE (one thread per term, the terms of a kind side by
// side so that warps do not diverge) and leaves the force on each of its 2-5 atoms in a per-(term, slot) buffer;
// k_bonded_sum, one thread per ATOM, walks the list of term instances the atom takes part in (CSR built once on the
// host from the topology) and adds them up in that fixed order -- no atomics, bitwise reproducible -- then adds the
// sum to the force array (or hands it to the integrator kernel that folds it in).  A protein's atom sits in ~35 term
// instances with fp64 trigonometry in each: walked serially by one thread per atom (still the layout of the
// single-kernel k_bonded_vv_second) that chain is long whatever the replica count.  A term's energy is booked when the atom in its
// slot 0 is owned.  Runs beside the pair kernel on a second stream, or after it (its plain store of the non-bonded
// force doubles as the zeroing of Forces.compute, forces.py:113-114).
#pragma once
#include <type_traits>

#include "context.cuh"
#include "pair.cuh"

namespace tmd {

constexpr int BONDED_THREADS = 128;

// kinds of term instance an atom entry can point at
enum { BK_BOND = 0, BK_ANGLE = 1, BK_DIHEDRAL = 2, BK_IMPROPER = 3, BK_PAIR14 = 4, BK_CMAP = 5, BK_UREY_BRADLEY = 6 };
constexpr int BK_KINDS = 7;

// packed atom entry: kind (3 bits) | slot in the term (3 bits) | term index (26 bits)
__host__ __device__ __forceinline__ unsigned bonded_entry(int kind, int slot, unsigned t) {
  return ((unsigned)kind << 29) | ((unsigned)slot << 26) | t;
}
__device__ __forceinline__ void bonded_unpack(unsigned ent, int& kind, int& slot, int& t) {
  kind = (int)(ent >> 29), slot = (int)((ent >> 26) & 7u), t = (int)(ent & 0x3ffffffu);
}

// P: type of the positions and parameter rows, float ("precision: single") or double ("precision: double")
template <typename P>
struct BondedTablesT {
  const int* atom_ptr;   // (natoms+1) CSR over atoms
  const int* entries;    // bonded_entry(kind, slot, term)
  BondedSetT<P> bonds, angles, torsions[2], pairs14;
  CmapSet cmap;
  BondedSetT<P> ub;  // Urey-Bradley: idx (n,2) = the ends of an angle, prm (n,2) = k_ub, s0
};

struct BoxView {
  int periodic;
  Vec3 L, invL;
};
__device__ __forceinline__ BoxView box_of(const DeviceState& S, int r) {
  const Grid* g = S.grid + r;
  BoxView b;
  b.periodic = g->periodic;
  b.L = {g->L[0], g->L[1], g->L[2]};
  b.invL = {g->invL[0], g->invL[1], g->invL[2]};
  return b;
}
__device__ __forceinline__ Vec3 load3(const float* p, size_t atom) {
  return {p[atom * 3 + 0], p[atom * 3 + 1], p[atom * 3 + 2]};
}
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

// What the bonded kernels of the two precisions do differently, on one replica; each term body is written once on top
// of it.  Arg: the kernels' argument the frame is made from (bonded_frame).  The two rinv6 round differently; each
// precision keeps the product its kernels have always formed.
template <typename P>
struct BondedFrame;
// fp32 positions: values from the fp64 difference of the fp32 coordinates, a bond's cutoff decision on the reference's
// fp32 difference.
template <>
struct BondedFrame<float> {
  using Arg = const float* __restrict__;  // charges scaled by sqrt(coulomb constant)
  using V = Vec3;
  const float* q;
  BoxView bx;
  __device__ __forceinline__ Vec3 load(const float* p, size_t atom) const { return load3(p, atom); }
  __device__ __forceinline__ Vec3d delta(Vec3 a, Vec3 b) const { return delta_f64(a, b, bx.periodic, bx.L); }
  __device__ __forceinline__ static double dist(const Vec3d& d) { return norm(d); }
  __device__ __forceinline__ static bool cutoff_on(const DeviceState& S) { return S.pp.has_cutoff; }
  __device__ __forceinline__ bool within_cutoff(const DeviceState& S, Vec3 a, Vec3 b) const {
    const Vec3 dref = delta_ref(a, b, bx.periodic, bx.L, bx.invL);
    return sqrt_rn(norm2_ref(dref.x, dref.y, dref.z)) <= S.pp.cutoff;
  }
  __device__ __forceinline__ static double rinv6(double rinv) { return rinv * rinv * rinv * rinv * rinv * rinv; }
};
// fp64 positions: the reference's fp64 rounding for the decision and the values.
template <>
struct BondedFrame<double> {
  using Arg = DeviceState64;
  using V = Vec3d;
  const double* q;  // charges scaled by sqrt(coulomb constant)
  const double* L;  // this replica's box
  int periodic, has_cutoff;
  double cutoff;
  __device__ __forceinline__ Vec3d load(const double* p, size_t atom) const { return load3d(p, atom); }
  __device__ __forceinline__ Vec3d delta(Vec3d a, Vec3d b) const { return delta64(a, b, periodic, L); }
  __device__ __forceinline__ static double dist(const Vec3d& d) { return sqrt_rn(norm2_ref(d.x, d.y, d.z)); }
  __device__ __forceinline__ bool cutoff_on(const DeviceState&) const { return has_cutoff; }
  __device__ __forceinline__ bool within_cutoff(const DeviceState&, Vec3d a, Vec3d b) const { return dist(delta(a, b)) <= cutoff; }
  __device__ __forceinline__ static double rinv6(double rinv) {
    const double r2 = rinv * rinv;
    return r2 * r2 * r2;
  }
};
__device__ __forceinline__ BondedFrame<float> bonded_frame(const DeviceState& S, const float* q, int r) {
  return {q, box_of(S, r)};
}
__device__ __forceinline__ BondedFrame<double> bonded_frame(const DeviceState& S, const DeviceState64& D, int r) {
  return {D.q, D.L + 3 * r, S.grid[r].periodic, D.pp.has_cutoff, D.pp.cutoff};
}

struct BondedEnergies {
  double bond = 0., angle = 0., dih = 0., imp = 0., lj = 0., el = 0.;
};

// Forces of term t of a kind on each of its atoms (fp64) and its energy; false if the term does not act (a bond
// beyond the cutoff).  n: atoms of the term.
struct TermForces {
  Vec3d f[5];
  double e = 0., e2 = 0.;  // e2: the Coulomb part of a 1-4 pair (e: its LJ part)
  int atom[5];
  int n = 0;
};

// CMAP correction map m at (phi, psi) [rad]: bicubic patch of the cell that holds the point (grid from -pi, spacing
// 2 pi / res, coefficients c[4a+b] of u^a v^b in the cell's unit coordinates).  E, dE/dphi, dE/dpsi; fp64.
__device__ __forceinline__ double cmap_energy(const CmapSet& C, int m, double phi, double psi, double& dphi, double& dpsi) {
  const int2 mp = C.maps[m];  // first cell, resolution
  const int n = mp.y;
  const double inv_h = (double)n * 0.15915494309189533577;  // n / (2 pi)
  const double x = (phi + 3.14159265358979323846) * inv_h, y = (psi + 3.14159265358979323846) * inv_h;
  const double fx = floor(x), fy = floor(y);
  const double u = x - fx, v = y - fy;
  int i = (int)fx % n, j = (int)fy % n;
  if (i < 0) i += n;
  if (j < 0) j += n;
  const double* c = C.coef + ((size_t)mp.x + (size_t)i * n + j) * 16;
  double e = 0., du = 0., dv = 0.;
#pragma unroll
  for (int a = 3; a >= 0; --a) {
    const double r0 = c[4 * a + 0], r1 = c[4 * a + 1], r2 = c[4 * a + 2], r3 = c[4 * a + 3];
    e = e * u + (((r3 * v + r2) * v + r1) * v + r0);
    dv = dv * u + ((3.0 * r3 * v + 2.0 * r2) * v + r1);
  }
#pragma unroll
  for (int b = 3; b >= 0; --b) du = du * v + ((3.0 * c[12 + b] * u + 2.0 * c[8 + b]) * u + c[4 + b]);
  dphi = du * inv_h;
  dpsi = dv * inv_h;
  return e;
}

// A CMAP term (a, b, c, d, e) from its four bond vectors r_k = x_k - x_(k+1): phi = dihedral(a, b, c, d),
// psi = dihedral(b, c, d, e), the two torsion force projections summed onto the five atoms.
__device__ __forceinline__ double cmap_term(const CmapSet& C, int t, const Vec3d& r01, const Vec3d& r12, const Vec3d& r23,
                                           const Vec3d& r34, Vec3d* f) {
  const TorsionGeom<double> g1 = torsion_geom(r01, r12, r23), g2 = torsion_geom(r12, r23, r34);
  double dphi, dpsi;
  const double e = cmap_energy(C, C.map_of[t], g1.phi, g2.phi, dphi, dpsi);
  Vec3d q0, q1, q2, q3;
  torsion_forces(g1, dphi, f[0], f[1], f[2], f[3]);
  torsion_forces(g2, dpsi, q0, q1, q2, q3);
  f[1] = f[1] + q0;
  f[2] = f[2] + q1;
  f[3] = f[3] + q2;
  f[4] = q3;
  return e;
}

template <typename P>
__device__ __forceinline__ bool bonded_term(const DeviceState& S, const BondedTablesT<P>& T, const BondedFrame<P>& X,
                                            const P* __restrict__ pos, size_t base, int kind, int t, TermForces& o) {
  using V = typename BondedFrame<P>::V;
  if (kind == BK_BOND || kind == BK_UREY_BRADLEY) {
    // E = k (r-r0)^2.  Bonds longer than the cutoff are skipped like the reference (forces.py:128-136); Urey-Bradley
    // terms (the ends of an angle, k_ub and s0) have no reference counterpart and are never cutoff-filtered.
    const BondedSetT<P>& B = kind == BK_BOND ? T.bonds : T.ub;
    const int i = B.idx[2 * t], j = B.idx[2 * t + 1];
    o.n = 2, o.atom[0] = i, o.atom[1] = j;
    const V pi = X.load(pos, base + i), pj = X.load(pos, base + j);
    if (kind == BK_BOND && X.cutoff_on(S) && !X.within_cutoff(S, pi, pj)) return false;  // reference decision
    const Vec3d d = X.delta(pi, pj);
    const double dist = X.dist(d);
    double dedr;
    bond_term<double>(dist, B.prm[2 * t], B.prm[2 * t + 1], o.e, dedr);
    const Vec3d fv = (dedr / dist) * d;  // force on j; i gets the opposite
    o.f[0] = {-fv.x, -fv.y, -fv.z};
    o.f[1] = fv;
    return true;
  }
  if (kind == BK_ANGLE) {
    const int a0 = T.angles.idx[3 * t], a1 = T.angles.idx[3 * t + 1], a2 = T.angles.idx[3 * t + 2];
    o.n = 3, o.atom[0] = a0, o.atom[1] = a1, o.atom[2] = a2;
    const V p1 = X.load(pos, base + a1);
    const Vec3d r21 = X.delta(X.load(pos, base + a0), p1);
    const Vec3d r23 = X.delta(X.load(pos, base + a2), p1);
    o.e = angle_term<double>(r21, r23, T.angles.prm[2 * t], T.angles.prm[2 * t + 1], o.f[0], o.f[1], o.f[2]);
    return true;
  }
  if (kind == BK_DIHEDRAL || kind == BK_IMPROPER) {
    const BondedSetT<P>& B = T.torsions[kind == BK_IMPROPER];
    o.n = 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) o.atom[k] = B.idx[4 * t + k];
    const V p0 = X.load(pos, base + o.atom[0]), p1 = X.load(pos, base + o.atom[1]);
    const V p2 = X.load(pos, base + o.atom[2]), p3 = X.load(pos, base + o.atom[3]);
    const Vec3d r12 = X.delta(p0, p1);
    const Vec3d r23 = X.delta(p1, p2);
    const Vec3d r34 = X.delta(p2, p3);
    const TorsionGeom<double> g = torsion_geom(r12, r23, r34);
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
    const V p0 = X.load(pos, base + o.atom[0]), p1 = X.load(pos, base + o.atom[1]), p2 = X.load(pos, base + o.atom[2]);
    const V p3 = X.load(pos, base + o.atom[3]), p4 = X.load(pos, base + o.atom[4]);
    o.e = cmap_term(T.cmap, t, X.delta(p0, p1), X.delta(p1, p2), X.delta(p2, p3), X.delta(p3, p4), o.f);
    return true;
  }
  // BK_PAIR14 (forces.py:185-236): LJ/scnb with no cutoff or switch, Coulomb/scee, never RF
  const int i = T.pairs14.idx[2 * t], j = T.pairs14.idx[2 * t + 1];
  o.n = 2, o.atom[0] = i, o.atom[1] = j;
  const Vec3d d = X.delta(X.load(pos, base + i), X.load(pos, base + j));
  const double dist = X.dist(d);
  const double rinv = 1.0 / dist;
  const P* prm = T.pairs14.prm + 4 * t;  // A, B, scnb, scee
  double dedr = 0.;
  if (S.pp.terms & T_LJ) {
    const double r6 = X.rinv6(rinv);
    const double a12 = prm[0] * r6 * r6, b6 = prm[1] * r6;
    o.e = (a12 - b6) / prm[2];
    dedr += (6.0 * b6 - 12.0 * a12) * rinv / prm[2];
  }
  if (S.pp.terms & T_ELEC) {
    const double e = (double)X.q[i] * (double)X.q[j] * rinv / prm[3];
    o.e2 = e;
    dedr -= e * rinv;
  }
  const Vec3d fv = (dedr * rinv) * d;
  o.f[0] = {-fv.x, -fv.y, -fv.z};
  o.f[1] = fv;
  return true;
}

__device__ __forceinline__ void book_energy(BondedEnergies& E, int kind, const TermForces& o) {
  if (kind == BK_BOND) E.bond += o.e;
  else if (kind == BK_ANGLE || kind == BK_UREY_BRADLEY) E.angle += o.e;  // Urey-Bradley energy is booked as angle energy
  else if (kind == BK_DIHEDRAL || kind == BK_CMAP) E.dih += o.e;  // CMAP energy is booked as dihedral energy
  else if (kind == BK_IMPROPER) E.imp += o.e;
  else E.lj += o.e, E.el += o.e2;
}

// Sum of the bonded forces on atom a of replica r (fp64), every term of the atom re-evaluated in this thread; energies
// booked by the atom in slot 0 of each term.  (k_bonded_vv_second: systems whose bonded kernel is not forked.)
__device__ __forceinline__ Vec3d bonded_force_on_atom(const DeviceState& S, const BondedTablesT<float>& T, const float* __restrict__ q_scaled,
                                                      const float* __restrict__ pos, int r, int a, BondedEnergies& E) {
  const size_t base = (size_t)r * S.natoms;
  const BondedFrame<float> X = bonded_frame(S, q_scaled, r);
  Vec3d f = {0., 0., 0.};
  for (int p = T.atom_ptr[a]; p < T.atom_ptr[a + 1]; ++p) {
    int kind, slot, t;
    bonded_unpack((unsigned)T.entries[p], kind, slot, t);
    TermForces o;
    if (!bonded_term(S, T, X, pos, base, kind, t, o)) continue;
    f = f + (slot == 0 ? o.f[0] : (slot == 1 ? o.f[1] : (slot == 2 ? o.f[2] : (slot == 3 ? o.f[3] : o.f[4]))));
    if (slot == 0) book_energy(E, kind, o);
  }
  return f;
}

// Where the force of (kind, term, slot) sits in the per-term buffer: slots of a kind side by side
struct TermLayout {
  int first[BK_KINDS];  // first term index (over all kinds, in the order of the BK_ enum) of each kind
  int slot0[BK_KINDS];  // first buffer slot of each kind
  int nterms, nslots;
};
__host__ __device__ __forceinline__ int term_arity(int kind) {
  return kind == BK_ANGLE ? 3 : (kind == BK_DIHEDRAL || kind == BK_IMPROPER ? 4 : (kind == BK_CMAP ? 5 : 2));
}

// block-level reduction of the bonded energies into the per-replica slots
template <typename P>
__device__ __forceinline__ void bonded_energy_reduce(const DeviceState& S, const BondedTablesT<P>& T, int r, const BondedEnergies& E,
                                                     double* __restrict__ energies, double* red) {
  double* Eo = energies + (size_t)r * TMD_NUM_ENERGIES;
  if (T.bonds.n) block_accumulate<BONDED_THREADS / 32>(E.bond, Eo + TMD_E_BONDS, red);
  if (T.angles.n || T.ub.n) block_accumulate<BONDED_THREADS / 32>(E.angle, Eo + TMD_E_ANGLES, red);
  if (T.torsions[0].n || T.cmap.n) block_accumulate<BONDED_THREADS / 32>(E.dih, Eo + TMD_E_DIHEDRALS, red);
  if (T.torsions[1].n) block_accumulate<BONDED_THREADS / 32>(E.imp, Eo + TMD_E_IMPROPERS, red);
  if (T.pairs14.n) {
    if (S.pp.terms & T_LJ) block_accumulate<BONDED_THREADS / 32>(E.lj, Eo + TMD_E_LJ, red);
    if (S.pp.terms & T_ELEC) block_accumulate<BONDED_THREADS / 32>(E.el, Eo + TMD_E_ELECTROSTATICS, red);
  }
}

// Pass 1: one thread per term.  Terms none of whose atoms this rank owns are skipped (decomposed runs, fp32 only).
template <typename P>
__global__ void __launch_bounds__(BONDED_THREADS)
k_bonded_terms(DeviceState S, BondedTablesT<P> T, TermLayout lay, typename BondedFrame<P>::Arg arg, const P* __restrict__ pos,
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
    const size_t base = (size_t)r * S.natoms;
    TermForces o;
    const bool acts = bonded_term(S, T, bonded_frame(S, arg, r), pos, base, kind, t, o);
    bool mine = S.own_all, books = S.own_all;
    if (!S.own_all) {
#pragma unroll
      for (int k = 0; k < 5; ++k) mine |= k < o.n && o.atom[k] >= S.own_lo && o.atom[k] < S.own_lo + S.own_n;
      books = o.atom[0] >= S.own_lo && o.atom[0] < S.own_lo + S.own_n;
    }
    if (mine) {
      double* out = term_f + ((size_t)r * lay.nslots + lay.slot0[kind] + (size_t)t * o.n) * 3;
#pragma unroll
      for (int k = 0; k < 5; ++k)
        if (k < o.n) {
          out[3 * k + 0] = acts ? o.f[k].x : 0.0;
          out[3 * k + 1] = acts ? o.f[k].y : 0.0;
          out[3 * k + 2] = acts ? o.f[k].z : 0.0;
        }
    }
    if (acts && books) book_energy(E, kind, o);
  }
  if (energies) {
    __shared__ double red[BONDED_THREADS / 32];
    bonded_energy_reduce(S, T, r, E, energies, red);
  }
}

// Pass 2: one thread per owned atom adds up its term instances in the order of its list.
template <typename P>
__global__ void __launch_bounds__(BONDED_THREADS)
k_bonded_sum(DeviceState S, BondedTablesT<P> T, TermLayout lay, const double* __restrict__ term_f, P* __restrict__ forces,
             double* __restrict__ scratch) {
  const int r = blockIdx.y;
  const int a = S.own_lo + blockIdx.x * blockDim.x + threadIdx.x;  // owned atoms only
  if (a >= S.own_lo + S.own_n) return;
  const size_t base = (size_t)r * S.natoms;
  const double* tf = term_f + (size_t)r * lay.nslots * 3;
  Vec3d f = {0., 0., 0.};
  const int p1 = T.atom_ptr[a + 1];
  for (int p = T.atom_ptr[a]; p < p1; ++p) {
    int kind, slot, t;
    bonded_unpack((unsigned)T.entries[p], kind, slot, t);
    const double* v = tf + ((size_t)lay.slot0[kind] + (size_t)t * term_arity(kind) + slot) * 3;
    f.x += v[0];
    f.y += v[1];
    f.z += v[2];
  }
  if constexpr (std::is_same<P, float>::value) {  // an fp64 context has neither the side stream nor the cluster path
    if (scratch) {
      // beside the pair kernel on another stream: the fp64 sums go to a scratch buffer, k_add_bonded (or the
      // integrator kernel) folds them into the forces afterwards (same single rounding)
      double* o = scratch + (base + a) * 3;
      o[0] = f.x;
      o[1] = f.y;
      o[2] = f.z;
      return;
    }
    if (S.cl.on) {
      // cluster path: the pair forces sit in slot order; this kernel brings them home and adds its own sums
      const float4 pf = S.cl.f[(size_t)r * (S.cl.slots + 1) + S.cl.inv[base + a]];
      float* out = forces + (base + a) * 3;
      out[0] = (float)((double)pf.x + f.x);
      out[1] = (float)((double)pf.y + f.y);
      out[2] = (float)((double)pf.z + f.z);
      return;
    }
  }
  if (p1 > T.atom_ptr[a]) {
    P* out = forces + (base + a) * 3;
    out[0] = (P)((double)out[0] + f.x);
    out[1] = (P)((double)out[1] + f.y);
    out[2] = (P)((double)out[2] + f.z);
  }
}

// forces += bonded sums of k_bonded_sum's scratch mode (owned atoms), rounded once like the in-place path
__global__ void __launch_bounds__(BONDED_THREADS)
k_add_bonded(int natoms, int lo, int cnt, float* __restrict__ forces, const double* __restrict__ scratch) {
  const int a = lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= lo + cnt) return;
  const size_t e = ((size_t)blockIdx.y * natoms + a) * 3;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const double s = scratch[e + d];
    if (s != 0.0) forces[e + d] = (float)((double)forces[e + d] + s);
  }
}

}  // namespace tmd
