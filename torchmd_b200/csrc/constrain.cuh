// constrain.cuh -- holonomic constraints: rigid water and bonds to hydrogen (tmd_set_constraints).
//
// A constraint group is a water (3 atoms, the O-H, O-H and H-H distances: analytic SETTLE) or a SHAKE cluster
// (one heavy atom and the 1-4 hydrogens bonded to it).  Groups are disjoint, so every group is one thread's work with no
// communication.  RATTLE around the velocity Verlet step (tmd_b200.cu, tmd_md_steps):
//   kick + drift  ->  k_constrain_pos (SETTLE / SHAKE against the pre-drift bond vectors, vel += dx/dt, and in
//                     tmd_md_steps the preparation of the force call)
//   force call    ->  Langevin + second half-kick  ->  k_constrain_vel (velocity projection, kinetic energy)
// All arithmetic is fp64 in both precisions; each coordinate or velocity is rounded once on the way out.
// Bond vectors use the minimum image (as the bonded terms do): the group is solved in coordinates relative to its
// first atom, and each atom gets its own displacement added in its own image.
#pragma once
#include "integrate.cuh"
#include "neighbor.cuh"

namespace tmd {

constexpr int CON_THREADS = 128;
constexpr int CON_MAX_ATOMS = 5;   // heavy atom + up to 4 hydrogens
constexpr int CON_MAX_CONS = 4;    // constraints per group (a water has 3)
constexpr int SHAKE_MAX_ITER = 1000;
constexpr double SHAKE_TOL = 1e-14;  // relative tolerance on |r|^2 - d^2: |r - d| <= 5e-15 d at convergence

struct CGroup {
  int atom[CON_MAX_ATOMS];  // atom[0]: the heavy atom, the anchor of the unwrapped frame
  int na, nc;
  int ca[CON_MAX_CONS], cb[CON_MAX_CONS];  // local atom indices of each constraint
  double d[CON_MAX_CONS];                  // constrained distances (A)
};

struct ConstraintTables {
  int ngroups;
  const CGroup* g;
  int nfree;                // atoms in no group (kinetic energy work items)
  const int* free_atoms;
  const double* L;          // (R,3) box lengths; an entry of 0 means no periodicity along that axis
};

__device__ __forceinline__ double con_image(double d, double L) { return L > 0.0 ? d - L * rint(d / L) : d; }

// positions of a group's atoms relative to atom[0], minimum image: small numbers whatever the image or the
// distance from the origin, so the fp64 solve resolves the distances to ~1e-16 A
template <typename T>
__device__ __forceinline__ void con_load(const CGroup& G, const T* __restrict__ x, size_t base, const double* L, double out[][3]) {
  const size_t a0 = (base + G.atom[0]) * 3;
  for (int k = 0; k < 3; ++k) out[0][k] = 0.0;
  for (int j = 1; j < G.na; ++j) {
    const size_t a = (base + G.atom[j]) * 3;
    for (int k = 0; k < 3; ++k) out[j][k] = con_image((double)x[a + k] - (double)x[a0 + k], L ? L[k] : 0.0);
  }
}

// SHAKE (Ryckaert et al. 1977) to convergence: moves the unconstrained positions `x` along the reference bond
// vectors of `ref` until every |x_a - x_b| = d.  Returns the iterations taken (SHAKE_MAX_ITER: not converged).
__device__ __forceinline__ int con_shake(const CGroup& G, const double im[], const double ref[][3], double x[][3]) {
  for (int it = 0; it < SHAKE_MAX_ITER; ++it) {
    bool done = true;
    for (int c = 0; c < G.nc; ++c) {
      const int a = G.ca[c], b = G.cb[c];
      double s[3], rr[3];
      for (int k = 0; k < 3; ++k) {
        s[k] = x[a][k] - x[b][k];
        rr[k] = ref[a][k] - ref[b][k];
      }
      const double d2 = G.d[c] * G.d[c];
      const double diff = d2 - (s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
      if (fabs(diff) <= SHAKE_TOL * d2) continue;
      done = false;
      const double g = diff / (2.0 * (im[a] + im[b]) * (s[0] * rr[0] + s[1] * rr[1] + s[2] * rr[2]));
      for (int k = 0; k < 3; ++k) {
        x[a][k] += g * im[a] * rr[k];
        x[b][k] -= g * im[b] * rr[k];
      }
    }
    if (done) return it;
  }
  return SHAKE_MAX_ITER;
}

// Analytic SETTLE (Miyamoto & Kollman, J. Comput. Chem. 13, 952 (1992)) for a water: O = atom 0, H = atoms 1, 2 of
// equal mass, d[0] = O-H, d[2] = H-H.  `ref`: the reference positions, `x`: the unconstrained new positions, both
// relative to their own oxygen; on return `x` holds the constrained positions (same frame).  The result is the exact
// solution of the SHAKE equations (displacements along the reference bond vectors), in closed form.  Returns false if
// the geometry has no solution (a step far too long).
__device__ __forceinline__ bool con_settle(const CGroup& G, double mO, double mH, const double ref[][3], double x[][3]) {
  const double wohh = mO + 2.0 * mH;
  const double rc = 0.5 * G.d[2];
  const double h = sqrt(G.d[0] * G.d[0] - rc * rc);
  const double ra = 2.0 * mH * h / wohh, rb = h - ra;  // canonical water: O (0, ra), H (-+rc, -rb), centre of mass at 0
  double com[3], a1[3], b1[3], c1[3], b0[3], c0[3];
  for (int k = 0; k < 3; ++k) {
    com[k] = (mO * x[0][k] + mH * (x[1][k] + x[2][k])) / wohh;
    a1[k] = x[0][k] - com[k];
    b1[k] = x[1][k] - com[k];
    c1[k] = x[2][k] - com[k];
    b0[k] = ref[1][k] - ref[0][k];
    c0[k] = ref[2][k] - ref[0][k];
  }
  // frame: z normal to the reference plane, x normal to z and the new oxygen
  double ez[3] = {b0[1] * c0[2] - b0[2] * c0[1], b0[2] * c0[0] - b0[0] * c0[2], b0[0] * c0[1] - b0[1] * c0[0]};
  double ex[3] = {a1[1] * ez[2] - a1[2] * ez[1], a1[2] * ez[0] - a1[0] * ez[2], a1[0] * ez[1] - a1[1] * ez[0]};
  double ey[3] = {ez[1] * ex[2] - ez[2] * ex[1], ez[2] * ex[0] - ez[0] * ex[2], ez[0] * ex[1] - ez[1] * ex[0]};
  const double nx = 1.0 / sqrt(ex[0] * ex[0] + ex[1] * ex[1] + ex[2] * ex[2]);
  const double ny = 1.0 / sqrt(ey[0] * ey[0] + ey[1] * ey[1] + ey[2] * ey[2]);
  const double nz = 1.0 / sqrt(ez[0] * ez[0] + ez[1] * ez[1] + ez[2] * ez[2]);
  for (int k = 0; k < 3; ++k) {
    ex[k] *= nx;
    ey[k] *= ny;
    ez[k] *= nz;
  }
  auto dot3 = [](const double* u, const double* v) { return u[0] * v[0] + u[1] * v[1] + u[2] * v[2]; };
  const double xb0 = dot3(ex, b0), yb0 = dot3(ey, b0), xc0 = dot3(ex, c0), yc0 = dot3(ey, c0);
  const double za1 = dot3(ez, a1);
  const double xb1 = dot3(ex, b1), yb1 = dot3(ey, b1), zb1 = dot3(ez, b1);
  const double xc1 = dot3(ex, c1), yc1 = dot3(ey, c1), zc1 = dot3(ez, c1);
  const double sinphi = za1 / ra;
  const double t = 1.0 - sinphi * sinphi;
  if (!(t > 0.0)) return false;
  const double cosphi = sqrt(t);
  const double sinpsi = (zb1 - zc1) / (2.0 * rc * cosphi);
  const double u = 1.0 - sinpsi * sinpsi;
  if (!(u > 0.0)) return false;
  const double cospsi = sqrt(u);
  const double ya2 = ra * cosphi;
  const double xb2 = -rc * cospsi;
  const double t1 = -rb * cosphi, t2 = rc * sinpsi * sinphi;
  const double yb2 = t1 - t2, yc2 = t1 + t2;
  // rotation about z that keeps the momentum balance of the reference frame
  const double alpha = xb2 * (xb0 - xc0) + yb0 * yb2 + yc0 * yc2;
  const double beta = xb2 * (yc0 - yb0) + xb0 * yb2 + xc0 * yc2;
  const double gamma = xb0 * yb1 - xb1 * yb0 + xc0 * yc1 - xc1 * yc0;
  const double ab2 = alpha * alpha + beta * beta;
  const double disc = ab2 - gamma * gamma;
  if (!(disc >= 0.0)) return false;
  const double sinthe = (alpha * gamma - beta * sqrt(disc)) / ab2;
  const double costhe = sqrt(1.0 - sinthe * sinthe);
  const double p[3][3] = {{-ya2 * sinthe, ya2 * costhe, za1},
                          {xb2 * costhe - yb2 * sinthe, xb2 * sinthe + yb2 * costhe, zb1},
                          {-xb2 * costhe - yc2 * sinthe, -xb2 * sinthe + yc2 * costhe, zc1}};
  for (int j = 0; j < 3; ++j)
    for (int k = 0; k < 3; ++k) x[j][k] = com[k] + ex[k] * p[j][0] + ey[k] * p[j][1] + ez[k] * p[j][2];
  return true;
}

__device__ __forceinline__ bool con_is_water(const CGroup& G) { return G.na == 3 && G.nc == 3; }

// Position constraint of every group: SETTLE for waters, SHAKE for X-H clusters.  `ref`: the positions the bond
// directions are taken from (the pre-drift positions inside a step; the positions themselves for a projection: then
// ref == pos, hence no __restrict__ on either).  With `vel`, each atom's velocity gets its displacement over dt
// (inv_dt = 1/dt).  `fail` is set when a group has no solution or did not converge.
// PREP (fp32, tmd_md_steps): the unconstrained atoms are work items too, and every atom ends with prepare_atom
// (neighbor.cuh), so the force call that follows finds its preparation done, as after k_vv_first_prepare.
template <typename T, bool PREP>
__global__ void __launch_bounds__(CON_THREADS)
k_constrain_pos(int natoms, ConstraintTables C, T* pos, const T* ref, T* __restrict__ vel, const T* __restrict__ masses,
                double inv_dt, int* __restrict__ fail, DeviceState S) {
  const int r = blockIdx.y;
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int parity = PREP ? (int)(S.counters[0] & 1ull) : 0;
  if (PREP && w == 0) S.flags[r * F_COUNT + F_REBUILD0 + (parity ^ 1)] = 0;  // as k_prepare
  const size_t base = (size_t)r * natoms;
  if (w >= C.ngroups) {
    if (PREP && w < C.ngroups + C.nfree) {
      const int i = C.free_atoms[w - C.ngroups];
      const size_t a = (base + i) * 3;
      prepare_atom(S, r, i, parity, (float)pos[a], (float)pos[a + 1], (float)pos[a + 2]);
    }
    return;
  }
  const CGroup G = C.g[w];
  const double* L = C.L ? C.L + (size_t)r * 3 : nullptr;
  double x[CON_MAX_ATOMS][3], x0[CON_MAX_ATOMS][3], q[CON_MAX_ATOMS][3], im[CON_MAX_ATOMS];
  con_load(G, pos, base, L, x);
  con_load(G, ref, base, L, q);
  for (int j = 0; j < G.na; ++j) {
    im[j] = 1.0 / (double)masses[G.atom[j]];
    for (int k = 0; k < 3; ++k) x0[j][k] = x[j][k];
  }
  const bool ok = con_is_water(G) ? con_settle(G, (double)masses[G.atom[0]], (double)masses[G.atom[1]], q, x)
                                  : con_shake(G, im, q, x) < SHAKE_MAX_ITER;
  if (!ok) *fail = 1;
  for (int j = 0; j < G.na; ++j) {
    const size_t a = (base + G.atom[j]) * 3;
    T xn[3];
    for (int k = 0; k < 3; ++k) {
      const double dx = x[j][k] - x0[j][k];
      xn[k] = (T)((double)pos[a + k] + dx);
      pos[a + k] = xn[k];
      if (vel) vel[a + k] = (T)((double)vel[a + k] + dx * inv_dt);
    }
    if (PREP) prepare_atom(S, r, G.atom[j], parity, (float)xn[0], (float)xn[1], (float)xn[2]);
  }
}

// Velocity constraint (RATTLE's second half): the velocities are projected so that every constrained bond has
// no relative velocity along it.  The group's multipliers solve M lambda = -G v exactly: in closed form for a water
// (SETTLE's velocity counterpart), by Gaussian elimination with partial pivoting for a cluster (at most 4 x 4), M_kl = sum_i G_k(i).G_l(i) / m_i.  With `ke`, threads past the groups add the
// kinetic energy of the unconstrained atoms, so one launch gives the step's kinetic energy after the projection.
template <typename T, bool KINETIC>
__global__ void __launch_bounds__(CON_THREADS)
k_constrain_vel(int natoms, ConstraintTables C, const T* __restrict__ pos, T* __restrict__ vel, const T* __restrict__ masses,
                double* __restrict__ ke) {
  const int r = blockIdx.y;
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t base = (size_t)r * natoms;
  double ek = 0.0;
  if (w < C.ngroups) {
    const CGroup G = C.g[w];
    const double* L = C.L ? C.L + (size_t)r * 3 : nullptr;
    double x[CON_MAX_ATOMS][3], v[CON_MAX_ATOMS][3], im[CON_MAX_ATOMS];
    con_load(G, pos, base, L, x);
    for (int j = 0; j < G.na; ++j) {
      im[j] = 1.0 / (double)masses[G.atom[j]];
      const size_t a = (base + G.atom[j]) * 3;
      for (int k = 0; k < 3; ++k) v[j][k] = (double)vel[a + k];
    }
    double rv[CON_MAX_CONS][3], M[CON_MAX_CONS][CON_MAX_CONS + 1];
    for (int c = 0; c < G.nc; ++c)
      for (int k = 0; k < 3; ++k) rv[c][k] = x[G.ca[c]][k] - x[G.cb[c]][k];
    for (int c = 0; c < G.nc; ++c) {
      for (int e = 0; e < G.nc; ++e) {
        // G_c(i) = +rv[c] at ca, -rv[c] at cb
        double s = 0.0;
        const double dd = rv[c][0] * rv[e][0] + rv[c][1] * rv[e][1] + rv[c][2] * rv[e][2];
        if (G.ca[c] == G.ca[e]) s += im[G.ca[c]] * dd;
        if (G.ca[c] == G.cb[e]) s -= im[G.ca[c]] * dd;
        if (G.cb[c] == G.ca[e]) s -= im[G.cb[c]] * dd;
        if (G.cb[c] == G.cb[e]) s += im[G.cb[c]] * dd;
        M[c][e] = s;
      }
      const int a = G.ca[c], b = G.cb[c];
      M[c][G.nc] = -(rv[c][0] * (v[a][0] - v[b][0]) + rv[c][1] * (v[a][1] - v[b][1]) + rv[c][2] * (v[a][2] - v[b][2]));
    }
    const int n = G.nc;
    double lam[CON_MAX_CONS];
    if (con_is_water(G)) {
      // SETTLE's velocity step: the 3 x 3 system in closed form (Cramer's rule)
      const double det = M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
                         M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
      for (int c = 0; c < 3; ++c) {
        double A[3][3];
        for (int i = 0; i < 3; ++i)
          for (int k = 0; k < 3; ++k) A[i][k] = (k == c) ? M[i][3] : M[i][k];
        lam[c] = (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
                  A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0])) / det;
      }
    } else {
    for (int p = 0; p < n; ++p) {
      int piv = p;
      for (int i = p + 1; i < n; ++i)
        if (fabs(M[i][p]) > fabs(M[piv][p])) piv = i;
      if (piv != p)
        for (int k = 0; k <= n; ++k) {
          const double t = M[p][k];
          M[p][k] = M[piv][k];
          M[piv][k] = t;
        }
      for (int i = p + 1; i < n; ++i) {
        const double f = M[i][p] / M[p][p];
        for (int k = p; k <= n; ++k) M[i][k] -= f * M[p][k];
      }
    }
    for (int p = n - 1; p >= 0; --p) {
      double s = M[p][n];
      for (int k = p + 1; k < n; ++k) s -= M[p][k] * lam[k];
      lam[p] = s / M[p][p];
    }
    }
    for (int c = 0; c < n; ++c)
      for (int k = 0; k < 3; ++k) {
        v[G.ca[c]][k] += lam[c] * im[G.ca[c]] * rv[c][k];
        v[G.cb[c]][k] -= lam[c] * im[G.cb[c]] * rv[c][k];
      }
    for (int j = 0; j < G.na; ++j) {
      const size_t a = (base + G.atom[j]) * 3;
      double v2 = 0.0;
      for (int k = 0; k < 3; ++k) {
        const T vk = (T)v[j][k];
        vel[a + k] = vk;
        v2 += (double)vk * (double)vk;
      }
      if (KINETIC) ek += 0.5 * (double)masses[G.atom[j]] * v2;
    }
  } else if (KINETIC && w < C.ngroups + C.nfree) {
    const int i = C.free_atoms[w - C.ngroups];
    const size_t a = (base + i) * 3;
    const double vx = (double)vel[a], vy = (double)vel[a + 1], vz = (double)vel[a + 2];
    ek = 0.5 * (double)masses[i] * (vx * vx + vy * vy + vz * vz);
  }
  if (KINETIC) {
    __shared__ double red[CON_THREADS / 32];
    block_accumulate<CON_THREADS / 32>(ek, ke + r, red);
  }
}

}  // namespace tmd
