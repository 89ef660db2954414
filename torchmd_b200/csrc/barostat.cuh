// barostat.cuh -- the molecule move of the Monte Carlo barostat (tmd_scale_molecules), templated on the precision T of
// the positions (float or double).
//
// Molecules are the connected components of the bond graph, held as a CSR (tmd_set_molecules): the atoms of a molecule
// in breadth-first order of a spanning tree of its bonds, and for each the atom it was reached from (the first atom is
// its own parent).  One thread per (molecule, replica):
//   unwrap along the tree       u_a = u_parent + minimum_image(r_a - r_parent), u_first = r_first
//   centroid                    c = mean of u_a
//   image of each atom          n_a = rint((r_a - u_a) / L), so r_a = u_a + n_a L
//   move                        r_a' = r_a + (s - 1) c + n_a (L' - L),  L' = s L
// The molecule moves rigidly with its centroid, its unwrapped geometry is that of the old box, and every atom keeps its
// own image in the new one: a water split across the box stays split, a chain longer than half the box keeps its bonds.
// All arithmetic is fp64; each coordinate is rounded to T once.
#pragma once
#include "context.cuh"

namespace tmd {

constexpr int MOL_THREADS = 128;

struct MolTables {
  int nmol, natoms;
  const int* ptr;     // (nmol + 1) CSR offsets into atoms
  const int* atoms;   // atoms of every molecule, breadth-first along its bond tree
  const int* parent;  // (aligned with atoms) the atom each one was reached from; the first atom of a molecule: itself
  double* u;          // (R, natoms, 3) scratch: unwrapped coordinates
};

__device__ __forceinline__ double mol_image(double d, double L) { return d - L * rint(d / L); }

// blockIdx.y = replica; scale (R,3) per-axis factors s, L (R,3) the box lengths before the move
template <typename T>
__global__ void __launch_bounds__(MOL_THREADS) k_scale_molecules(MolTables m, T* __restrict__ pos, const double* __restrict__ scale,
                                                               const double* __restrict__ L) {
  const int r = blockIdx.y;
  const int mol = blockIdx.x * blockDim.x + threadIdx.x;
  if (mol >= m.nmol) return;
  const size_t base = (size_t)r * m.natoms;
  const int k0 = m.ptr[mol], k1 = m.ptr[mol + 1];
  double box[3], s[3];
  for (int d = 0; d < 3; ++d) {
    box[d] = L[3 * r + d];
    s[d] = scale[3 * r + d];
  }
  double c[3] = {0.0, 0.0, 0.0};
  for (int k = k0; k < k1; ++k) {
    const int a = m.atoms[k], p = m.parent[k];
    double* ua = m.u + (base + a) * 3;
    const T* ra = pos + (base + a) * 3;
    if (p == a) {
      for (int d = 0; d < 3; ++d) ua[d] = (double)ra[d];
    } else {
      const double* up = m.u + (base + p) * 3;
      const T* rp = pos + (base + p) * 3;
      for (int d = 0; d < 3; ++d) ua[d] = up[d] + mol_image((double)ra[d] - (double)rp[d], box[d]);
    }
    for (int d = 0; d < 3; ++d) c[d] += ua[d];
  }
  const double inv = 1.0 / (double)(k1 - k0);
  double shift[3], dL[3];
  for (int d = 0; d < 3; ++d) {
    shift[d] = (s[d] - 1.0) * (c[d] * inv);
    dL[d] = s[d] * box[d] - box[d];
  }
  for (int k = k0; k < k1; ++k) {
    const int a = m.atoms[k];
    const double* ua = m.u + (base + a) * 3;
    T* ra = pos + (base + a) * 3;
    for (int d = 0; d < 3; ++d) {
      const double x = (double)ra[d];
      const double n = rint((x - ua[d]) / box[d]);
      ra[d] = (T)(x + (shift[d] + n * dL[d]));
    }
  }
}

}  // namespace tmd
