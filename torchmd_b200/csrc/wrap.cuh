// wrap.cuh -- molecules back into the periodic box by their centre (Wrapper.wrap,
// wrapper.py:8-30).
//
// The reference loops over the molecule groups in Python (33,333 iterations of ~5 torch ops
// for the 100k-atom water box, every output period).  Here: one warp per (group, replica),
// groups as a CSR over atom indices; atoms that belong to no bond are groups of one atom
// (the reference's "nongrouped" branch is the same arithmetic with a one-atom sum).
// Arithmetic, per dimension, in the reference's order with single rounded operations:
//   com = (sum of the group's coordinates) / len ;  offset = floor(com / box) * box ;
//   pos -= offset
// The sum runs sequentially in the stored atom order for groups of up to 32 atoms and as a
// lane-strided tree above that (torch's own order for long reductions differs as well; the
// offset only depends on which box image the centre falls into).
#pragma once
#include "context.cuh"

namespace tmd {

constexpr int WRAP_WARPS = 8;

// flag[0] = 1 if every box length of every replica is zero (the reference returns at once)
// T: float ("precision: single") or double ("precision: double"), the dtype of the positions and the box
template <typename T>
__global__ void k_wrap_boxflag(const T* __restrict__ box, int nrep, int* __restrict__ flag) {
  int nonzero = 0;
  for (int e = threadIdx.x; e < nrep * 3; e += blockDim.x) nonzero |= (box[(e / 3) * 9 + (e % 3) * 4] != T(0));
  nonzero = __syncthreads_or(nonzero);
  if (threadIdx.x == 0) flag[0] = nonzero ? 0 : 1;
}

template <typename T>
__global__ void __launch_bounds__(WRAP_WARPS * 32)
k_wrap(int natoms, int ngroups, const int* __restrict__ group_ptr, const int* __restrict__ group_atoms,
       T* __restrict__ pos, const T* __restrict__ box, const int* __restrict__ allzero) {
  if (allzero[0]) return;
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * WRAP_WARPS + (threadIdx.x >> 5);
  const int r = blockIdx.y;
  if (g >= ngroups) return;
  const int b = group_ptr[g], n = group_ptr[g + 1] - b;
  if (n <= 0) return;
  T* p = pos + (size_t)r * natoms * 3;
  const T L[3] = {box[r * 9 + 0], box[r * 9 + 4], box[r * 9 + 8]};
  T sum[3] = {T(0), T(0), T(0)};
  if (n <= 32) {
    T v[3] = {T(0), T(0), T(0)};
    if (lane < n) {
      const size_t a = (size_t)group_atoms[b + lane] * 3;
      v[0] = p[a];
      v[1] = p[a + 1];
      v[2] = p[a + 2];
    }
    for (int m = 0; m < n; ++m) {  // every lane forms the same sequential sum
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const T t = __shfl_sync(0xffffffffu, v[d], m);
        sum[d] = (m == 0) ? t : add_rn(sum[d], t);
      }
    }
  } else {
    for (int e = lane; e < n; e += 32) {
      const size_t a = (size_t)group_atoms[b + e] * 3;
#pragma unroll
      for (int d = 0; d < 3; ++d) sum[d] = add_rn(sum[d], p[a + d]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d)
      for (int o = 16; o; o >>= 1) sum[d] = add_rn(sum[d], __shfl_xor_sync(0xffffffffu, sum[d], o));
  }
  T off[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) off[d] = wrap_offset(sum[d], n, L[d]);
  for (int e = lane; e < n; e += 32) {
    const size_t a = (size_t)group_atoms[b + e] * 3;
#pragma unroll
    for (int d = 0; d < 3; ++d) p[a + d] = sub_rn(p[a + d], off[d]);
  }
}

}  // namespace tmd

struct tmd_wrapper {
  int device = 0;
  int natoms = 0, ngroups = 0;
  int* group_ptr = nullptr;
  int* group_atoms = nullptr;
  int* flag = nullptr;
};
