// fused.cuh -- integrator kernels fused with the force assembly (cluster path, tmd_md_steps).
//
// After the pair kernel of a step the per-atom work of the reference's loop body
// (integrator.py:115-120: forces.compute's bonded part, langevin, _second_VV) is one pass over the atoms:
// bring the atom's pair force home from slot order, add its bonded terms (fp64, atom-centric: bonded.cuh),
// store the total force, kick.  One launch and one round trip of the forces through memory instead of two.
#pragma once
#include "bonded.cuh"
#include "cluster.cuh"
#include "integrate.cuh"

namespace tmd {

template <bool THERMOSTAT, bool KINETIC>
__global__ void __launch_bounds__(BONDED_THREADS)
k_bonded_vv_second(DeviceState S, BondedTablesT<float> T, const float* __restrict__ q_scaled, const float* __restrict__ pos,
                   float* __restrict__ forces, double* __restrict__ energies, float* __restrict__ vel,
                   const float* __restrict__ masses, float dt, float hdt, float neg_gamma, const float* __restrict__ vcoeff,
                   const float* __restrict__ noise, uint64_t seed, uint64_t step_offset, double* __restrict__ ke,
                   const int* __restrict__ ladder) {
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // whole system (cluster path)
  const uint64_t step = step_offset + S.counters[1];
  BondedEnergies E;
  double ek = 0.0;
  if (i < S.natoms) {
    const size_t slot = (size_t)r * S.natoms + i;
    const size_t a = slot * 3;
    Vec3d fb = {0., 0., 0.};
    if (T.atom_ptr && T.atom_ptr[i + 1] > T.atom_ptr[i]) fb = bonded_force_on_atom(S, T, q_scaled, pos, r, i, E);
    const float4 pf = S.cl.f[(size_t)r * (S.cl.slots + 1) + S.cl.inv[slot]];
    const float f[3] = {(float)((double)pf.x + fb.x), (float)((double)pf.y + fb.y), (float)((double)pf.z + fb.z)};
    const float m = masses[i];
    float xi[3] = {0.f, 0.f, 0.f};
    float vc = 0.f;
    if (THERMOSTAT) {
      vc = langevin_scale(vcoeff, ladder, r, S.natoms, i);
      langevin_noise(noise, seed, step, slot, xi);
    }
    float v2 = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      forces[a + d] = f[d];
      float v = vel[a + d];
      langevin_kick<THERMOSTAT>(v, f[d], m, xi[d], vc, neg_gamma, dt, hdt);
      vel[a + d] = v;
      v2 += v * v;
    }
    if (KINETIC) ek = 0.5 * (double)m * (double)v2;
  }
  __shared__ double red[BONDED_THREADS / 32];
  if (KINETIC) block_accumulate<BONDED_THREADS / 32>(ek, ke + r, red);
  if (energies && T.atom_ptr) bonded_energy_reduce(S, T, r, E, energies, red);
}

// The bonded kernel ran beside the pair kernel on a second stream and left its fp64 sums in `scratch`
// (tmd_b200.cu, enqueue_forces): total force = pair force of the atom's slot + bonded sum, rounded once.
__global__ void __launch_bounds__(INTEG_THREADS)
k_cadd_bonded(DeviceState S, float* __restrict__ forces, const double* __restrict__ scratch) {
  const int r = blockIdx.y;
  const int i = S.own_lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.own_lo + S.own_n) return;
  const size_t slot = (size_t)r * S.natoms + i;
  const float4 pf = S.cl.f[(size_t)r * (S.cl.slots + 1) + S.cl.inv[slot]];
  const double sx = scratch ? scratch[slot * 3] : 0.0, sy = scratch ? scratch[slot * 3 + 1] : 0.0, sz = scratch ? scratch[slot * 3 + 2] : 0.0;
  forces[slot * 3 + 0] = (float)((double)pf.x + sx);
  forces[slot * 3 + 1] = (float)((double)pf.y + sy);
  forces[slot * 3 + 2] = (float)((double)pf.z + sz);
}

// ... and the same folded into the second half-kick (tmd_md_steps)
template <bool THERMOSTAT, bool KINETIC>
__global__ void __launch_bounds__(INTEG_THREADS)
k_cvv_second_fold(DeviceState S, float* __restrict__ vel, float* __restrict__ forces, const float* __restrict__ masses, float dt,
                  float hdt, float neg_gamma, const float* __restrict__ vcoeff, const float* __restrict__ noise, uint64_t seed,
                  uint64_t step_offset, double* __restrict__ ke, const double* __restrict__ scratch,
                  const int* __restrict__ ladder) {
  const int r = blockIdx.y;
  const int i = S.own_lo + blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t step = step_offset + S.counters[1];
  double ek = 0.0;
  if (i < S.own_lo + S.own_n) {
    const size_t slot = (size_t)r * S.natoms + i;
    const size_t a = slot * 3;
    const float4 pf = S.cl.f[(size_t)r * (S.cl.slots + 1) + S.cl.inv[slot]];
    const float f[3] = {(float)((double)pf.x + scratch[a]), (float)((double)pf.y + scratch[a + 1]), (float)((double)pf.z + scratch[a + 2])};
    const float m = masses[i];
    float xi[3] = {0.f, 0.f, 0.f};
    float vc = 0.f;
    if (THERMOSTAT) {
      vc = langevin_scale(vcoeff, ladder, r, S.natoms, i);
      langevin_noise(noise, seed, step, slot, xi);
    }
    float v2 = 0.f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      forces[a + d] = f[d];
      float v = vel[a + d];
      langevin_kick<THERMOSTAT>(v, f[d], m, xi[d], vc, neg_gamma, dt, hdt);
      vel[a + d] = v;
      v2 += v * v;
    }
    if (KINETIC) ek = 0.5 * (double)m * (double)v2;
  }
  if (KINETIC) {
    __shared__ double red[INTEG_THREADS / 32];
    block_accumulate<INTEG_THREADS / 32>(ek, ke + r, red);
  }
}

// Between two steps of one tmd_md_steps call, the second half of step n and the first half of step n+1 touch the
// same atoms with nothing in between (integrator.py:115-120 then :112-114 of the next iteration): one pass brings
// the pair force home, adds the bonded sum, finishes the kick of step n, kicks and drifts for step n+1 and prepares
// the next force call (list check, slot records) from the position it still holds -- k_cvv_second_fold followed by
// k_vv_first_prepare without the round trip of forces and velocities through memory and without the second launch.
// The forces buffer is not written: the last step of the call ends with k_cvv_second_fold, which stores it.
// Philox position of step n: counters[2], the copy of counters[1] that step n's pair kernel took (this kernel
// advances counters[1] for step n+1 while its other threads are still reading).
template <bool THERMOSTAT>
__global__ void __launch_bounds__(INTEG_THREADS)
k_cstep_boundary(DeviceState S, float* __restrict__ pos, float* __restrict__ vel, const float* __restrict__ masses, float dt,
                 float hdt, float neg_gamma, const float* __restrict__ vcoeff, uint64_t seed, uint64_t step_offset,
                 const double* __restrict__ scratch, const int* __restrict__ ladder) {
  const int parity = (int)(S.counters[0] & 1ull);
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // whole system
  const uint64_t step = step_offset + S.counters[2];
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[1] += 1;  // Philox position of step n+1
  if (i == 0) S.flags[r * F_COUNT + F_REBUILD0 + (parity ^ 1)] = 0;
  if (i >= S.natoms) return;
  const size_t slot = (size_t)r * S.natoms + i;
  const size_t a = slot * 3;
  const float4 pf = S.cl.f[(size_t)r * (S.cl.slots + 1) + S.cl.inv[slot]];
  const float f[3] = {(float)((double)pf.x + scratch[a]), (float)((double)pf.y + scratch[a + 1]), (float)((double)pf.z + scratch[a + 2])};
  const float m = masses[i];
  float xi[3] = {0.f, 0.f, 0.f};
  float vc = 0.f;
  if (THERMOSTAT) {
    vc = langevin_scale(vcoeff, ladder, r, S.natoms, i);
    normal3(seed, step, slot, xi);
  }
  float x[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    float v = vel[a + d];
    const float acc = langevin_kick<THERMOSTAT>(v, f[d], m, xi[d], vc, neg_gamma, dt, hdt);  // end of step n, one a for both
    x[d] = kick_drift(pos + a + d, v, acc, dt, hdt);
    pos[a + d] = x[d];
    vel[a + d] = v;
  }
  prepare_atom(S, r, i, parity, x[0], x[1], x[2]);
}

}  // namespace tmd
