// integrate.cuh -- velocity Verlet + Langevin kick (K5, K6) and kinetic energy.
//
// Replaces integrator.py:61-74 (_first_VV, langevin, _second_VV) and
// kinetic_energy (integrator.py:8-30).  Pure streaming kernels, one thread per
// atom; the arithmetic keeps the reference's operation order with single rounded
// ops, so with injected noise the trajectory matches the reference fp32 path to
// the last bit as long as the forces do.
#pragma once
#include "context.cuh"
#include "neighbor.cuh"
#include "pair.cuh"
#include "ptx.cuh"

namespace tmd {

constexpr int INTEG_THREADS = 256;

// The per-atom arithmetic of the step, one coordinate at a time, in the reference's operation order with single
// rounded ops; T = float or double.  Every integrator kernel (here and in fused.cuh) is built from these.
//
// First half (integrator.py:61-64), a = F/m: returns *x + (vel*dt + ((0.5*a)*dt)*dt), then vel += (0.5*dt)*a.  (x is
// read only where the drift is added, after the force and the velocity: the kernels keep their load order.)
template <typename T>
__device__ __forceinline__ T kick_drift(const T* x, T& v, T acc, T dt, T hdt) {
  const T drift = add_rn(mul_rn(v, dt), mul_rn(mul_rn(mul_rn(T(0.5), acc), dt), dt));
  const T xn = add_rn(*x, drift);
  v = add_rn(v, mul_rn(hdt, acc));
  return xn;
}
// Second half (integrator.py:72-74 then 67-69): [vel += ((-gamma*vel)*dt + xi*vcoeff)], then vel += (0.5*dt)*a.
// Returns a = F/m, formed after the Langevin term, for a caller that kicks again (k_cstep_boundary).
template <bool THERMOSTAT, typename T>
__device__ __forceinline__ T langevin_kick(T& v, T f, T m, T xi, T vc, T neg_gamma, T dt, T hdt) {
  if (THERMOSTAT) v = add_rn(v, add_rn(mul_rn(mul_rn(neg_gamma, v), dt), mul_rn(xi, vc)));
  const T acc = div_rn(f, m);
  v = add_rn(v, mul_rn(hdt, acc));
  return acc;
}

template <typename T>
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_first(int natoms, int lo, int cnt, unsigned long long* counters, T* __restrict__ pos,
           T* __restrict__ vel, const T* __restrict__ forces, const T* __restrict__ masses,
           T dt, T hdt) {
  const int r = blockIdx.y;
  const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;  // atoms [lo, lo+cnt) only
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) counters[1] += 1;  // Philox position of this step
  if (i >= lo + cnt) return;
  const T m = masses[i];
  const size_t a = ((size_t)r * natoms + i) * 3;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const T acc = div_rn(forces[a + d], m);
    T v = vel[a + d];
    pos[a + d] = kick_drift(pos + a + d, v, acc, dt, hdt);
    vel[a + d] = v;
  }
}

// k_vv_first followed by k_prepare (neighbor.cuh) in one pass over the atoms: the thread that moved an atom still
// holds its new position, so the list check and the refresh of the sorted records cost no second read of the
// positions and no second launch.  Whole-system runs only (a decomposed run prepares after the exchange).
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_first_prepare(DeviceState S, float* __restrict__ pos, float* __restrict__ vel, const float* __restrict__ forces,
                   const float* __restrict__ masses, float dt, float hdt) {
  const int parity = (int)(S.counters[0] & 1ull);
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[1] += 1;  // Philox position of this step
  if (i == 0) S.flags[r * F_COUNT + F_REBUILD0 + (parity ^ 1)] = 0;
  if (i >= S.natoms) return;
  const float m = masses[i];
  const size_t a = ((size_t)r * S.natoms + i) * 3;
  float x[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float acc = div_rn(forces[a + d], m);
    float v = vel[a + d];
    x[d] = kick_drift(pos + a + d, v, acc, dt, hdt);
    pos[a + d] = x[d];
    vel[a + d] = v;
  }
  prepare_atom(S, r, i, parity, x[0], x[1], x[2]);
}

// ---- fused integrate + exchange (decomposed runs, include/tmd_b200.h tmd_dd_*) -----------
struct PeerTable {
  float* pos[TMD_MAX_PEERS];        // the buffer written this step, on every rank (own rank included)
  unsigned* flags[TMD_MAX_PEERS];   // flag array of every rank: flags[p][q] = last step rank q finished pushing to p
  int world, rank;
};

// k_vv_first for the owned atoms, new positions stored into every rank's write buffer; the
// last block to finish publishes this rank's step number in every rank's flag array.
// sync: [0] block ticket (returns to 0), [1] steps pushed so far.
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_first_push(int natoms, int lo, int cnt, unsigned long long* counters, const float* __restrict__ pos_in,
                float* __restrict__ vel, const float* __restrict__ forces, const float* __restrict__ masses,
                float dt, float hdt, PeerTable pt, unsigned* __restrict__ sync) {
  const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;  // single replica
  if (blockIdx.x == 0 && threadIdx.x == 0) counters[1] += 1;  // Philox position of this step
  if (i < lo + cnt) {
    const float m = masses[i];
    const size_t a = (size_t)i * 3;
    float x[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float acc = div_rn(forces[a + d], m);
      float v = vel[a + d];
      x[d] = kick_drift(pos_in + a + d, v, acc, dt, hdt);
      vel[a + d] = v;
    }
    for (int p = 0; p < pt.world; ++p) {
      float* dst = pt.pos[p] + a;
      dst[0] = x[0];
      dst[1] = x[1];
      dst[2] = x[2];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();  // this block's stores (ordered before the barrier) precede the ticket
    const unsigned done = atomicAdd(sync + 0, 1u);
    if (done == gridDim.x - 1) {
      __threadfence_system();
      sync[0] = 0;
      const unsigned epoch = sync[1] + 1u;
      sync[1] = epoch;
      for (int p = 0; p < pt.world; ++p) st_release_sys(pt.flags[p] + pt.rank, epoch);
    }
  }
}

// One warp: lane q waits for rank q's flag of the current step.  sync[2]: steps waited for so far.
__global__ void k_wait_peers(const unsigned* __restrict__ flags_local, unsigned* __restrict__ sync, int world,
                             int* __restrict__ errflag) {
  const int q = threadIdx.x;
  unsigned target = 0;
  if (q == 0) target = sync[2] + 1u;
  target = __shfl_sync(0xffffffffu, target, 0);
  if (q < world) {
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(flags_local + q) - target) < 0) {
      if (clock64() - t0 > 6000000000ll) {  // ~3 s: a peer died or the step counts diverged
        *errflag = 1;
        break;
      }
      __nanosleep(40);
    }
  }
  __syncwarp();
  if (q == 0) sync[2] = target;
}

// Philox4x32-10 counter-based generator (Salmon et al., SC'11).
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int round = 0; round < 10; ++round) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}
// three N(0,1) draws for (atom slot, step): Box-Muller on Philox output
__device__ __forceinline__ void normal3(uint64_t seed, uint64_t step, uint64_t slot, float out[3]) {
  const uint4 u = philox4x32_10(make_uint4((unsigned)slot, (unsigned)(slot >> 32), (unsigned)step, (unsigned)(step >> 32)),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  const float two_pi = 6.283185307179586f;
  const float u0 = ((float)(u.x >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float u1 = ((float)(u.y >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float u2 = ((float)(u.z >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float u3 = ((float)(u.w >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float r0 = sqrtf(-2.0f * logf(u0)), r1 = sqrtf(-2.0f * logf(u2));
  float s, c;
  sincosf(two_pi * u1, &s, &c);
  out[0] = r0 * c;
  out[1] = r0 * s;
  out[2] = r1 * cosf(two_pi * u3);
}
// the fp64 draws: two Philox4x32-10 blocks of the same stream (the second with the top counter bit set), 53-bit
// uniforms, Box-Muller in fp64
__device__ __forceinline__ double u53(unsigned hi, unsigned lo) {
  return ((double)(((unsigned long long)(hi >> 5) << 26) | (lo >> 6)) + 0.5) * (1.0 / 9007199254740992.0);
}
__device__ __forceinline__ void normal3(uint64_t seed, uint64_t step, uint64_t slot, double out[3]) {
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
// The Langevin noise of atom slot `slot` at `step`: the injected noise[3*slot..] if given, else the Philox draw.
template <typename T>
__device__ __forceinline__ void langevin_noise(const T* __restrict__ noise, uint64_t seed, uint64_t step, size_t slot, T xi[3]) {
  if (noise) {
    xi[0] = noise[3 * slot]; xi[1] = noise[3 * slot + 1]; xi[2] = noise[3 * slot + 2];
  } else {
    normal3(seed, step, slot, xi);
  }
}

// The Langevin noise scale of atom i of replica r: vcoeff is one (N,1) row, or with a temperature ladder (remd.cuh) an
// (R,N,1) table of which replica r reads row ladder[r].  The branch is uniform (a kernel argument).
template <typename T>
__device__ __forceinline__ T langevin_scale(const T* __restrict__ vcoeff, const int* __restrict__ ladder, int r, int natoms, int i) {
  return ladder ? vcoeff[(size_t)ladder[r] * natoms + i] : vcoeff[i];
}

// langevin_kick on every atom, optionally followed by the kinetic energy.
template <typename T, bool THERMOSTAT, bool KINETIC, bool FOLD>
__device__ __forceinline__ void vv_second_body(int natoms, int lo, int cnt, const unsigned long long* __restrict__ counters,
                                               T* __restrict__ vel, const T* __restrict__ forces,
                                               const T* __restrict__ masses, T dt, T hdt, T neg_gamma,
                                               const T* __restrict__ vcoeff, const T* __restrict__ noise,
                                               uint64_t seed, uint64_t step_offset, double* __restrict__ ke,
                                               float* forces_rw, const double* __restrict__ scratch,
                                               const int* __restrict__ ladder) {
  const int r = blockIdx.y;
  const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t step = step_offset + counters[1];  // device-resident step count: graph replayable
  double ek = 0.0;
  if (i < lo + cnt) {
    const T m = masses[i];
    const size_t slot = (size_t)r * natoms + i;
    const size_t a = slot * 3;
    T xi[3] = {T(0), T(0), T(0)};
    T vc = T(0);
    if (THERMOSTAT) {
      vc = langevin_scale(vcoeff, ladder, r, natoms, i);
      langevin_noise(noise, seed, step, slot, xi);
    }
    T v2 = T(0);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      T f;
      if constexpr (FOLD) {  // k_add_bonded's work (bonded.cuh): the bonded sums of the overlapped k_bonded_sum, rounded once
        f = forces_rw[a + d];
        const double sb = scratch[a + d];
        if (sb != 0.0) {
          f = (float)((double)f + sb);
          forces_rw[a + d] = f;
        }
      } else {
        f = forces[a + d];
      }
      T v = vel[a + d];
      langevin_kick<THERMOSTAT>(v, f, m, xi[d], vc, neg_gamma, dt, hdt);
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

template <typename T, bool THERMOSTAT, bool KINETIC>
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_second(int natoms, int lo, int cnt, const unsigned long long* __restrict__ counters,
            T* __restrict__ vel, const T* __restrict__ forces,
            const T* __restrict__ masses, T dt, T hdt, T neg_gamma,
            const T* __restrict__ vcoeff, const T* __restrict__ noise, uint64_t seed,
            uint64_t step_offset, double* __restrict__ ke, const int* __restrict__ ladder) {
  vv_second_body<T, THERMOSTAT, KINETIC, false>(natoms, lo, cnt, counters, vel, forces, masses, dt, hdt, neg_gamma, vcoeff, noise,
                                                seed, step_offset, ke, nullptr, nullptr, ladder);
}

// k_add_bonded + k_vv_second in one pass (tmd_md_steps with the bonded kernel overlapped on a second stream): the
// forces get the bonded sums with the same single rounding and are written back for the next half-kick.
template <bool THERMOSTAT, bool KINETIC>
__global__ void __launch_bounds__(INTEG_THREADS)
k_vv_second_fold(int natoms, int lo, int cnt, const unsigned long long* __restrict__ counters,
                 float* __restrict__ vel, float* __restrict__ forces,
                 const float* __restrict__ masses, float dt, float hdt, float neg_gamma,
                 const float* __restrict__ vcoeff, const float* __restrict__ noise, uint64_t seed,
                 uint64_t step_offset, double* __restrict__ ke, const double* __restrict__ scratch,
                 const int* __restrict__ ladder) {
  vv_second_body<float, THERMOSTAT, KINETIC, true>(natoms, lo, cnt, counters, vel, nullptr, masses, dt, hdt, neg_gamma, vcoeff,
                                                   noise, seed, step_offset, ke, forces, scratch, ladder);
}

template <typename T>
__global__ void __launch_bounds__(INTEG_THREADS)
k_kinetic(int natoms, int lo, int cnt, const T* __restrict__ vel, const T* __restrict__ masses,
          double* __restrict__ ke) {
  const int r = blockIdx.y;
  const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;
  double ek = 0.0;
  if (i < lo + cnt) {
    const size_t a = ((size_t)r * natoms + i) * 3;
    const T vx = vel[a], vy = vel[a + 1], vz = vel[a + 2];
    ek = 0.5 * (double)masses[i] * (double)(vx * vx + vy * vy + vz * vz);
  }
  __shared__ double red[INTEG_THREADS / 32];
  block_accumulate<INTEG_THREADS / 32>(ek, ke + r, red);
}

}  // namespace tmd
