// remd.cuh -- temperature replica exchange (parallel tempering) on the device: the decision and the velocity scaling.
//
// The context holds a ladder of R temperatures (tmd_set_temperature_ladder) and a caller-owned (R,) int32 device array
// `ladder`, a permutation of 0..R-1: ladder[r] is the temperature index of replica r, and the Langevin kernels read
// replica r's noise scale from row ladder[r] of the (R, N, 1) vcoeff table.  An attempt rewrites only the contents of
// `ladder`, so the captured step graphs, which hold its address, stay valid.
#pragma once
#include "integrate.cuh"

namespace tmd {

constexpr int REMD_MAX_REPLICAS = 1024;  // one block holds the ladder's inverse in shared memory
constexpr unsigned REMD_DOMAIN = 0x40000000u;  // counter word 1 of the exchange draws: the Langevin slots stay below 2^30 there
constexpr double REMD_BOLTZMAN = 0.001987191;  // kcal/(mol K), the integrator's

// The uniform of pair (k, k+1) at attempt a: u53 of Philox4x32-10 on the counter (k, REMD_DOMAIN, a lo, a hi).
__device__ __forceinline__ double remd_uniform(uint64_t seed, uint64_t attempt, int k) {
  const uint4 w = philox4x32_10(make_uint4((unsigned)k, REMD_DOMAIN, (unsigned)attempt, (unsigned)(attempt >> 32)),
                                make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
  return u53(w.x, w.y);
}

// One attempt, one block of at least R threads.  U_r = sum_{t < nterms} energies[r*stride + t] in term order (fp64);
// owner[k] = the replica at temperature k; pairs (k, k+1) with k = attempt (mod 2) try a swap with
// D = (beta_k - beta_{k+1}) (U_owner[k] - U_owner[k+1]), accepted when D >= 0 or u < exp(D).  Every pair tried draws.
// factor[r] = sqrt(T_new / T_old) of replica r (1 where it kept its temperature); counts[2k] attempts, [2k+1] accepts.
__global__ void k_remd_exchange(int R, const double* __restrict__ energies, int stride, int nterms,
                                const double* __restrict__ temps, int* __restrict__ ladder, uint64_t seed, uint64_t attempt,
                                double* __restrict__ factor, long long* __restrict__ counts) {
  __shared__ int owner[REMD_MAX_REPLICAS];
  __shared__ int next[REMD_MAX_REPLICAS];
  const int r = threadIdx.x;
  int before = 0;
  if (r < R) {
    before = ladder[r];
    owner[before] = r;
    next[r] = before;
  }
  __syncthreads();
  const int k = (int)(attempt & 1ull) + 2 * r;
  if (k + 1 < R) {
    const int i = owner[k], j = owner[k + 1];
    double ui = 0.0, uj = 0.0;
    for (int t = 0; t < nterms; ++t) {
      ui += energies[(size_t)i * stride + t];
      uj += energies[(size_t)j * stride + t];
    }
    const double bk = 1.0 / (REMD_BOLTZMAN * temps[k]), bk1 = 1.0 / (REMD_BOLTZMAN * temps[k + 1]);
    const double delta = (bk - bk1) * (ui - uj);
    const double u = remd_uniform(seed, attempt, k);
    const bool accept = delta >= 0.0 || u < exp(delta);
    counts[2 * k] += 1;
    if (accept) {
      counts[2 * k + 1] += 1;
      next[i] = k + 1;
      next[j] = k;
    }
  }
  __syncthreads();
  if (r < R) {
    const int after = next[r];
    factor[r] = after == before ? 1.0 : sqrt(temps[after] / temps[before]);
    if (after != before) ladder[r] = after;
  }
}

// v = (T)((double)v * factor[r]) for the replicas whose temperature changed: one rounding per component.
template <typename T>
__global__ void __launch_bounds__(INTEG_THREADS)
k_remd_scale(int natoms, T* __restrict__ vel, const double* __restrict__ factor) {
  const int r = blockIdx.y;
  const double f = factor[r];
  if (f == 1.0) return;
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)natoms * 3) return;
  T* v = vel + (size_t)r * natoms * 3 + e;
  *v = (T)((double)*v * f);
}

}  // namespace tmd
