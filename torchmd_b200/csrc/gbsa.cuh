// gbsa.cuh -- Generalized Born implicit solvent, OBC2 (Onufriev, Bashford, Case 2004; AMBER igb=5), with the optional
// ACE non-polar term, for systems without a box.  Per replica (blockIdx.y), templated on the precision T of the pair
// arithmetic (float or double); every per-atom sum is fp64.  Three passes per force call:
//   k_gb_radii    I_i = sum_j HCT(r_ij; rho_i, S_j)  ->  Born radius B_i and the chain factor dB_i / dI_i
//   k_gb_energy   E_pol = -1/2 (1 - 1/eps) sum_i sum_j qi qj / f_ij (i = j included), E_np = sum_i np (R_i + 1.4)^2
//                 (R_i / B_i)^6, and dE/dB_i
//   k_gb_forces   per atom i: the pair derivative at fixed radii plus the chain through I_i and every I_j, ADDED to
//                 forces (as k_pme_gather does)
// Each pass gives a warp to an atom i: its lanes take the partners j of shared-memory tiles in a fixed order, each lane
// sums in fp64, and a fixed xor-shuffle tree reduces the warp.  No atomics touch a force or a radius, so every pass
// is bitwise reproducible from call to call.  Charges carry sqrt(coulomb constant), as in the pair kernels.
#pragma once

#include "context.cuh"

namespace tmd {

constexpr int GB_WARPS = 8;                // atoms i per block
constexpr int GB_THREADS = GB_WARPS * 32;  // also the partners j per shared-memory tile
constexpr double GB_ALPHA = 1.0, GB_BETA = 0.8, GB_GAMMA = 4.85;  // OBC2
constexpr double GB_OFFSET = 0.09;         // A: rho = R - offset
constexpr double GB_PROBE = 1.4;           // A: solvent probe radius of the non-polar term

struct GbArgs {
  int natoms;
  const double* rho;   // (N) offset radius R - 0.09
  const double* scr;   // (N) scaled radius S = screen * rho
  const double* rad;   // (N) radius R
  const double* q;     // (N) charge * sqrt(coulomb constant)
  double* born;        // (R,N) Born radius B
  double* chain;       // (R,N) dB / dI
  double* dedb;        // (R,N) dE / dB
  double pref;         // -(1 - 1 / solvent dielectric)
  double np;           // 4 pi sigma (surface tension, kcal/mol/A^2); 0: no non-polar term
};

__host__ __device__ __forceinline__ float gb_log(float x) { return logf(x); }
__host__ __device__ __forceinline__ double gb_log(double x) { return log(x); }
__host__ __device__ __forceinline__ float gb_exp(float x) { return expf(x); }
__host__ __device__ __forceinline__ double gb_exp(double x) { return exp(x); }
__host__ __device__ __forceinline__ float gb_sqrt(float x) { return sqrtf(x); }
__host__ __device__ __forceinline__ double gb_sqrt(double x) { return sqrt(x); }

// Below xmax the separated-sphere term uses its series (n terms), above it the closed form.
template <typename T>
struct GbSeries;
template <>
struct GbSeries<float> {
  static constexpr float xmax = 0.5f;
  static constexpr int n = 12;  // truncation (1/4)^12 = 6e-8 relative
};
template <>
struct GbSeries<double> {
  static constexpr double xmax = 0.1;
  static constexpr int n = 8;  // truncation 0.01^8 = 1e-16 relative
};

// HCT descreening term of a sphere of scaled radius S at distance r (> 0) from an atom of offset radius rho, and its
// derivative d/dr.  With U = r + S and L = max(rho, |r - S|), zero unless rho < U:
//   1/L - 1/U + r/4 (1/U^2 - 1/L^2) + 1/(2r) ln(L/U) + S^2/(4r) (1/L^2 - 1/U^2)  [+ 2 (1/rho - 1/L) if rho < S - r]
// It is 2 (1/4 pi) times the integral of |x|^-4 over the part of the sphere outside radius rho.  When the sphere lies
// wholly outside (r - S >= rho) this is f(x)/r with x = S/r and f(x) = x/(1-x^2) - artanh(x), whose O(1/r) parts cancel
// to O(x^3 / r): f is then summed as its series sum_k 2k/(2k+1) x^(2k+1) for small x, and d/dr = -(f + 2 x^3/(1-x^2)^2)/r^2.
template <typename T>
__host__ __device__ __forceinline__ T gb_hct(T r, T rho, T S, T* dI) {
  const T U = r + S;
  if (!(rho < U)) {
    *dI = T(0);
    return T(0);
  }
  const T ir = T(1) / r;
  if (r - S >= rho) {
    const T x = S * ir, x2 = x * x, w = T(1) / (T(1) - x2);
    T f;
    if (x < GbSeries<T>::xmax) {
      T s = T(2 * GbSeries<T>::n) / T(2 * GbSeries<T>::n + 1);
#pragma unroll
      for (int k = GbSeries<T>::n - 1; k >= 1; --k) s = s * x2 + T(2 * k) / T(2 * k + 1);
      f = x2 * x * s;
    } else {
      f = x * w - T(0.5) * gb_log(U / (r - S));
    }
    *dI = -(f + T(2) * x2 * x * w * w) * ir * ir;
    return f * ir;
  }
  const T d = r - S;
  const bool engulfed = rho < -d;  // sphere i inside sphere j
  const T L = engulfed ? -d : rho;
  const T lp = engulfed ? T(-1) : T(0);  // dL/dr
  const T iL = T(1) / L, iU = T(1) / U, iL2 = iL * iL, iU2 = iU * iU;
  const T lnr = gb_log(L * iU);
  const T S2 = S * S;
  T I = iL - iU + T(0.25) * r * (iU2 - iL2) + T(0.5) * ir * lnr + T(0.25) * S2 * ir * (iL2 - iU2);
  T dd = -lp * iL2 + iU2 + T(0.25) * (iU2 - iL2) + T(0.5) * r * (lp * iL2 * iL - iU2 * iU) - T(0.5) * ir * ir * lnr +
         T(0.5) * ir * (lp * iL - iU) - T(0.25) * S2 * ir * ir * (iL2 - iU2) + T(0.5) * S2 * ir * (iU2 * iU - lp * iL2 * iL);
  if (engulfed) {
    I += T(2) * (T(1) / rho - iL);
    dd += T(2) * lp * iL2;
  }
  *dI = dd;
  return I;
}

// Per atom: offset radius rho, Born radius B, dB/dI and dE/dB from the fp64 sums (host and device; oracle/gbsa.py).
__host__ __device__ __forceinline__ void gb_born(double I, double rho, double R, double* B, double* dBdI) {
  const double psi = 0.5 * rho * I;
  const double t = tanh(psi * (GB_ALPHA - psi * (GB_BETA - GB_GAMMA * psi)));
  const double b = 1.0 / (1.0 / rho - t / R);
  *B = b;
  *dBdI = b * b * (1.0 - t * t) * (GB_ALPHA - psi * (2.0 * GB_BETA - 3.0 * GB_GAMMA * psi)) / R * 0.5 * rho;
}

__device__ __forceinline__ double gb_warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Records of one tile of partners: x, y, z and up to five per-atom values.
template <typename T>
struct GbRec {
  T x, y, z, a, b, c, d, e;
};

// Stage partners [j0, j0 + GB_THREADS) of the replica at `base` into tile; fill(j, rec) supplies the per-atom values.
template <typename T, typename Fill>
__device__ __forceinline__ void gb_stage(GbRec<T>* tile, const T* pos, size_t base, int j0, int n, Fill fill) {
  const int j = j0 + (int)threadIdx.x;
  if (j < n) {
    GbRec<T> rec;
    rec.x = pos[3 * (base + j)];
    rec.y = pos[3 * (base + j) + 1];
    rec.z = pos[3 * (base + j) + 2];
    fill(j, rec);
    tile[threadIdx.x] = rec;
  }
}

template <typename T>
__global__ void __launch_bounds__(GB_THREADS) k_gb_radii(GbArgs a, const T* __restrict__ pos) {
  __shared__ GbRec<T> tile[GB_THREADS];
  const int r = blockIdx.y, n = a.natoms, lane = threadIdx.x & 31;
  const int i = blockIdx.x * GB_WARPS + (threadIdx.x >> 5);
  const bool active = i < n;
  const size_t base = (size_t)r * n;
  const int ic = active ? i : 0;
  const T xi = pos[3 * (base + ic)], yi = pos[3 * (base + ic) + 1], zi = pos[3 * (base + ic) + 2];
  const T rho = (T)a.rho[ic];
  double acc = 0.0;
  for (int j0 = 0; j0 < n; j0 += GB_THREADS) {
    __syncthreads();
    gb_stage<T>(tile, pos, base, j0, n, [&](int j, GbRec<T>& rec) { rec.a = (T)a.scr[j]; });
    __syncthreads();
    if (!active) continue;
    const int m = n - j0 < GB_THREADS ? n - j0 : GB_THREADS;
    for (int k = lane; k < m; k += 32) {
      if (j0 + k == i) continue;
      const GbRec<T> p = tile[k];
      const T dx = xi - p.x, dy = yi - p.y, dz = zi - p.z;
      T dI;
      acc += (double)gb_hct<T>(gb_sqrt(dx * dx + dy * dy + dz * dz), rho, p.a, &dI);
    }
  }
  acc = gb_warp_sum(acc);
  if (active && lane == 0) gb_born(acc, a.rho[i], a.rad[i], a.born + base + i, a.chain + base + i);
}

template <typename T>
__global__ void __launch_bounds__(GB_THREADS) k_gb_energy(GbArgs a, const T* __restrict__ pos, double* __restrict__ energies) {
  __shared__ GbRec<T> tile[GB_THREADS];
  __shared__ double red[GB_WARPS];
  const int r = blockIdx.y, n = a.natoms, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * GB_WARPS + w;
  const bool active = i < n;
  const size_t base = (size_t)r * n;
  const int ic = active ? i : 0;
  const T xi = pos[3 * (base + ic)], yi = pos[3 * (base + ic) + 1], zi = pos[3 * (base + ic) + 2];
  const T bi = (T)a.born[base + ic];
  double se = 0.0, sb = 0.0;  // sum_j qj / f_ij, sum_j qj e (1 + r^2 / 4D) B_j / f^3
  for (int j0 = 0; j0 < n; j0 += GB_THREADS) {
    __syncthreads();
    gb_stage<T>(tile, pos, base, j0, n, [&](int j, GbRec<T>& rec) {
      rec.a = (T)a.q[j];
      rec.b = (T)a.born[base + j];
    });
    __syncthreads();
    if (!active) continue;
    const int m = n - j0 < GB_THREADS ? n - j0 : GB_THREADS;
    for (int k = lane; k < m; k += 32) {
      const GbRec<T> p = tile[k];
      const T dx = xi - p.x, dy = yi - p.y, dz = zi - p.z;
      const T r2 = dx * dx + dy * dy + dz * dz;  // 0 for j = i: f = B_i
      const T D = bi * p.b, u = r2 / (T(4) * D), e = gb_exp(-u);
      const T f2 = r2 + D * e, inv_f = T(1) / gb_sqrt(f2);
      se += (double)(p.a * inv_f);
      sb += (double)(p.a * e * (T(1) + u) * p.b * inv_f * inv_f * inv_f);
    }
  }
  se = gb_warp_sum(se);
  sb = gb_warp_sum(sb);
  double ei = 0.0;
  if (active && lane == 0) {
    const double qi = a.q[i], B = a.born[base + i], R = a.rad[i];
    ei = 0.5 * a.pref * qi * se;
    double g = -0.5 * a.pref * qi * sb;
    if (a.np != 0.0) {
      const double s = R / B, s2 = s * s, enp = a.np * (R + GB_PROBE) * (R + GB_PROBE) * s2 * s2 * s2;
      ei += enp;
      g -= 6.0 * enp / B;
    }
    a.dedb[base + i] = g;
  }
  if (energies) {
    if (lane == 0) red[w] = ei;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int k = 0; k < GB_WARPS; ++k) s += red[k];
      atomicAdd(energies + (size_t)r * TMD_NUM_ENERGIES + TMD_E_ELECTROSTATICS, s);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(GB_THREADS) k_gb_forces(GbArgs a, const T* __restrict__ pos, T* __restrict__ forces) {
  __shared__ GbRec<T> tile[GB_THREADS];
  const int r = blockIdx.y, n = a.natoms, lane = threadIdx.x & 31;
  const int i = blockIdx.x * GB_WARPS + (threadIdx.x >> 5);
  const bool active = i < n;
  const size_t base = (size_t)r * n;
  const int ic = active ? i : 0;
  const T xi = pos[3 * (base + ic)], yi = pos[3 * (base + ic) + 1], zi = pos[3 * (base + ic) + 2];
  const T bi = (T)a.born[base + ic], rhoi = (T)a.rho[ic], si = (T)a.scr[ic];
  const T pqi = (T)(a.pref * a.q[ic]);
  const T gi = (T)(a.dedb[base + ic] * a.chain[base + ic]);  // dE/dI_i
  double fx = 0.0, fy = 0.0, fz = 0.0;
  for (int j0 = 0; j0 < n; j0 += GB_THREADS) {
    __syncthreads();
    gb_stage<T>(tile, pos, base, j0, n, [&](int j, GbRec<T>& rec) {
      rec.a = (T)a.q[j];
      rec.b = (T)a.born[base + j];
      rec.c = (T)a.rho[j];
      rec.d = (T)a.scr[j];
      rec.e = (T)(a.dedb[base + j] * a.chain[base + j]);
    });
    __syncthreads();
    if (!active) continue;
    const int m = n - j0 < GB_THREADS ? n - j0 : GB_THREADS;
    for (int k = lane; k < m; k += 32) {
      if (j0 + k == i) continue;
      const GbRec<T> p = tile[k];
      const T dx = xi - p.x, dy = yi - p.y, dz = zi - p.z;
      const T r2 = dx * dx + dy * dy + dz * dz, rr = gb_sqrt(r2);
      const T D = bi * p.b, e = gb_exp(-r2 / (T(4) * D));
      const T inv_f = T(1) / gb_sqrt(r2 + D * e);
      T dij, dji;
      gb_hct<T>(rr, rhoi, p.d, &dij);  // dI_i / dr
      gb_hct<T>(rr, p.c, si, &dji);    // dI_j / dr
      // -dE/dr / r: the pair at fixed radii, then the radii of i and j
      const T c = pqi * p.a * (T(1) - T(0.25) * e) * inv_f * inv_f * inv_f - (gi * dij + p.e * dji) / rr;
      fx += (double)(c * dx);
      fy += (double)(c * dy);
      fz += (double)(c * dz);
    }
  }
  fx = gb_warp_sum(fx);
  fy = gb_warp_sum(fy);
  fz = gb_warp_sum(fz);
  if (active && lane == 0) {
    T* f = forces + 3 * (base + i);
    f[0] = (T)((double)f[0] + fx);
    f[1] = (T)((double)f[1] + fy);
    f[2] = (T)((double)f[2] + fz);
  }
}

}  // namespace tmd
