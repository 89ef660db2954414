// pme.cuh -- reciprocal space of particle-mesh Ewald (smooth PME, Essmann et al. 1995), per replica (blockIdx.y),
// templated on the precision T of the FFT grid (float or double).  The chain of one force call:
//   k_pme_spread       charges onto the grid with order-5 B-splines, 64-bit fixed-point atomics (order-independent sum)
//   k_pme_fft<FIRST>   z lines: integer grid -> T (and zeroed for the next call), forward DFT
//   k_pme_fft<FWD>     y lines, forward
//   k_pme_fft<CONV>    x lines: forward, times the influence function G(m) (energy 1/2 sum G |S|^2 on energy calls),
//                      inverse
//   k_pme_fft<INV>     y lines, then z lines, inverse: the grid holds phi = dE/dQ
//   k_pme_gather       per atom (no atomics): -q grad(theta) . phi, plus the exclusion correction, ADDED to the forces
//                      (on the cluster path to the slot-order accumulators of the pair kernel)
// Grid layout [x][y][z], z fastest.  DFTs are unnormalised (forward e^-, inverse e^+), so phi = IDFT(G DFT(Q)) needs no
// scale.  The 1D transforms are mixed-radix 2/3/5 Stockham passes in shared memory, a block per group of lines.
#pragma once
#include <algorithm>

#include "context.cuh"

namespace tmd {

constexpr int PME_ORDER = 5;
constexpr int PME_MAX_N = 512;  // largest grid dimension the line kernels hold in shared memory
constexpr int PME_THREADS = 128;

template <typename T>
struct Cplx {
  T x, y;
};

struct PmeArgs {
  int natoms;
  int K[3];
  long long ktot;                 // K[0] * K[1] * K[2]
  double scale, inv_scale;        // fixed point of the charge grid: value * 2^e
  const double* q;                // (N) charge * sqrt(coulomb constant)
  const double* L;                // (R,3) box lengths
  unsigned long long* qgrid;      // (R, ktot) fixed-point charge grid; all zero between calls
  void* cgrid;                    // (R, ktot) Cplx<T>
  const double* tw;               // twiddles e^{-2 pi i t / K_d}: K[0] + K[1] + K[2] (cos, sin) pairs
  const void* infl;               // (R, ktot) T: influence function G(m)
  const double* econst;           // (R) self + neutralising-background energy
  const int* excl_ptr;            // CSR exclusions (original indices, both directions); null without any
  const int* excl_idx;
  double alpha, beta;             // Ewald splitting parameter, 2 alpha / sqrt(pi)
  // cluster path (fp32): the gather adds into the slot-order accumulators the pair kernel filled, which every later
  // kernel (unsort, bonded fold, fused half-kick) brings home; null on the full rows
  float4* cl_f;                   // [rep * cl_stride + slot]
  const int* cl_inv;              // [rep * natoms + atom] -> slot
  long long cl_stride;            // slots + 1
};

// Order-5 B-spline weights th[j] of grid point floor(u) + j and their derivatives d th / du (oracle/pme.py, bspline).
__host__ __device__ __forceinline__ void pme_bspline(double w, double th[PME_ORDER], double dth[PME_ORDER]) {
  const int n = PME_ORDER;
  th[n - 1] = 0.0;
  th[0] = 1.0 - w;
  th[1] = w;
#pragma unroll
  for (int j = 3; j < n; ++j) {
    const double div = 1.0 / (j - 1);
    th[j - 1] = div * w * th[j - 2];
#pragma unroll
    for (int k = 1; k < j - 1; ++k) th[j - k - 1] = div * ((w + k) * th[j - k - 2] + (j - k - w) * th[j - k - 1]);
    th[0] = div * (1.0 - w) * th[0];
  }
  dth[0] = -th[0];
#pragma unroll
  for (int k = 1; k < n; ++k) dth[k] = th[k - 1] - th[k];
  const double div = 1.0 / (n - 1);
  th[n - 1] = div * w * th[n - 2];
#pragma unroll
  for (int k = 1; k < n - 1; ++k) th[n - k - 1] = div * ((w + k) * th[n - k - 2] + (n - k - w) * th[n - k - 1]);
  th[0] = div * (1.0 - w) * th[0];
}

// Grid coordinate u = K * frac(x / L) in fp64: first point and spline weights along one axis.
__device__ __forceinline__ int pme_axis(double x, double L, int K, double th[PME_ORDER], double dth[PME_ORDER]) {
  double f = x / L;
  f -= floor(f);
  double u = f * K;
  int i0 = (int)floor(u);
  double w = u - i0;
  if (i0 >= K) {  // f rounded up to 1
    i0 = 0;
    w = 0.0;
  }
  pme_bspline(w, th, dth);
  return i0;
}

template <typename T>
__global__ void __launch_bounds__(PME_THREADS) k_pme_spread(PmeArgs a, const T* __restrict__ pos) {
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.natoms) return;
  const size_t ai = (size_t)r * a.natoms + i;
  const double q = a.q[i];
  if (q == 0.0) return;
  double th[3][PME_ORDER], dth[PME_ORDER];
  int i0[3];
  for (int d = 0; d < 3; ++d) i0[d] = pme_axis((double)pos[3 * ai + d], a.L[3 * r + d], a.K[d], th[d], dth);
  unsigned long long* g = a.qgrid + (size_t)r * a.ktot;
  for (int x = 0; x < PME_ORDER; ++x) {
    const int gx = (i0[0] + x) % a.K[0];
    const double qx = q * th[0][x] * a.scale;
    for (int y = 0; y < PME_ORDER; ++y) {
      const int gy = (i0[1] + y) % a.K[1];
      const double qxy = qx * th[1][y];
      const size_t row = ((size_t)gx * a.K[1] + gy) * a.K[2];
      for (int z = 0; z < PME_ORDER; ++z) {
        const int gz = (i0[2] + z) % a.K[2];
        atomicAdd(g + row + gz, (unsigned long long)llrint(qxy * th[2][z]));  // two's complement: exact, any order
      }
    }
  }
}

enum { PME_FIRST = 0, PME_FWD = 1, PME_CONV = 2, PME_INV = 3 };

// Shared-memory capacity of one block, in complex values per buffer: a block transforms nl = pme_lines_per_block(n)
// lines at once, stored point-major (buf[t * nl + l]), so that along the strided axes the nl lines that are neighbours
// along z are read and written as contiguous runs.
template <typename T>
struct PmeCap {
  static constexpr int value = sizeof(T) == 8 ? 1024 : 2048;
};
// log2 of the lines per block: the largest power of two up to 32 that fits (one line along z, the contiguous axis)
template <typename T>
inline int pme_lines_log2(int n, int axis) {
  int lg = 0;
  while (axis != 2 && lg < 5 && (2 << lg) * n <= PmeCap<T>::value) ++lg;
  return lg;
}

// nl DFTs of length n in shared memory (a -> the returned buffer), sign -1 forward / +1 inverse.  Stockham autosort: a
// pass of radix R over Ns already-combined points, for j < n/R with k = j mod Ns,
//   v_r = a[j + r n/R] w^(k r n/(Ns R)),  V = DFT_R(v),  b[(j/Ns) Ns R + k + s Ns] = V_s.
// wt[t] = e^{-2 pi i t / n} (conjugated here for the inverse).
template <typename T>
__device__ Cplx<T>* pme_line_dft(Cplx<T>* a, Cplx<T>* b, int n, int lg, const Cplx<T>* wt, bool inverse) {
  const int nl = 1 << lg;
  int Ns = 1;
  int m = n;
  while (m > 1) {
    const int R = (m % 2 == 0) ? 2 : (m % 3 == 0) ? 3 : 5;
    m /= R;
    const int nr = n / R;
    const int step0 = n / (Ns * R);
    for (int w = threadIdx.x; w < nr * nl; w += blockDim.x) {
      const int l = w & (nl - 1), j = w >> lg;
      const int k = j % Ns;
      Cplx<T> v[5];
      const int step = k * step0;  // step * r < n
      v[0] = a[j * nl + l];
      for (int r = 1; r < R; ++r) {
        const Cplx<T> x = a[(j + r * nr) * nl + l];
        const Cplx<T> tw = wt[step * r];
        const T c = tw.x, s = inverse ? -tw.y : tw.y;
        v[r] = Cplx<T>{x.x * c - x.y * s, x.x * s + x.y * c};
      }
      Cplx<T>* out = b + ((j - k) * R + k) * nl + l;
      if (R == 2) {
        out[0] = Cplx<T>{v[0].x + v[1].x, v[0].y + v[1].y};
        out[Ns * nl] = Cplx<T>{v[0].x - v[1].x, v[0].y - v[1].y};
        continue;
      }
      for (int s_ = 0; s_ < R; ++s_) {
        Cplx<T> acc = v[0];
        int rs = 0;  // (r * s_) mod R
        for (int r = 1; r < R; ++r) {
          rs += s_;
          if (rs >= R) rs -= R;
          const Cplx<T> tw = wt[rs * nr];
          const T c = tw.x, s = inverse ? -tw.y : tw.y;
          acc.x += v[r].x * c - v[r].y * s;
          acc.y += v[r].x * s + v[r].y * c;
        }
        out[s_ * Ns * nl] = acc;
      }
    }
    __syncthreads();
    Cplx<T>* t = a;
    a = b;
    b = t;
    Ns *= R;
  }
  return a;
}

// Lines along `axis` (0 x, 1 y, 2 z), 2^lg per block (pme_lines_log2): blockIdx.x = group of lines, blockIdx.y =
// replica.
template <typename T, int KIND>
__global__ void __launch_bounds__(PME_THREADS) k_pme_fft(PmeArgs a, int axis, int lg, double* __restrict__ energies) {
  __shared__ Cplx<T> buf[2][PmeCap<T>::value];
  __shared__ Cplx<T> wt[PME_MAX_N];
  __shared__ double red[PME_THREADS / 32];
  const int nl = 1 << lg;
  const int r = blockIdx.y;
  const int n = a.K[axis];
  const int b = axis == 0 ? 1 : 0, c = axis == 2 ? 1 : 2;  // the other two axes, c the faster one
  const long long sK[3] = {(long long)a.K[1] * a.K[2], a.K[2], 1};
  const long long nlines = a.ktot / n;
  const long long stride = sK[axis];
  auto base_of = [&](long long line) { return (line / a.K[c]) * sK[b] + (line % a.K[c]) * sK[c]; };
  Cplx<T>* g = static_cast<Cplx<T>*>(a.cgrid) + (size_t)r * a.ktot;
  const double* tw = a.tw + 2 * (axis == 0 ? 0 : axis == 1 ? a.K[0] : a.K[0] + a.K[1]);
  const long long line0 = (long long)blockIdx.x * nl;
  for (int t = threadIdx.x; t < n; t += blockDim.x) wt[t] = Cplx<T>{(T)tw[2 * t], (T)tw[2 * t + 1]};
  for (int w = threadIdx.x; w < n * nl; w += blockDim.x) {
    const int l = w & (nl - 1), t = w >> lg;
    if (line0 + l >= nlines) continue;
    const long long e = base_of(line0 + l) + t * stride;
    if (KIND == PME_FIRST) {
      unsigned long long* qg = a.qgrid + (size_t)r * a.ktot + e;
      const long long v = (long long)*qg;
      *qg = 0ull;  // the next spread starts from zero
      buf[0][w] = Cplx<T>{(T)((double)v * a.inv_scale), T(0)};
    } else {
      buf[0][w] = g[e];
    }
  }
  __syncthreads();
  Cplx<T>* res = pme_line_dft<T>(buf[0], buf[1], n, lg, wt, KIND == PME_INV);
  if (KIND == PME_CONV) {
    const T* G = static_cast<const T*>(a.infl) + (size_t)r * a.ktot;
    double e = 0.0;
    for (int w = threadIdx.x; w < n * nl; w += blockDim.x) {
      const int l = w & (nl - 1), t = w >> lg;
      if (line0 + l >= nlines) continue;
      const T gm = G[base_of(line0 + l) + t * stride];
      const Cplx<T> s = res[w];
      if (energies) e += (double)gm * ((double)s.x * (double)s.x + (double)s.y * (double)s.y);
      res[w] = Cplx<T>{s.x * gm, s.y * gm};
    }
    if (energies) {
      for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
    }
    __syncthreads();
    if (energies && threadIdx.x == 0) {
      double s = 0.0;
      for (int w = 0; w < PME_THREADS / 32; ++w) s += red[w];
      s *= 0.5;
      if (blockIdx.x == 0) s += a.econst[r];
      atomicAdd(energies + (size_t)r * TMD_NUM_ENERGIES + TMD_E_ELECTROSTATICS, s);
    }
    Cplx<T>* other = (res == buf[0]) ? buf[1] : buf[0];
    res = pme_line_dft<T>(res, other, n, lg, wt, true);
  }
  for (int w = threadIdx.x; w < n * nl; w += blockDim.x) {
    const int l = w & (nl - 1), t = w >> lg;
    if (line0 + l < nlines) g[base_of(line0 + l) + t * stride] = res[w];
  }
}

// Per atom: reciprocal force -q sum_k phi(k) grad theta(k), and the exclusion correction -k qi qj erf(a r)/r of every
// excluded partner (minimum image, fp64; the energy of each pair is counted by its lower index), ADDED to forces.
template <typename T>
__global__ void __launch_bounds__(PME_THREADS) k_pme_gather(PmeArgs a, const T* __restrict__ pos, T* __restrict__ forces,
                                                          double* __restrict__ energies) {
  __shared__ double red[PME_THREADS / 32];
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double e = 0.0;
  if (i < a.natoms) {
    const size_t ai = (size_t)r * a.natoms + i;
    const double q = a.q[i];
    const double Lx = a.L[3 * r], Ly = a.L[3 * r + 1], Lz = a.L[3 * r + 2];
    const double xi = (double)pos[3 * ai], yi = (double)pos[3 * ai + 1], zi = (double)pos[3 * ai + 2];
    double fx = 0.0, fy = 0.0, fz = 0.0;
    if (q != 0.0) {
      double th[3][PME_ORDER], dth[3][PME_ORDER];
      const int x0 = pme_axis(xi, Lx, a.K[0], th[0], dth[0]);
      const int y0 = pme_axis(yi, Ly, a.K[1], th[1], dth[1]);
      const int z0 = pme_axis(zi, Lz, a.K[2], th[2], dth[2]);
      const Cplx<T>* g = static_cast<const Cplx<T>*>(a.cgrid) + (size_t)r * a.ktot;
      double gx = 0.0, gy = 0.0, gz = 0.0;
      for (int x = 0; x < PME_ORDER; ++x) {
        const int ix = (x0 + x) % a.K[0];
        for (int y = 0; y < PME_ORDER; ++y) {
          const int iy = (y0 + y) % a.K[1];
          const Cplx<T>* row = g + ((size_t)ix * a.K[1] + iy) * a.K[2];
          double sz = 0.0, dz = 0.0;
          for (int z = 0; z < PME_ORDER; ++z) {
            const double p = (double)row[(z0 + z) % a.K[2]].x;
            sz += p * th[2][z];
            dz += p * dth[2][z];
          }
          gx += dth[0][x] * th[1][y] * sz;
          gy += th[0][x] * dth[1][y] * sz;
          gz += th[0][x] * th[1][y] * dz;
        }
      }
      fx = -q * gx * (a.K[0] / Lx);
      fy = -q * gy * (a.K[1] / Ly);
      fz = -q * gz * (a.K[2] / Lz);
    }
    if (a.excl_ptr) {
      for (int p = a.excl_ptr[i]; p < a.excl_ptr[i + 1]; ++p) {
        const int j = a.excl_idx[p];
        const double qq = q * a.q[j];
        if (qq == 0.0) continue;
        const size_t aj = (size_t)r * a.natoms + j;
        double dx = xi - (double)pos[3 * aj], dy = yi - (double)pos[3 * aj + 1], dz = zi - (double)pos[3 * aj + 2];
        dx -= Lx * rint(dx / Lx);
        dy -= Ly * rint(dy / Ly);
        dz -= Lz * rint(dz / Lz);
        const double s = dx * dx + dy * dy + dz * dz;
        const double rr = sqrt(s), rinv = 1.0 / rr;
        const double ep = -qq * erf(a.alpha * rr) * rinv;
        if (j > i) e += ep;
        const double dedr = -(ep + qq * a.beta * exp(-a.alpha * a.alpha * s)) * rinv;
        const double c = -dedr * rinv;
        fx += c * dx;
        fy += c * dy;
        fz += c * dz;
      }
    }
    if (a.cl_f) {
      float4* f = a.cl_f + (size_t)r * a.cl_stride + a.cl_inv[ai];
      f->x = (float)((double)f->x + fx);
      f->y = (float)((double)f->y + fy);
      f->z = (float)((double)f->z + fz);
    } else {
      T* f = forces + 3 * ai;
      f[0] = (T)((double)f[0] + fx);
      f[1] = (T)((double)f[1] + fy);
      f[2] = (T)((double)f[2] + fz);
    }
  }
  if (energies) {
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int w = 0; w < PME_THREADS / 32; ++w) s += red[w];
      if (s != 0.0) atomicAdd(energies + (size_t)r * TMD_NUM_ENERGIES + TMD_E_ELECTROSTATICS, s);
    }
  }
}

// Influence function of replica blockIdx.y from its box a.L, alpha and the B-spline moduli |b(m)|^2 (mod: K[0] + K[1] +
// K[2] values, the grid's and not the box's, so uploaded once):
//   G(m) = exp(-pi^2 m^2 / alpha^2) / (pi V m^2 |b_x|^2 |b_y|^2 |b_z|^2),  G(0) = 0,
// with m_d = (index, folded to [-K/2, K/2]) / L_d.  Runs at finalisation and on every tmd_rescale_box.
template <typename T>
__global__ void __launch_bounds__(PME_THREADS) k_pme_influence(PmeArgs a, const double* __restrict__ mod) {
  const int r = blockIdx.y;
  const double L0 = a.L[3 * r], L1 = a.L[3 * r + 1], L2 = a.L[3 * r + 2];
  const double V = L0 * L1 * L2;
  T* G = static_cast<T*>(const_cast<void*>(a.infl)) + (size_t)r * a.ktot;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < a.ktot; idx += (long long)gridDim.x * blockDim.x) {
    const int z = (int)(idx % a.K[2]);
    const int y = (int)((idx / a.K[2]) % a.K[1]);
    const int x = (int)(idx / ((long long)a.K[1] * a.K[2]));
    const double mx = (x > a.K[0] / 2 ? x - a.K[0] : x) / L0;
    const double my = (y > a.K[1] / 2 ? y - a.K[1] : y) / L1;
    const double mz = (z > a.K[2] / 2 ? z - a.K[2] : z) / L2;
    const double m2 = mx * mx + my * my + mz * mz;
    const double den = M_PI * V * m2 * mod[x] * mod[a.K[0] + y] * mod[a.K[0] + a.K[1] + z];
    G[idx] = m2 > 0.0 ? (T)(exp(-M_PI * M_PI * m2 / (a.alpha * a.alpha)) / den) : T(0);
  }
}

}  // namespace tmd
