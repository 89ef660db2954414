// The line-DFT kernel of particle-mesh Ewald (torchmd_b200/csrc/pme.cuh, k_pme_fft) on the host SIMT interpreter, one
// line at a time -- TEST INFRASTRUCTURE for tests/test_pme_on_interpreter.py, which compares it with numpy.fft:
//   g++ -std=c++17 -O1 -fPIC -shared -ffp-contract=off -I tests/simt/stub -I torchmd_b200/csrc -o tests/simt/libpme_fft.so tests/simt/pme_fft.cpp
#include <cuda_runtime.h>

#include <vector>

#include "pme.cuh"

using namespace tmd;

template <typename T>
static void line_dft(int n, int inverse, double* data) {
  std::vector<Cplx<T>> g(n);
  for (int t = 0; t < n; ++t) g[t] = Cplx<T>{(T)data[2 * t], (T)data[2 * t + 1]};
  // a grid of 1 x 1 x n: the z twiddles follow the K[0] + K[1] = 2 entries of x and y
  std::vector<double> tw(2 * (2 + n), 0.0);
  for (int t = 0; t < n; ++t) {
    tw[2 * (2 + t)] = cos(2.0 * M_PI * t / n);
    tw[2 * (2 + t) + 1] = -sin(2.0 * M_PI * t / n);
  }
  PmeArgs a{};
  a.K[0] = a.K[1] = 1;
  a.K[2] = n;
  a.ktot = n;
  a.cgrid = g.data();
  a.tw = tw.data();
  simt::run_grid(dim3(1, 1), dim3(PME_THREADS), [&]() {
    if (inverse) k_pme_fft<T, PME_INV>(a, 2, 0, nullptr);
    else k_pme_fft<T, PME_FWD>(a, 2, 0, nullptr);
  });
  for (int t = 0; t < n; ++t) {
    data[2 * t] = (double)g[t].x;
    data[2 * t + 1] = (double)g[t].y;
  }
}

// data: n complex values (re, im interleaved), transformed in place; unnormalised, e^- forward, e^+ inverse
extern "C" int simt_pme_line_dft(int n, int bits, int inverse, double* data) {
  if (n < 1 || n > PME_MAX_N) return -1;
  if (bits == 64) line_dft<double>(n, inverse, data);
  else line_dft<float>(n, inverse, data);
  return 0;
}
