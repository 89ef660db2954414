// The influence-function kernel of particle-mesh Ewald (torchmd_b200/csrc/pme.cuh, k_pme_influence) on the host SIMT
// interpreter -- TEST INFRASTRUCTURE for tests/test_barostat_on_interpreter.py, which compares it with the host formula:
//   g++ -std=c++17 -O1 -fPIC -shared -ffp-contract=off -I tests/simt/stub -I torchmd_b200/csrc -o tests/simt/libpme_influence.so tests/simt/pme_influence.cpp
#include <cuda_runtime.h>

#include <vector>

#include "pme.cuh"

using namespace tmd;

// G (R, K0*K1*K2) of the boxes L (R,3) with moduli mod (K0 + K1 + K2), in fp64 (bits 64) or fp32 widened to fp64
extern "C" int simt_pme_influence(int R, const int* K, const double* L, double alpha, const double* mod, int bits, double* G) {
  PmeArgs a{};
  for (int d = 0; d < 3; ++d) a.K[d] = K[d];
  a.ktot = (long long)K[0] * K[1] * K[2];
  a.L = L;
  a.alpha = alpha;
  const size_t n = (size_t)R * a.ktot;
  if (bits == 64) {
    a.infl = G;
    simt::run_grid(dim3(3, R), dim3(PME_THREADS), [&]() { k_pme_influence<double>(a, mod); });
  } else {
    std::vector<float> g(n);
    a.infl = g.data();
    simt::run_grid(dim3(3, R), dim3(PME_THREADS), [&]() { k_pme_influence<float>(a, mod); });
    for (size_t i = 0; i < n; ++i) G[i] = (double)g[i];
  }
  return 0;
}
