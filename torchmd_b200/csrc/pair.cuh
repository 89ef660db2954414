// pair.cuh -- the non-bonded pair kernel (K3): LJ (+switch), Coulomb / reaction
// field, repulsion, repulsionCG over the full Verlet list.
//
// Replaces, per step and replica, the reference's all-pairs distance pass, cutoff
// mask, per-term evaluation and index_add_ scatter (forces.py:264-319, 381-491).
//
// Mapping: one warp per atom (sorted order), lanes stride over the atom's
// neighbour row.  Row reads are coalesced 128-byte lines; partner records are
// 16-byte gathers that hit L1/L2 because atoms are sorted by cell.  Every pair is
// seen from both sides (full list), so forces need no atomics and no scatter:
// each warp reduces its atom's force with shuffles and writes it once.  The
// cutoff decision uses the reference's exact fp32 predicate (physics.cuh).
#pragma once
#include "context.cuh"
#include "ptx.cuh"

namespace tmd {

#ifndef PAIR_WARPS_N
#define PAIR_WARPS_N 8
#endif
constexpr int PAIR_WARPS = PAIR_WARPS_N;
#ifndef PAIR_MINBLOCKS
#define PAIR_MINBLOCKS 6  // CTAs per SM the register allocation must allow: 40 regs, a neighbour loop without spills on sm_90a
#endif

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-level sum of one double per thread -> atomicAdd into *dst by thread 0.
template <int NWARPS>
__device__ __forceinline__ void block_accumulate(double v, double* dst, double* smem /*NWARPS*/) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < NWARPS; ++w) t += smem[w];
    if (t != 0.0) atomicAdd(dst, t);
  }
}

// ENERGY   also accumulate the per-term energies (only the last step of a fused run needs them)
// PERIODIC minimum image on; SAFE: guard-free minimum image (see min_image_fast)
// MODE     0 = pair terms selected at run time, 1 = LJ+switch + reaction-field Coulomb,
//          2 = pair terms selected at run time with real-space Ewald electrostatics (particle-mesh Ewald)
template <bool ENERGY, bool PERIODIC, bool SAFE, int MODE>
__global__ void __launch_bounds__(PAIR_WARPS * 32, PAIR_MINBLOCKS)
k_pair(DeviceState S, float* __restrict__ forces, double* __restrict__ energies) {
  const int r = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int kk = blockIdx.x * PAIR_WARPS + (threadIdx.x >> 5);
  const int N = S.natoms;
  const size_t base = (size_t)r * N;
  const PairParams pp = S.pp;
  float e_el = 0.f, e_lj = 0.f, e_rep = 0.f, e_cg = 0.f;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[0] += 1;  // next call: other flag

  if (kk < S.own_n) {
    // whole system: rows in sorted order; decomposed run: the rows of the owned atoms
    const int k = S.own_all ? kk : S.inv[base + S.own_lo + kk];
    const float4* __restrict__ xq = S.xq_s + (size_t)r * (N + 1);  // (record N is the NaN sentinel the list build pads rows with)
    const int* __restrict__ row = S.nbr + (base + k) * (size_t)S.row_cap;
    const int n = S.nnbr[base + k];
    const float4 pi = xq[k];
    const int ti = S.type_s[base + k] * S.ntypes;
    const bool need_ab = MODE == 1 ? true : (pp.terms & (T_LJ | T_REP | T_REPCG)) != 0;
    float Lx = 0.f, Ly = 0.f, Lz = 0.f, iLx = 0.f, iLy = 0.f, iLz = 0.f;
    if (PERIODIC) {
      const Grid* g = S.grid + r;
      Lx = g->L[0]; Ly = g->L[1]; Lz = g->L[2];
      iLx = g->invL[0]; iLy = g->invL[1]; iLz = g->invL[2];
    }
    float fx = 0.f, fy = 0.f, fz = 0.f;

    // One interaction of atom i with a listed partner.  A list entry carries the partner's
    // sorted index in its low 24 bits and its atom type in the high 8 (packed at build
    // time), so the LJ table row is known without a second gather; `pj` is the partner's
    // position/charge record.
    auto interact = [&](int entry, const float4 pj) {
      const float dx0 = sub_rn(pi.x, pj.x), dy0 = sub_rn(pi.y, pj.y), dz0 = sub_rn(pi.z, pj.z);
      float wx = dx0, wy = dy0, wz = dz0;
      float rx = 0.f, ry = 0.f, rz = 0.f;
      if (PERIODIC) {
        if (SAFE) {
          wx = min_image_fast(dx0, Lx, iLx, rx);
          wy = min_image_fast(dy0, Ly, iLy, ry);
          wz = min_image_fast(dz0, Lz, iLz, rz);
        } else {
          wx = min_image_exact(dx0, Lx, iLx, rx);
          wy = min_image_exact(dy0, Ly, iLy, ry);
          wz = min_image_exact(dz0, Lz, iLz, rz);
        }
      }
      float s = norm2_ref(wx, wy, wz);  // the reference's own rounding: decides in/out
      if (s <= pp.s_max) {
        if (PERIODIC && (rx != 0.f || ry != 0.f || rz != 0.f)) {
          // straddles the box: the VALUES get the bits fl(pi-pj) dropped and the unrounded image
          // shift L*n (physics.cuh, straddle_value)
          wx = straddle_value(pi.x, pj.x, dx0, Lx, rx);
          wy = straddle_value(pi.y, pj.y, dy0, Ly, ry);
          wz = straddle_value(pi.z, pj.z, dz0, Lz, rz);
          s = wx * wx + wy * wy + wz * wz;
        }
        float2 ab = make_float2(0.f, 0.f);
        if (need_ab) ab = __ldg(S.AB + ti + (entry >> 24));
        float rinv;
        const float dedr = pair_terms<MODE>(pp, s, pi.w * pj.w, ab.x, ab.y, e_el, e_lj, e_rep, e_cg, rinv);
        const float c = dedr * rinv;  // force on i is -unit*dE/dr = -(w/r) dE/dr
        fx -= wx * c;
        fy -= wy * c;
        fz -= wz * c;
      }
    };
    // Lanes stride the row two entries per iteration.  The entries of the NEXT iteration are
    // loaded before the current pairs are computed (the row streams from HBM once per step,
    // evict-first); partner records are gathered at use and the latency is covered by
    // occupancy: this simple loop at 40 registers (6 CTAs/SM) rather than a deeper software
    // pipeline that needs 56-64 registers.
    {
      int e = lane;
      int j0 = (e < n) ? __ldcs(row + e) : -1;
      int j1 = (e + 32 < n) ? __ldcs(row + e + 32) : -1;
      while (e < n) {
        const int jn0 = (e + 64 < n) ? __ldcs(row + e + 64) : -1;
        const int jn1 = (e + 96 < n) ? __ldcs(row + e + 96) : -1;
        if (j0 >= 0) interact(j0, xq[j0 & 0xffffff]);
        if (j1 >= 0) interact(j1, xq[j1 & 0xffffff]);
        j0 = jn0;
        j1 = jn1;
        e += 64;
      }
    }
    fx = warp_sum(fx);
    fy = warp_sum(fy);
    fz = warp_sum(fz);
    if (lane == 0) {
      float* f = forces + (base + S.perm[base + k]) * 3;
      f[0] = fx;
      f[1] = fy;
      f[2] = fz;
    }
  }
  if (ENERGY) {
    __shared__ double red[PAIR_WARPS];
    double* E = energies + (size_t)r * TMD_NUM_ENERGIES;
    const uint32_t terms = MODE == 1 ? (T_LJ | T_ELEC) : pp.terms;
    // every pair is visited from both of its atoms
    if (terms & T_ELEC) block_accumulate<PAIR_WARPS>(0.5 * (double)e_el, E + TMD_E_ELECTROSTATICS, red);
    if (terms & T_LJ) block_accumulate<PAIR_WARPS>(0.5 * (double)e_lj, E + TMD_E_LJ, red);
    if (terms & T_REP) block_accumulate<PAIR_WARPS>(0.5 * (double)e_rep, E + TMD_E_REPULSION, red);
    if (terms & T_REPCG) block_accumulate<PAIR_WARPS>(0.5 * (double)e_cg, E + TMD_E_REPULSIONCG, red);
  }
}

// ---- periodic boxes: fixed-point separations -------------------------------------------
// Same mapping and list as k_pair.  The partner records hold fixed-point coordinates
// (physics.cuh, fx_encode): the separation is one integer subtraction per component --
// minimum image included, exact to L/2^32 -- instead of the reference's rounded
// subtract / multiply / round / multiply / subtract chain, and pairs that straddle the box
// need no compensation.  The decision stays the reference's: outside the band
// s_max -+ margin the two squared distances provably agree; inside it (about 1e-4 of the
// pairs) the reference arithmetic is re-done on the original positions.
// SMALLT: the LJ table (<= 16 types) is staged in shared memory.
#ifndef FX_SMALLT_MAX_N
#define FX_SMALLT_MAX_N 16  // (tests build a variant with a smaller limit to reach the global-table path with few types)
#endif
constexpr int FX_SMALLT_MAX = FX_SMALLT_MAX_N;
constexpr int FX_PLANE_BYTES = FX_SMALLT_MAX * FX_SMALLT_MAX * 4;  // A plane, then B plane, in the packed kernels' staged table
#ifndef PAIR_FX_MINBLOCKS
#define PAIR_FX_MINBLOCKS 5  // 48 registers: at 40 (6 CTAs/SM) ptxas for sm_90a spills inside the neighbour loop
#endif

// Partner record of a replica's fixed-point array at byte offset `off` from `base` (an
// integer the compiler cannot see through, so the replica's base stays in a register pair
// instead of being re-derived per pair).
__device__ __forceinline__ int4 fx_record(unsigned long long base, unsigned off) { return ldg_s32x4(base + off); }

template <bool ENERGY, int MODE, bool SMALLT>
__global__ void __launch_bounds__(PAIR_WARPS * 32, PAIR_FX_MINBLOCKS)
k_pair_fx(DeviceState S, float* __restrict__ forces, double* __restrict__ energies) {
  const int r = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int kk = blockIdx.x * PAIR_WARPS + (threadIdx.x >> 5);
  const int N = S.natoms;
  const size_t base = (size_t)r * N;
  const PairParams pp = S.pp;
  float e_el = 0.f, e_lj = 0.f, e_rep = 0.f, e_cg = 0.f;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[0] += 1;  // next call: other flag

  __shared__ float2 ab_s[SMALLT ? FX_SMALLT_MAX * FX_SMALLT_MAX : 1];
  if (SMALLT) {
    static_assert(FX_SMALLT_MAX * FX_SMALLT_MAX <= PAIR_WARPS * 32, "one table entry per thread");
    if (S.AB && (int)threadIdx.x < S.ntypes * S.ntypes) ab_s[threadIdx.x] = S.AB[threadIdx.x];  // no table without an LJ-type term
    TMD_KEEP_STORES();  // the table is read back through lds_* below
    __syncthreads();
  }

  if (kk < S.own_n) {
    const int k = S.own_all ? kk : S.inv[base + S.own_lo + kk];
    const int4* __restrict__ xf = S.xf_s + (size_t)r * (N + 1);
    unsigned long long xf_base = reinterpret_cast<unsigned long long>(xf);
    TMD_PIN_L(xf_base);
    const int* __restrict__ row = S.nbr + (base + k) * (size_t)S.row_cap;
    const int n = S.nnbr[base + k];
    const int4 pi = xf[k];
    const float qi = __int_as_float(pi.w);
    const int ti = S.type_s[base + k] * S.ntypes;
    const smem_addr ab_row = smem_address(ab_s) + (unsigned)ti * 8u;  // this atom's row of the staged table
    const bool need_ab = MODE == 1 ? true : (pp.terms & (T_LJ | T_REP | T_REPCG)) != 0;
    const Grid* g = S.grid + r;
    const float ux = g->fx_unit[0], uy = g->fx_unit[1], uz = g->fx_unit[2];
    // decision band around the reference's threshold; a non-finite coordinate somewhere
    // (margin = inf) sends every pair to the reference arithmetic
    const float margin = fmaf(g->fx_c1, __int_as_float(S.flags[r * F_COUNT + F_PMAX]), g->fx_c0);
    const float s_hi = pp.s_max + margin, s_lo = pp.s_max - margin;
    float fx = 0.f, fy = 0.f, fz = 0.f;

    float s_skipped = INFINITY;  // smallest squared distance not taken below: <= s_hi means a pair sits in the decision band
    auto accumulate = [&](int entry, float wx, float wy, float wz, float s, float qj) {
      float2 ab = make_float2(0.f, 0.f);
      if (need_ab) {
        if (SMALLT) {
          ab = lds_f32x2(ab_row + (((unsigned)entry >> 24) << 3));
        } else {
          ab = __ldg(S.AB + ti + (entry >> 24));
        }
      }
      float rinv;
      const float dedr = pair_terms<MODE>(pp, s, qi * qj, ab.x, ab.y, e_el, e_lj, e_rep, e_cg, rinv);
      const float c = dedr * rinv;  // force on i is -unit*dE/dr = -(w/r) dE/dr
      fx -= wx * c;
      fy -= wy * c;
      fz -= wz * c;
    };
    auto interact = [&](int entry, const int4 pj) {
      const float wx = fx_delta(pi.x, pj.x, ux), wy = fx_delta(pi.y, pj.y, uy), wz = fx_delta(pi.z, pj.z, uz);
      const float s = fmaf(wz, wz, fmaf(wy, wy, wx * wx));
      if (s < s_lo) accumulate(entry, wx, wy, wz, s, __int_as_float(pj.w));
      else s_skipped = fminf(s_skipped, s);
    };
    {
      int e = lane;
      int j0 = (e < n) ? __ldcs(row + e) : -1;
      int j1 = (e + 32 < n) ? __ldcs(row + e + 32) : -1;
      while (e < n) {
        const int jn0 = (e + 64 < n) ? __ldcs(row + e + 64) : -1;
        const int jn1 = (e + 96 < n) ? __ldcs(row + e + 96) : -1;
        if (j0 >= 0) interact(j0, fx_record(xf_base, ((unsigned)j0 << 4) & 0x0ffffff0u));
        if (j1 >= 0) interact(j1, fx_record(xf_base, ((unsigned)j1 << 4) & 0x0ffffff0u));
        j0 = jn0;
        j1 = jn1;
        e += 64;
      }
    }
    if (__any_sync(0xffffffffu, s_skipped <= s_hi)) {
      // rare (a few percent of the rows): re-scan the row and give the pairs inside the band
      // the reference's own decision on the original positions
      const float4* __restrict__ xq = S.xq_s + (size_t)r * (N + 1);
      for (int e = lane; e < n; e += 32) {
        const int entry = row[e];
        const int j = entry & 0xffffff;
        const int4 pj = xf[j];
        const float wx = fx_delta(pi.x, pj.x, ux), wy = fx_delta(pi.y, pj.y, uy), wz = fx_delta(pi.z, pj.z, uz);
        const float s = fmaf(wz, wz, fmaf(wy, wy, wx * wx));
        if (!(s < s_lo) && s <= s_hi) {
          const float4 a = xq[k], b = xq[j];
          if (ref_inside(a.x, a.y, a.z, b.x, b.y, b.z, g->L[0], g->L[1], g->L[2], g->invL[0], g->invL[1],
                         g->invL[2], pp.s_max))
            accumulate(entry, wx, wy, wz, s, __int_as_float(pj.w));
        }
      }
    }
    fx = warp_sum(fx);
    fy = warp_sum(fy);
    fz = warp_sum(fz);
    if (lane == 0) {
      float* f = forces + (base + S.perm[base + k]) * 3;
      f[0] = fx;
      f[1] = fy;
      f[2] = fz;
    }
  }
  if (ENERGY) {
    __shared__ double red[PAIR_WARPS];
    double* E = energies + (size_t)r * TMD_NUM_ENERGIES;
    const uint32_t terms = MODE == 1 ? (T_LJ | T_ELEC) : pp.terms;
    if (terms & T_ELEC) block_accumulate<PAIR_WARPS>(0.5 * (double)e_el, E + TMD_E_ELECTROSTATICS, red);
    if (terms & T_LJ) block_accumulate<PAIR_WARPS>(0.5 * (double)e_lj, E + TMD_E_LJ, red);
    if (terms & T_REP) block_accumulate<PAIR_WARPS>(0.5 * (double)e_rep, E + TMD_E_REPULSION, red);
    if (terms & T_REPCG) block_accumulate<PAIR_WARPS>(0.5 * (double)e_cg, E + TMD_E_REPULSIONCG, red);
  }
}

// ---- fixed-point separations + fp32x2 arithmetic ---------------------------------------------
// k_pair_fx for every combination of the "lj" and "electrostatics" terms (with or without
// switching / reaction field; <= 16 atom types; explicit-force convention) with the two list
// entries a lane handles per iteration evaluated TOGETHER in fp32x2 operations (physics.cuh,
// pair_coef2): one arithmetic chain for two partners, with the signs arranged so that no
// negation is needed.  Decisions, band handling and list layout are those of k_pair_fx; a
// partner that is not taken contributes through a zeroed coefficient.
#ifndef PAIR_FX2_MINBLOCKS
#define PAIR_FX2_MINBLOCKS 4  // 64 registers: no spills in the loop
#endif

// (A_0, A_1), (B_0, B_1) of two partners: from the staged planes (<= 16 types) or from the table in global memory
template <bool SMALLT>
__device__ __forceinline__ void lj_pair_entries(smem_addr ab_row, const float2* __restrict__ ab_global, bool lj_on, unsigned en0,
                                                unsigned en1, F2& A, F2& B) {
  if (SMALLT) {
    const smem_addr a0 = ab_row + ((en0 >> 24) << 2), a1 = ab_row + ((en1 >> 24) << 2);
    A = f2(lds_f32(a0), lds_f32(a1));
    B = f2(lds_f32_at<FX_PLANE_BYTES>(a0), lds_f32_at<FX_PLANE_BYTES>(a1));
  } else {
    const float2 v0 = __ldg(ab_global + (en0 >> 24)), v1 = __ldg(ab_global + (en1 >> 24));
    A = lj_on ? f2(v0.x, v1.x) : f2(0.f);  // (the staged planes are zeroed instead when the term is off)
    B = lj_on ? f2(v0.y, v1.y) : f2(0.f);
  }
}

template <bool ENERGY, bool SMALLT, bool EW>
__device__ __forceinline__ void pair_fx2_body(const DeviceState& S, const SwitchConsts& sc, float* __restrict__ forces,
                                              double* __restrict__ energies) {
  const int r = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int kk = blockIdx.x * PAIR_WARPS + (threadIdx.x >> 5);
  const int N = S.natoms;
  const size_t base = (size_t)r * N;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[0] += 1;  // next call: other flag

  // LJ table staged as two planes (A, B): the packed operands (A_0, A_1), (B_0, B_1) of the two
  // partners are then loaded straight into register pairs
  __shared__ float ab_s[SMALLT ? 2 * FX_SMALLT_MAX * FX_SMALLT_MAX : 1];
  if (SMALLT && (int)threadIdx.x < S.ntypes * S.ntypes) {
    const float2 v = (S.pp.terms & T_LJ) ? S.AB[threadIdx.x] : make_float2(0.f, 0.f);  // term off: zero table
    ab_s[threadIdx.x] = v.x;
    ab_s[FX_SMALLT_MAX * FX_SMALLT_MAX + threadIdx.x] = v.y;
  }
  TMD_KEEP_STORES();
  __syncthreads();
  float e_el = 0.f, e_lj = 0.f;
  if (kk < S.own_n) {
  const int k = S.own_all ? kk : S.inv[base + S.own_lo + kk];
  const int4* __restrict__ xf = S.xf_s + (size_t)r * (N + 1);
  unsigned long long xf_base = reinterpret_cast<unsigned long long>(xf);
  TMD_PIN_L(xf_base);
  const int* __restrict__ row = S.nbr + (base + k) * (size_t)S.row_cap;
  const int n = S.nnbr[base + k];
  const int4 pi = xf[k];
  float nqi = (S.pp.terms & T_ELEC) ? -__int_as_float(pi.w) : 0.f;  // term off: no charge
  if (!ENERGY) TMD_PIN_F(nqi);  // (otherwise the select is redone from the constant bank for every pair; the energy variant has no register to spare)
  const int ti = S.type_s[base + k] * S.ntypes;
  smem_addr ab_row = smem_address(ab_s) + (unsigned)ti * 4u;
  TMD_PIN_R(ab_row);  // keep it in a register (otherwise re-derived from the CTA's shared window per pair)
  const float2* __restrict__ ab_global = S.AB + ti;  // used when the table is not staged
  const Grid* g = S.grid + r;
  const F2 ux = f2(g->fx_unit[0]), uy = f2(g->fx_unit[1]), uz = f2(g->fx_unit[2]);
  const float margin = fmaf(g->fx_c1, __int_as_float(S.flags[r * F_COUNT + F_PMAX]), g->fx_c0);
  const float s_hi = S.pp.s_max + margin, s_lo = S.pp.s_max - margin;
  // d = fl(s - s_lo) has the sign of s - s_lo, and fl is monotone: s <= s_hi implies d <= fl(s_hi - s_lo).  For
  // d >= +0 the bit pattern orders like the value and a negative d has the top bit set, so the smallest d >= 0 seen is
  // the unsigned minimum of the bit patterns, and "some pair was inside the band" is one comparison after the loop.
  // An empty slot (record 0) may raise it spuriously, which only costs the pass.
  const F2 ns_lo = f2(-s_lo);
  unsigned d_min = 0xffffffffu;
  F2 FX = f2(0.f), FY = f2(0.f), FZ = f2(0.f);  // the two halves are added at the end
  F2 ELJ = f2(0.f), NEEL = f2(0.f);             // switched LJ energy / minus the Coulomb energy

  // two list entries evaluated together: slots e0 and e0 + 32 of the row
  // a slot past the end of the row holds entry 0 (reads record 0) and is masked by its position
  auto entry_at = [&](int e) { return (e < n) ? __ldcs(row + e) : 0; };
  auto record_of = [&](int j) { return ldg_s32x4(mad_wide_u32((unsigned)j & 0xffffffu, 16u, xf_base)); };
  auto pair2r = [&](int e0, int j0, int j1, const int4 p0, const int4 p1) {
    const bool v0 = e0 < n, v1 = e0 + 32 < n;
    const unsigned en0 = (unsigned)j0, en1 = (unsigned)j1;
    const F2 wx = f2_mul(f2((float)(int)((unsigned)pi.x - (unsigned)p0.x), (float)(int)((unsigned)pi.x - (unsigned)p1.x)), ux);
    const F2 wy = f2_mul(f2((float)(int)((unsigned)pi.y - (unsigned)p0.y), (float)(int)((unsigned)pi.y - (unsigned)p1.y)), uy);
    const F2 wz = f2_mul(f2((float)(int)((unsigned)pi.z - (unsigned)p0.z), (float)(int)((unsigned)pi.z - (unsigned)p1.z)), uz);
    const F2 s = f2_fma(wz, wz, f2_fma(wy, wy, f2_mul(wx, wx)));
    const F2 d = f2_add(s, ns_lo);
    const bool in0 = v0 && d.x < 0.f, in1 = v1 && d.y < 0.f;
    d_min = min(d_min, min(__float_as_uint(d.x), __float_as_uint(d.y)));
    if (in0 || in1) {
      F2 A, B;
      lj_pair_entries<SMALLT>(ab_row, ab_global, (S.pp.terms & T_LJ) != 0, en0, en1, A, B);
      const F2 nqq = f2_mul(f2(nqi), f2(__int_as_float(p0.w), __int_as_float(p1.w)));
      F2 elj, neel;
      F2 nc = pair_coef2<ENERGY, EW>(sc, s, nqq, A, B, f2(rsqrt_seed(s.x), rsqrt_seed(s.y)),
                                     f2(neg_rcp_seed(s.x), neg_rcp_seed(s.y)), elj, neel);
      nc = f2(in0 ? nc.x : 0.f, in1 ? nc.y : 0.f);  // a select, not a product: the other half may hold inf/NaN
      FX = f2_fma(wx, nc, FX);
      FY = f2_fma(wy, nc, FY);
      FZ = f2_fma(wz, nc, FZ);
      if (ENERGY) {
        ELJ = f2_add(ELJ, f2(in0 ? elj.x : 0.f, in1 ? elj.y : 0.f));
        NEEL = f2_add(NEEL, f2(in0 ? neel.x : 0.f, in1 ? neel.y : 0.f));
      }
    }
  };
  auto pair2 = [&](int e0, int j0, int j1) { pair2r(e0, j0, j1, record_of(j0), record_of(j1)); };
  {
    int e = lane;
    int j0 = entry_at(e), j1 = entry_at(e + 32);
    while (e < n) {
      const int jn0 = entry_at(e + 64), jn1 = entry_at(e + 96);
      pair2(e, j0, j1);
      j0 = jn0;
      j1 = jn1;
      e += 64;
    }
  }
  float fx = FX.x + FX.y, fy = FY.x + FY.y, fz = FZ.x + FZ.y;
  if (ENERGY) {
    e_lj = ELJ.x + ELJ.y;
    e_el = -(NEEL.x + NEEL.y);
  }
  if (__any_sync(0xffffffffu, d_min <= __float_as_uint(s_hi - s_lo))) {
    // pairs inside the decision band: the reference's own decision, scalar arithmetic
    const float4* __restrict__ xq = S.xq_s + (size_t)r * (N + 1);
    const PairParams pp = S.pp;
    const float qi = __int_as_float(pi.w);
    float e_rep = 0.f, e_cg = 0.f;
    for (int eb = lane; eb < n; eb += 32) {
      const int entry = row[eb];
      const int j = entry & 0xffffff;
      const int4 pj = xf[j];
      const float wx = fx_delta(pi.x, pj.x, ux.x), wy = fx_delta(pi.y, pj.y, uy.x), wz = fx_delta(pi.z, pj.z, uz.x);
      const float s = fmaf(wz, wz, fmaf(wy, wy, wx * wx));
      if (!(s < s_lo) && s <= s_hi) {
        const float4 a = xq[k], b = xq[j];
        if (ref_inside(a.x, a.y, a.z, b.x, b.y, b.z, g->L[0], g->L[1], g->L[2], g->invL[0], g->invL[1], g->invL[2],
                       pp.s_max)) {
          const float2 ab = __ldg(S.AB + ti + (entry >> 24));  // (pair_terms<0> ignores it when LJ is off)
          float rinv;
          const float dedr = pair_terms<EW ? 2 : 0>(pp, s, qi * __int_as_float(pj.w), ab.x, ab.y, e_el, e_lj, e_rep, e_cg, rinv);
          const float c = dedr * rinv;
          fx -= wx * c;
          fy -= wy * c;
          fz -= wz * c;
        }
      }
    }
  }
  fx = warp_sum(fx);
  fy = warp_sum(fy);
  fz = warp_sum(fz);
  if (lane == 0) {
    float* f = forces + (base + S.perm[base + k]) * 3;
    f[0] = fx;
    f[1] = fy;
    f[2] = fz;
  }
  }  // kk < own_n
  if (ENERGY) {
    __shared__ double red[PAIR_WARPS];
    double* E = energies + (size_t)r * TMD_NUM_ENERGIES;
    block_accumulate<PAIR_WARPS>(0.5 * (double)e_el, E + TMD_E_ELECTROSTATICS, red);  // every pair is seen from both atoms
    block_accumulate<PAIR_WARPS>(0.5 * (double)e_lj, E + TMD_E_LJ, red);
  }
}
template <bool ENERGY, bool SMALLT>
__global__ void __launch_bounds__(PAIR_WARPS * 32, PAIR_FX2_MINBLOCKS)
k_pair_fx2(DeviceState S, SwitchConsts sc, float* __restrict__ forces, double* __restrict__ energies) {
  pair_fx2_body<ENERGY, SMALLT, false>(S, sc, forces, energies);
}
// particle-mesh Ewald contexts: real-space Ewald electrostatics (sc from make_switch_consts_ewald)
template <bool ENERGY, bool SMALLT>
__global__ void __launch_bounds__(PAIR_WARPS * 32, PAIR_FX2_MINBLOCKS)
k_pair_fx2_ew(DeviceState S, SwitchConsts sc, float* __restrict__ forces, double* __restrict__ energies) {
  pair_fx2_body<ENERGY, SMALLT, true>(S, sc, forces, energies);
}

// ---- systems without a box: fp32x2 arithmetic on the float records -------------------------
// Without periodicity the reference's separation is the plain rounded difference p_i - p_j and
// its squared length fma(z,z,fma(y,y,x*x)) -- both exist as packed operations with identical
// rounding per half, so the cutoff decision of two partners is taken exactly, together, with
// no band and no second pass.  Same term coverage and table staging as k_pair_fx2.
template <bool ENERGY, bool SMALLT>
__global__ void __launch_bounds__(PAIR_WARPS * 32, PAIR_FX2_MINBLOCKS)
k_pair2_open(DeviceState S, SwitchConsts sc, float* __restrict__ forces, double* __restrict__ energies) {
  const int r = blockIdx.y;
  const int lane = threadIdx.x & 31;
  const int kk = blockIdx.x * PAIR_WARPS + (threadIdx.x >> 5);
  const int N = S.natoms;
  const size_t base = (size_t)r * N;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) S.counters[0] += 1;  // next call: other flag

  __shared__ float ab_s[SMALLT ? 2 * FX_SMALLT_MAX * FX_SMALLT_MAX : 1];
  if (SMALLT && (int)threadIdx.x < S.ntypes * S.ntypes) {
    const float2 v = (S.pp.terms & T_LJ) ? S.AB[threadIdx.x] : make_float2(0.f, 0.f);
    ab_s[threadIdx.x] = v.x;
    ab_s[FX_SMALLT_MAX * FX_SMALLT_MAX + threadIdx.x] = v.y;
  }
  TMD_KEEP_STORES();
  __syncthreads();
  F2 ELJ = f2(0.f), NEEL = f2(0.f);
  if (kk < S.own_n) {
    const int k = S.own_all ? kk : S.inv[base + S.own_lo + kk];
    const float4* __restrict__ xq = S.xq_s + (size_t)r * (N + 1);
    const int* __restrict__ row = S.nbr + (base + k) * (size_t)S.row_cap;
    const int n = S.nnbr[base + k];
    const float4 pi = xq[k];
    const float nqi = (S.pp.terms & T_ELEC) ? -pi.w : 0.f;
    const int ti = S.type_s[base + k] * S.ntypes;
    smem_addr ab_row = smem_address(ab_s) + (unsigned)ti * 4u;
  TMD_PIN_R(ab_row);  // keep it in a register (otherwise re-derived from the CTA's shared window per pair)
    const float2* __restrict__ ab_global = S.AB + ti;
    const float s_max = S.pp.s_max;
    F2 FX = f2(0.f), FY = f2(0.f), FZ = f2(0.f);

    int e = lane;
    int j0 = (e < n) ? __ldcs(row + e) : -1;
    int j1 = (e + 32 < n) ? __ldcs(row + e + 32) : -1;
    while (e < n) {
      const int jn0 = (e + 64 < n) ? __ldcs(row + e + 64) : -1;
      const int jn1 = (e + 96 < n) ? __ldcs(row + e + 96) : -1;
      const bool v0 = j0 >= 0, v1 = j1 >= 0;
      const unsigned en0 = v0 ? (unsigned)j0 : 0u, en1 = v1 ? (unsigned)j1 : 0u;  // an empty slot reads record 0 and is masked
      const float4 p0 = xq[en0 & 0xffffffu], p1 = xq[en1 & 0xffffffu];
      // the reference's rounded differences and squared length (forces.py:368-372), two partners per operation
      const F2 wx = f2_add(f2(pi.x), f2(-p0.x, -p1.x));
      const F2 wy = f2_add(f2(pi.y), f2(-p0.y, -p1.y));
      const F2 wz = f2_add(f2(pi.z), f2(-p0.z, -p1.z));
      const F2 s = f2_fma(wz, wz, f2_fma(wy, wy, f2_mul(wx, wx)));
      const bool in0 = v0 && s.x <= s_max, in1 = v1 && s.y <= s_max;
      if (in0 || in1) {
        F2 A, B;
        lj_pair_entries<SMALLT>(ab_row, ab_global, (S.pp.terms & T_LJ) != 0, en0, en1, A, B);
        const F2 nqq = f2_mul(f2(nqi), f2(p0.w, p1.w));
        F2 elj, neel;
        F2 nc = pair_coef2<ENERGY>(sc, s, nqq, A, B, f2(rsqrt_seed(s.x), rsqrt_seed(s.y)),
                                   f2(neg_rcp_seed(s.x), neg_rcp_seed(s.y)), elj, neel);
        nc = f2(in0 ? nc.x : 0.f, in1 ? nc.y : 0.f);
        FX = f2_fma(wx, nc, FX);
        FY = f2_fma(wy, nc, FY);
        FZ = f2_fma(wz, nc, FZ);
        if (ENERGY) {
          ELJ = f2_add(ELJ, f2(in0 ? elj.x : 0.f, in1 ? elj.y : 0.f));
          NEEL = f2_add(NEEL, f2(in0 ? neel.x : 0.f, in1 ? neel.y : 0.f));
        }
      }
      j0 = jn0;
      j1 = jn1;
      e += 64;
    }
    const float fx = warp_sum(FX.x + FX.y), fy = warp_sum(FY.x + FY.y), fz = warp_sum(FZ.x + FZ.y);
    if (lane == 0) {
      float* f = forces + (base + S.perm[base + k]) * 3;
      f[0] = fx;
      f[1] = fy;
      f[2] = fz;
    }
  }
  if (ENERGY) {
    __shared__ double red[PAIR_WARPS];
    double* E = energies + (size_t)r * TMD_NUM_ENERGIES;
    block_accumulate<PAIR_WARPS>(-0.5 * (double)(NEEL.x + NEEL.y), E + TMD_E_ELECTROSTATICS, red);  // every pair is seen from both atoms
    block_accumulate<PAIR_WARPS>(0.5 * (double)(ELJ.x + ELJ.y), E + TMD_E_LJ, red);
  }
}

}  // namespace tmd
