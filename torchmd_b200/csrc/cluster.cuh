// cluster.cuh -- the cluster half-list path of the non-bonded pair loop.
//
// Replaces, like pair.cuh, the reference's all-pairs distance pass, cutoff mask, per-term evaluation
// and index_add_ scatter (forces.py:264-319, 381-491), for the production set-up: a cutoff, pair terms
// out of {lj, electrostatics}, explicit-force convention, <= CL_MAXT atom types, the whole system on
// one context.  Everything else keeps the full Verlet rows of neighbor.cuh / pair.cuh.
//
// Layout.  Atoms are sorted by cell row (cells of ~4 A; z-major, x fastest) and, inside a row, by x;
// every row is padded to a multiple of CL slots, so CL consecutive slots form an "i-cluster" that never
// straddles a row: a box of about 2.5 x 4 x 4 A.  The list of a cluster holds the slots of all atoms of
// LATER clusters within cutoff + skin of the cluster's bounding box (half list: each pair is listed
// once), one 32-bit entry each (24-bit slot, 8-bit atom type): ~340 entries per cluster of 4 in
// liquid water at 10 A, 34 MB for 100k atoms against 180 MB of full rows.  Partners with an excluded
// pair in the cluster, and the cluster's own atoms, sit in a short "masked" region with one mask byte
// per entry.
//
// Kernel k_cpair: one warp per cluster (persistent warps, consecutive clusters on one SM so that the
// gathered partner records stay in L1); the cluster's entry list is brought into shared memory by one
// bulk (TMA) copy, double-buffered against the previous cluster's arithmetic; lane = one partner j;
// the CL atoms of the cluster sit in registers two by two as the halves of fp32x2 operations,
// so a lane evaluates (i0, j), (i1, j) with one instruction stream.  Forces: i in registers across
// the whole list, one shuffle reduction per cluster; j summed over the cluster's atoms in the lane,
// then ONE 16-byte reduction to L2 per entry (red.global.add.v4.f32) -- Newton's third law at one
// reduction per CL pairs.  Periodic boxes use the fixed-point records of physics.cuh (fx_encode): the
// separation X_i - X_j wraps to the minimum image by itself, exact to L/2^32 whatever boxes the two atoms
// have drifted into; the cutoff decision stays the reference's: outside the band s_max -+ margin the two
// squared distances provably agree, the ~1e-5 of the pairs inside it are re-decided by cl_exact_pass with
// the reference's own arithmetic on the raw positions.  Without a box the reference's chain (sub, fma chain,
// s <= s_max) is evaluated directly in packed operations.  Neighbour sets stay bit-exact either way.
#pragma once
#include <type_traits>

#include "context.cuh"
#include "neighbor.cuh"
#include "pair.cuh"
#include "ptx.cuh"

namespace tmd {

#ifndef CL_C
#define CL_C 4
#endif
constexpr int CL = CL_C;       // atoms per i-cluster
constexpr int CL_H = CL / 2;   // packed pairs per cluster
static_assert(CL == 2 || CL == 4 || CL == 8, "cluster size");
constexpr int CL_MAXT = 128;   // atom types (the per-warp LJ table in dynamic shared memory is sized by the actual count)
constexpr int CL_XCAP = 192;   // excluded-partner entries of one cluster the list build can hold
#ifndef CL_WARPS_N
#define CL_WARPS_N 8
#endif
constexpr int CL_WARPS = CL_WARPS_N;
#ifndef CL_UNROLL
#define CL_UNROLL 1  // batches per loop iteration
#endif
#ifndef CL_MINBLOCKS
#define CL_MINBLOCKS 2  // up to 128 registers: no spills on sm_90a
#endif
constexpr int CL_UNROLL_N = CL_UNROLL;
constexpr int CLB_WARPS = 4;   // list build: warps per CTA
constexpr int CLB_MAXSEG = 160;
// dynamic shared memory of k_cpair / k_cpair_ew (entry buffers + LJ table): a context whose lists would need more takes
// the full rows (finalize); the interpreter build (tests/simt) holds exactly this much in a static buffer
constexpr size_t CL_SMEM_MAX = (size_t)180 * 1024;

__device__ __forceinline__ size_t cl_slot_base(const ClusterState& C, int r) { return (size_t)r * (C.slots + 1); }
__device__ __forceinline__ size_t cl_cluster_base(const ClusterState& C, int r) { return (size_t)r * C.nclusters_cap; }

// ---- rebuild, phase 1: cell of every atom, arrival slot in the cell's bucket ------------------------
constexpr int CL_BUCKET = 32;  // atoms a cell's bucket holds (cells of ~4 A hold about six in a liquid)
__global__ void k_cbin(DeviceState S, const float* __restrict__ pos) {
  const int r = blockIdx.y;
  const int parity = (int)(S.counters[0] & 1ull);
  if (!S.flags[r * F_COUNT + F_REBUILD0 + parity]) return;
  const int ncells = S.grid[r].ncells;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < S.natoms; i += gridDim.x * blockDim.x) {
    const size_t a = (size_t)r * S.natoms + i;
    const float x = pos[a * 3 + 0], y = pos[a * 3 + 1], z = pos[a * 3 + 2];
    int c = cell_of_point(S.grid[r], x, y, z);
    if (!isfinite(x + y + z)) {  // blown-up coordinates: report, and spread them so no cell degenerates
      S.flags[r * F_COUNT + F_FARPOS] = 1;
      c = i % ncells;
    }
    S.cell_of[a] = c;
    const int k = atomicAdd(S.cell_count + (size_t)r * (S.max_cells + 1) + c, 1);
    atomicAdd(S.cl.row_tot + (size_t)r * (S.cl.max_rows + 1) + c / S.grid[r].n[0], 1);  // atoms per cell row
    if (!S.own_all && i >= S.own_lo && i < S.own_lo + S.own_n) atomicAdd(S.cl.cell_owned + (size_t)r * (S.max_cells + 1) + c, 1);
    if (k < CL_BUCKET) S.cl.bucket[((size_t)r * S.max_cells + c) * CL_BUCKET + k] = i;
    else atomicOr(S.flags + r * F_COUNT + F_CLFAIL, 32);  // a cell this crowded: not a system for this path
    S.pos_ref[a] = make_float4(x, y, z, 0.0f);
  }
}

// ---- rebuild, phase 2: first slot of every cell row (one CTA per replica), then of every cell ------
// Rows (cells of equal y, z) are padded to a multiple of CL slots.  k_cbin counted the atoms per row.
__global__ void __launch_bounds__(1024) k_cscan(DeviceState S) {
  const int r = blockIdx.x;
  const int parity = (int)(S.counters[0] & 1ull);
  if (!S.flags[r * F_COUNT + F_REBUILD0 + parity]) return;
  __shared__ int warp_tot[32];
  const ClusterState& C = S.cl;
  const Grid& g = S.grid[r];
  const int n0 = g.n[0], nrows = g.n[1] * g.n[2];
  int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  int* rtot = C.row_tot + (size_t)r * (C.max_rows + 1);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int nt = blockDim.x;
  const int chunk = (nrows + nt - 1) / nt;
  const int rb = threadIdx.x * chunk, re = min(nrows, rb + chunk);
  int sum = 0;
  for (int row = rb; row < re; ++row) sum += (rtot[row] + CL - 1) / CL * CL;
  int incl = sum;
  for (int o = 1; o < 32; o <<= 1) {
    int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int t = lane < nw ? warp_tot[lane] : 0;
    int ti = t;
    for (int o = 1; o < 32; o <<= 1) {
      int v = __shfl_up_sync(0xffffffffu, ti, o);
      if (lane >= o) ti += v;
    }
    warp_tot[lane] = ti - t;
  }
  __syncthreads();
  int run = warp_tot[wid] + incl - sum;
  for (int row = rb; row < re; ++row) {
    const int t = (rtot[row] + CL - 1) / CL * CL;
    rtot[row] = run;  // the row's first slot
    run += t;
  }
  if (re == nrows && rb < nrows) {
    rtot[nrows] = run;
    start[nrows * n0] = run;
    C.nslots[r] = run;
    if (run > C.slots) atomicOr(S.flags + r * F_COUNT + F_CLFAIL, 16);  // (cannot happen: slots >= N + rows * (CL-1))
  }
}
// A warp per row: cell offsets inside the row (coalesced loads, shuffle scan), the padding records behind the
// row's atoms, the running count of owned atoms (decomposed runs).
__global__ void k_ccells(DeviceState S) {
  const int r = blockIdx.y;
  const int parity = (int)(S.counters[0] & 1ull);
  if (!S.flags[r * F_COUNT + F_REBUILD0 + parity]) return;
  const ClusterState& C = S.cl;
  const Grid& g = S.grid[r];
  const int n0 = g.n[0], nrows = g.n[1] * g.n[2];
  const int* cnt = S.cell_count + (size_t)r * (S.max_cells + 1);
  int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  const int* rtot = C.row_tot + (size_t)r * (C.max_rows + 1);
  const int lane = threadIdx.x & 31;
  const size_t sb = cl_slot_base(C, r);
  for (int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < nrows; row += gridDim.x * (blockDim.x >> 5)) {
    int base = rtot[row];
    const int pad_end = rtot[row + 1];
    int obase = 0;
    for (int c0 = 0; c0 < n0; c0 += 32) {
      const int c = c0 + lane;
      const int v = c < n0 ? cnt[row * n0 + c] : 0;
      int inc = v;
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
      }
      if (c < n0) start[row * n0 + c] = base + inc - v;
      base += __shfl_sync(0xffffffffu, inc, 31);
      if (!S.own_all) {
        const int ov = c < n0 ? C.cell_owned[(size_t)r * (S.max_cells + 1) + row * n0 + c] : 0;
        int oi = ov;
        for (int o = 1; o < 32; o <<= 1) {
          const int u = __shfl_up_sync(0xffffffffu, oi, o);
          if (lane >= o) oi += u;
        }
        if (c < n0) C.owned_pre[(size_t)r * (S.max_cells + 1) + row * n0 + c] = obase + oi;
        obase += __shfl_sync(0xffffffffu, oi, 31);
      }
    }
    for (int s = base + lane; s < pad_end; s += 32) {
      C.perm[sb + s] = -1;
      C.xq[sb + s] = make_float4(0.f, 0.f, 0.f, 0.f);
      C.f[sb + s] = make_float4(0.f, 0.f, 0.f, 0.f);
      C.xw[sb + s] = make_float4(1.0e30f, 1.0e30f, 1.0e30f, 0.f);
      if (C.xf) C.xf[sb + s] = make_int4(0, 0, 0, 0);
    }
  }
}

// ---- rebuild, phase 3: order every cell by x, emit the slot records -------------------------------------
// One thread per atom: its slot is the cell's first slot plus the number of atoms of the cell's bucket that
// precede it by (folded x, atom index) -- deterministic whatever order the atoms arrived in.
__global__ void k_csort(DeviceState S) {
  const int r = blockIdx.y;
  const int parity = (int)(S.counters[0] & 1ull);
  if (!S.flags[r * F_COUNT + F_REBUILD0 + parity]) return;
  const ClusterState& C = S.cl;
  const Grid& g = S.grid[r];
  const size_t base = (size_t)r * S.natoms, sb = cl_slot_base(C, r);
  const int* cnt = S.cell_count + (size_t)r * (S.max_cells + 1);
  const int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < S.natoms; i += gridDim.x * blockDim.x) {
    const int c = S.cell_of[base + i];
    const int n = min(cnt[c], CL_BUCKET);
    const float4 p = S.pos_ref[base + i];
    const float x = g.periodic ? p.x - g.L[0] * floorf(p.x * g.invL[0]) : p.x;
    const int* bk = C.bucket + ((size_t)r * S.max_cells + c) * CL_BUCKET;
    int rk = 0;
    bool listed = false;
    for (int k = 0; k < n; ++k) {
      const int j = bk[k];
      if (j == i) {
        listed = true;
        continue;
      }
      const float xr = S.pos_ref[base + j].x;
      const float xo = g.periodic ? xr - g.L[0] * floorf(xr * g.invL[0]) : xr;
      rk += (xo < x || (xo == x && j < i)) ? 1 : 0;
    }
    if (!listed) continue;  // (bucket overflow, already flagged: the build is discarded)
    const int s = start[c] + rk;
    C.inv[base + i] = s;
    C.perm[sb + s] = i;
    C.xq[sb + s] = make_float4(p.x, p.y, p.z, S.q[i]);
    C.f[sb + s] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (C.xf)
      C.xf[sb + s] = make_int4(fx_encode(p.x, g.fx_inv[0]), fx_encode(p.y, g.fx_inv[1]), fx_encode(p.z, g.fx_inv[2]),
                               __float_as_int(S.q[i]));
    float wx = p.x, wy = p.y, wz = p.z;
    if (g.periodic) {
      wx -= g.L[0] * floorf(wx * g.invL[0]);
      wy -= g.L[1] * floorf(wy * g.invL[1]);
      wz -= g.L[2] * floorf(wz * g.invL[2]);
    }
    C.xw[sb + s] = make_float4(wx, wy, wz, __int_as_float(S.type[i]));
  }
}

// ---- rebuild, phase 4: the cluster lists -------------------------------------------------------------
struct ClSeg {
  int begin, len;      // slots [begin, begin + len)
  float sx, sy, sz;    // image shift of these candidates into the cluster's frame
  int own;             // segment of the cluster's own row: partners chosen per cluster (cyclic half of the row)
};
struct ClBuildShared {
  ClSeg seg[CLB_WARPS][CLB_MAXSEG];
  int pre[CLB_WARPS][CLB_MAXSEG + 1];
  int xslot[CLB_WARPS][CL_XCAP];
  unsigned char xbits[CLB_WARPS][CL_XCAP];
};

__global__ void __launch_bounds__(CLB_WARPS * 32) k_cbuild(DeviceState S) {
  const int r = blockIdx.y;
  const int parity = (int)(S.counters[0] & 1ull);
  int* fl = S.flags + r * F_COUNT;
  if (!fl[F_REBUILD0 + parity]) return;
  __shared__ ClBuildShared sh;
  const ClusterState& C = S.cl;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  const Grid& g = S.grid[r];
  const size_t base = (size_t)r * S.natoms, sb = cl_slot_base(C, r), cb = cl_cluster_base(C, r);
  const int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  const int ns = C.nslots[r], ncl = ns / CL;
  const int n0 = g.n[0], n1 = g.n[1], n2 = g.n[2];
  const float rl = S.rlist, rl2 = S.rlist2;
  const int stride_e = C.mcap + C.ecap;
  if (blockIdx.x == 0 && threadIdx.x == 0) fl[F_NREBUILD] += 1;
  {  // the cell counters have served this build: clean for the next one
    int* cnt = S.cell_count + (size_t)r * (S.max_cells + 1);
    for (int cc = blockIdx.x * blockDim.x + threadIdx.x; cc < g.ncells; cc += gridDim.x * blockDim.x) {
      cnt[cc] = 0;
      if (!S.own_all) C.cell_owned[(size_t)r * (S.max_cells + 1) + cc] = 0;
    }
    for (int rr = blockIdx.x * blockDim.x + threadIdx.x; rr <= C.max_rows; rr += gridDim.x * blockDim.x)
      C.row_tot[(size_t)r * (C.max_rows + 1) + rr] = 0;
  }

  for (int c = blockIdx.x * CLB_WARPS + w; c < C.nclusters_cap; c += gridDim.x * CLB_WARPS) {
    if (c >= ncl) {
      if (lane == 0) C.meta[cb + c] = make_int2(0, 0);
      continue;
    }
    const int s0 = c * CL;
    // ---- the cluster: bounding box of its real atoms (folded coordinates), frame of its first atom
    float4 pw = make_float4(1.0e30f, 1.0e30f, 1.0e30f, 0.f);
    if (lane < CL) pw = C.xw[sb + s0 + lane];
    const bool real = pw.x < 1.0e29f;
    const unsigned realmask = __ballot_sync(0xffffffffu, real) & ((1u << CL) - 1u);
    float lo[3] = {real ? pw.x : INFINITY, real ? pw.y : INFINITY, real ? pw.z : INFINITY};
    float hi[3] = {real ? pw.x : -INFINITY, real ? pw.y : -INFINITY, real ? pw.z : -INFINITY};
#pragma unroll
    for (int d = 0; d < 3; ++d)
      for (int o = CL / 2; o; o >>= 1) {
        lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
        hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
      }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = __shfl_sync(0xffffffffu, lo[d], 0);
      hi[d] = __shfl_sync(0xffffffffu, hi[d], 0);
    }
    float ax[CL], ay[CL], az[CL];
#pragma unroll
    for (int k = 0; k < CL; ++k) {
      ax[k] = __shfl_sync(0xffffffffu, pw.x, k);
      if (!((realmask >> k) & 1u)) ax[k] = 1.0e15f;
      ay[k] = __shfl_sync(0xffffffffu, pw.y, k);
      az[k] = __shfl_sync(0xffffffffu, pw.z, k);
    }
    const float rl2x = rl2 * 1.00001f;  // (rounding of the float test must never drop a pair the skin argument counts on)
    if (realmask == 0) {  // (cannot happen: padding only ever completes a cluster)
      if (lane == 0) C.meta[cb + c] = make_int2(0, 0);
      continue;
    }
    const int first = __ffs(realmask) - 1;
    // decomposed run: does the cluster hold an atom this rank owns?  If not, only owned partners matter.
    bool owned_lane = true;
    if (!S.own_all) {
      const int a = (lane < CL && real) ? C.perm[sb + s0 + lane] : -1;
      owned_lane = a >= S.own_lo && a < S.own_lo + S.own_n;
    }
    const bool o_c = S.own_all || __any_sync(0xffffffffu, owned_lane && lane < CL && real);
    const int* owned_pre = S.cl.owned_pre + (size_t)r * (S.max_cells + 1);
    // a list holds pairs up to rl + (cluster extent) apart along an axis: that must stay below half the box
    if (lane == 0 && g.periodic &&
        (hi[0] - lo[0] > C.max_extent || hi[1] - lo[1] > C.max_extent || hi[2] - lo[2] > C.max_extent))
      atomicOr(fl + F_CLFAIL, 1);
    // ---- excluded partners of the cluster's atoms: (slot, bit of the cluster atom)
    int nx = 0;
    if (S.excl_ptr) {
      for (int k = 0; k < CL; ++k) {
        if (!((realmask >> k) & 1u)) continue;
        const int a = C.perm[sb + s0 + k];
        const int e1 = S.excl_ptr[a + 1];
        for (int e0 = S.excl_ptr[a]; e0 < e1; e0 += 32) {
          const int e = e0 + lane;
          int sj = -1;
          if (e < e1) sj = C.inv[base + S.excl_idx[e]];
          const bool keep = sj >= 0;  // (any slot: with the cyclic half-shell rule a listed partner may sit before the cluster)
          const unsigned bal = __ballot_sync(0xffffffffu, keep);
          if (keep) {
            const int p = nx + __popc(bal & lt);
            if (p < CL_XCAP) {
              sh.xslot[w][p] = sj;
              sh.xbits[w][p] = (unsigned char)(1u << k);
            }
          }
          nx += __popc(bal);
        }
      }
      if (nx > CL_XCAP) {
        if (lane == 0) atomicOr(fl + F_CLFAIL, 4);
        nx = CL_XCAP;
      }
    }
    __syncwarp();
    // slot range of the set: most candidates lie outside it and skip the search
    int xlo = 0x7fffffff, xhi = -1;
    for (int k = lane; k < nx; k += 32) {
      xlo = min(xlo, sh.xslot[w][k]);
      xhi = max(xhi, sh.xslot[w][k]);
    }
    xlo = __reduce_min_sync(0xffffffffu, xlo);
    xhi = __reduce_max_sync(0xffffffffu, xhi);
    auto excluded_bits = [&](int sj) {
      unsigned m = 0;
      for (int k = 0; k < nx; ++k)
        if (sh.xslot[w][k] == sj) m |= sh.xbits[w][k];
      return m;
    };
    unsigned* entA = C.entries + (cb + c) * (size_t)stride_e;
    unsigned* entB = entA + C.mcap;
    unsigned char* mskA = C.masks + (cb + c) * (size_t)C.mcap;
    int nA = 0, nB = 0;
    // ---- the cluster's own atoms: atom k as partner of the atoms before it
    {
      unsigned m = 0;
      unsigned en = 0;
      if (lane >= 1 && lane < CL && real && o_c) {
        m = (realmask & ((1u << lane) - 1u)) & ~excluded_bits(s0 + lane);
        en = (unsigned)(s0 + lane) | ((unsigned)__float_as_int(pw.w) << 24);
      }
      const unsigned bal = __ballot_sync(0xffffffffu, m != 0);
      if (m) {
        const int p = __popc(bal & lt);
        entA[p] = en;
        mskA[p] = (unsigned char)m;
      }
      nA = __popc(bal);
    }
    // ---- candidate rows -> segments of consecutive slots
    const float wy = n1 > 1 ? 1.0f / g.inv_w[1] : 0.f, wz = n2 > 1 ? 1.0f / g.inv_w[2] : 0.f;
    // the cluster's row, from the binning itself (the slot order is the order of the binned cells)
    const int row_c = S.cell_of[base + C.perm[sb + s0 + first]] / n0;
    const int cy = row_c % n1, cz = row_c / n1;
    const int ry = n1 > 1 ? g.reach[1] : 0, rz = n2 > 1 ? g.reach[2] : 0;
    const int row_s = start[row_c * n0], row_ncl = (start[(row_c + 1) * n0] - row_s) / CL;  // the own row's clusters
    const int ci_row = (s0 - row_s) / CL;
    // Which of two clusters lists a pair?  The one that sees the other's row at an offset in the "upper" half-space
    // (dz > 0, or dz == 0 and dy > 0; inside the own row: the next half of the cyclic cluster order, see the sweep).
    // Offsets are unique (the box holds at least 2 * reach + 1 rows), so the rule is antisymmetric, and every cluster
    // gets the same half of its surroundings wherever it sits -- a plain "later slots" rule gives the first planes of
    // a periodic box twice the work of the middle ones and the last planes none.
    const int nry = 2 * ry + 1, nrows_c = rz * nry + ry + 1;
    int nseg = 0;
    for (int q0 = 0; q0 < nrows_c; q0 += 32) {
      const int q = q0 + lane;
      // up to three segments per row (x images -1, 0, +1)
      int sbeg[3] = {0, 0, 0}, slen[3] = {0, 0, 0};
      float shx[3] = {0.f, 0.f, 0.f}, shy = 0.f, shz = 0.f;
      bool own_row = false;
      if (q < nrows_c) {
        const int dz = q <= ry ? 0 : 1 + (q - ry - 1) / nry;
        const int dy = q <= ry ? q : (q - ry - 1) % nry - ry;
        int yy = cy + dy, zz = cz + dz;
        bool ok = true;
        if (g.periodic) {
          if (yy < 0) yy += n1, shy = -g.L[1];
          else if (yy >= n1) yy -= n1, shy = g.L[1];
          if (zz < 0) zz += n2, shz = -g.L[2];
          else if (zz >= n2) zz -= n2, shz = g.L[2];
          ok = yy >= 0 && yy < n1 && zz >= 0 && zz < n2;
          // (a row reached twice -- box narrower than the sweep -- cannot happen: the host requires n >= 2*reach+1)
        } else {
          ok = yy >= 0 && yy < n1 && zz >= 0 && zz < n2;
        }
        const int rr = zz * n1 + yy;
        own_row = ok && q == 0;
        if (ok) {
          // distance in y, z between the box and the row's slab (with a margin for the binning's rounding)
          const float ylo = g.origin[1] + yy * wy + shy - 1.0e-3f, yhi = ylo + wy + 2.0e-3f;
          const float zlo = g.origin[2] + zz * wz + shz - 1.0e-3f, zhi = zlo + wz + 2.0e-3f;
          const float ey = n1 > 1 ? fmaxf(fmaxf(lo[1] - yhi, ylo - hi[1]), 0.f) : 0.f;
          const float ez = n2 > 1 ? fmaxf(fmaxf(lo[2] - zhi, zlo - hi[2]), 0.f) : 0.f;
          const float rem = rl2 - ey * ey - ez * ez;
          if (rem > 0.f) {
            const float rx = sqrtf(fmaxf(rem, 0.f)) + 1.0e-3f;
            const float fx0 = (lo[0] - rx - g.origin[0]) * g.inv_w[0], fx1 = (hi[0] + rx - g.origin[0]) * g.inv_w[0];
            int cx0 = (int)floorf(fx0), cx1 = (int)floorf(fx1);
            if (n0 == 1) cx0 = cx1 = 0;
            if (!g.periodic) {
              cx0 = max(cx0, 0);
              cx1 = min(cx1, n0 - 1);
              if (cx0 <= cx1 && (o_c || owned_pre[rr * n0 + cx1] - (cx0 ? owned_pre[rr * n0 + cx0 - 1] : 0) > 0)) {
                sbeg[1] = start[rr * n0 + cx0];
                slen[1] = start[rr * n0 + cx1 + 1] - sbeg[1];
              }
            } else {
              if (cx1 - cx0 + 1 > n0) cx0 = 0, cx1 = n0 - 1;  // (excluded by the host's size condition)
#pragma unroll
              for (int k = -1; k <= 1; ++k) {
                const int a0 = max(cx0, k * n0) - k * n0, a1 = min(cx1, (k + 1) * n0 - 1) - k * n0;
                if (a0 <= a1 && (o_c || owned_pre[rr * n0 + a1] - (a0 ? owned_pre[rr * n0 + a0 - 1] : 0) > 0)) {
                  sbeg[k + 1] = start[rr * n0 + a0];
                  slen[k + 1] = start[rr * n0 + a1 + 1] - sbeg[k + 1];
                  shx[k + 1] = k * g.L[0];
                }
              }
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const bool has = slen[k] > 0;
        const unsigned bal = __ballot_sync(0xffffffffu, has);
        if (has) {
          const int p = nseg + __popc(bal & lt);
          if (p < CLB_MAXSEG) sh.seg[w][p] = ClSeg{sbeg[k], slen[k], shx[k], shy, shz, own_row ? 1 : 0};
        }
        nseg += __popc(bal);
      }
    }
    if (nseg > CLB_MAXSEG) {
      if (lane == 0) atomicOr(fl + F_CLFAIL, 8);
      nseg = CLB_MAXSEG;
    }
    __syncwarp();
    // exclusive prefix of the segment lengths (one warp: serial over chunks of 32)
    int total = 0;
    for (int q0 = 0; q0 < nseg; q0 += 32) {
      const int q = q0 + lane;
      const int len = q < nseg ? sh.seg[w][q].len : 0;
      int incl = len;
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      if (q < nseg) sh.pre[w][q] = total + incl - len;
      total += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) sh.pre[w][nseg] = total;
    __syncwarp();
    // ---- sweep the candidates
    int sg = 0;
    for (int idx0 = 0; idx0 < total; idx0 += 32) {
      const int idx = idx0 + lane;
      bool take = false;
      int sj = 0;
      unsigned tj = 0;
      if (idx < total) {
        while (idx >= sh.pre[w][sg + 1]) ++sg;
        const ClSeg sgm = sh.seg[w][sg];
        sj = sgm.begin + (idx - sh.pre[w][sg]);
        const float4 p = C.xw[sb + sj];
        const float x = p.x + sgm.sx, y = p.y + sgm.sy, z = p.z + sgm.sz;
        // within the list radius of one of the cluster's atoms (a bounding-box test keeps ~15 % more partners: the
        // corners of the box hold no atom); padding records are 1e30 away, a missing cluster atom is at 1e15
        float d2 = INFINITY;
#pragma unroll
        for (int k = 0; k < CL; ++k) {
          const float ux = x - ax[k], uy = y - ay[k], uz = z - az[k];
          d2 = fminf(d2, fmaf(ux, ux, fmaf(uy, uy, uz * uz)));
        }
        take = d2 < rl2x;
        if (sgm.own) {  // own row: the clusters in the next half of the row's cyclic order
          const int cj = (sj - row_s) / CL;
          int dd = cj - ci_row;
          if (dd < 0) dd += row_ncl;
          take = take && dd != 0 && (2 * dd < row_ncl || (2 * dd == row_ncl && cj > ci_row));
        }
        tj = (unsigned)__float_as_int(p.w);
        if (take && !o_c) {  // a cluster without owned atoms keeps the partners this rank owns
          const int aj = C.perm[sb + sj];
          take = aj >= S.own_lo && aj < S.own_lo + S.own_n;
        }
      }
      unsigned xb = 0;
      if (take && sj >= xlo && sj <= xhi) xb = excluded_bits(sj);
      const bool plain = take && xb == 0;
      const unsigned m = realmask & ~xb;
      const bool special = take && xb != 0 && m != 0;
      const unsigned balB = __ballot_sync(0xffffffffu, plain), balA = __ballot_sync(0xffffffffu, special);
      const unsigned en = (unsigned)sj | (tj << 24);
      if (plain) {
        const int p = nB + __popc(balB & lt);
        if (p < C.ecap) entB[p] = en;
      }
      if (special) {
        const int p = nA + __popc(balA & lt);
        if (p < C.mcap) {
          entA[p] = en;
          mskA[p] = (unsigned char)m;
        }
      }
      nB += __popc(balB);
      nA += __popc(balA);
    }
    (void)rl;
    // ---- close the regions: pad to whole batches with the dummy record
    if (lane == 0) {
      atomicMax(fl + F_MAXNBR, 2 * (nA + nB));
      atomicMax(fl + F_CLMAXA, nA);
      atomicMax(fl + F_CLMAXB, nB);
      if (nA > C.mcap || nB > C.ecap) fl[F_OVERFLOW] = 1;
    }
    nA = min(nA, C.mcap);
    nB = min(nB, C.ecap);
    const int pA = (nA + 31) & ~31, pB = (nB + 31) & ~31;
    for (int p = nA + lane; p < pA; p += 32) {
      entA[p] = (unsigned)C.slots;
      mskA[p] = 0;
    }
    for (int p = nB + lane; p < pB; p += 32) entB[p] = (unsigned)C.slots;
    if (lane == 0) C.meta[cb + c] = make_int2(pA | (int)(realmask << 24), pB);
  }
}

// ---- the pair kernel ----------------------------------------------------------------------------------
// LJ table of a cluster: per partner type and packed pair (A_i0, A_i1, B_i0, B_i1), (12 A_i0, 12 A_i1, 6 B_i0, 6 B_i1)
struct ClTab {
  float4 ab, dab;
};

// MINUS the force coefficient (dE/dr)/r of two pairs: pair_coef2 of physics.cuh with the LJ factors 12 A, 6 B
// taken from the table (two operations fewer).
// EW: real-space Ewald electrostatics (physics.cuh, ewald_ndedr2) in place of the reaction field.
template <bool ENERGY, bool EW = false>
__device__ __forceinline__ F2 cl_coef2(const SwitchConsts& c, F2 s, F2 nqq, const ClTab& t, F2& e_lj, F2& ne_el) {
  const F2 y = f2(rsqrt_seed(s.x), rsqrt_seed(s.y));
  const F2 h = f2_mul(s, y);
  const F2 u = f2_fma(f2_mul(h, f2(-0.5f)), y, f2(0.5f));
  const F2 rinv = f2_fma(y, u, y);
  const F2 r = f2_mul(s, rinv);
  // -1/r^2 to ~0.5 ulp from its own hardware seed: the r^-12 wall multiplies its error by six (a close O-O pair
  // would otherwise cost ~3e-5 kcal/mol/A of the 1e-4 budget)
  const F2 nz = f2(neg_rcp_seed(s.x), neg_rcp_seed(s.y));
  const F2 nr2 = f2_fma(nz, f2_fma(s, nz, f2(1.0f)), nz);
  const F2 nr6 = f2_mul(f2_mul(nr2, nr2), nr2);       // -1/r^6
  const F2 A = f2(t.ab.x, t.ab.y), B = f2(t.ab.z, t.ab.w), A12 = f2(t.dab.x, t.dab.y), B6 = f2(t.dab.z, t.dab.w);
  const F2 e = f2_mul(nr6, f2_fma(A, nr6, B));        // A/r^12 - B/r^6
  const F2 nf = f2_mul(f2_mul(nr6, f2_fma(A12, nr6, B6)), rinv);  // -(dE/dr) = (12 A/r^12 - 6 B/r^6)/r
  F2 tt = f2_fma(r, f2(c.inv_sw_width), f2(c.neg_switch_dist * c.inv_sw_width));
  tt = f2(fmaxf(tt.x, 0.0f), fmaxf(tt.y, 0.0f));
  const F2 t2 = f2_mul(tt, tt);
  const F2 sw = f2_fma(f2_mul(t2, tt), f2_fma(tt, f2_fma(tt, f2(-6.0f), f2(15.0f)), f2(-10.0f)), f2(1.0f));
  const F2 ndsw = f2_mul(t2, f2_fma(tt, f2_fma(tt, f2(c.d1), f2(c.d2)), f2(c.d3)));
  const F2 nfsw = f2_fma(sw, nf, f2_mul(f2_mul(e, ndsw), rinv));  // the reference's s dE/dr + E s'/r (forces.py:410-412)
  if constexpr (EW) {
    F2 ec;
    const F2 ndedr = f2_add(ewald_ndedr2(c, nqq, r, rinv, nr2, ec), nfsw);
    if (ENERGY) {
      e_lj = f2_mul(e, sw);
      ne_el = f2_mul(f2_mul(nqq, ec), rinv);
    }
    return f2_mul(ndedr, rinv);
  }
  const F2 ndedr = f2_fma(nqq, f2_fma(f2(c.two_krf), r, nr2), nfsw);
  if (ENERGY) {
    e_lj = f2_mul(e, sw);
    ne_el = f2_mul(nqq, f2_add(f2_fma(f2(c.krf), s, rinv), f2(c.neg_crf)));
  }
  return f2_mul(ndedr, rinv);
}

struct ClPairShared {
  unsigned long long bar[CL_WARPS][2];
  double red[CL_WARPS];
};

// Pairs of cluster c inside the decision band of a periodic box: the reference's own decision on the raw
// positions, one pair at a time, forces straight to the accumulators.  Rare (about one cluster in a hundred).
// (Arguments by value: a reference to the kernel's parameter block would force a local copy of it.)
struct ClExactArgs {
  const int4* xf;        // slot records of this replica
  const float4* xq;
  const float4* xw;
  float4* f;
  const unsigned* ent;   // this cluster's entries / masks
  const unsigned char* msk;
  const Grid* g;
  const float2* AB;
  int mcap, slots, c, ntypes;
  const int* perm;       // decomposed runs: energy share by ownership
  int own_lo, own_n, own_all;
  unsigned terms;
  float s_lo, s_hi, s_max;
};
template <bool ENERGY, bool EW>
__device__ __forceinline__ float2 cl_exact_body(const ClExactArgs& a, int2 mt, const SwitchConsts& sc) {
  const int lane = threadIdx.x & 31;
  const Grid* g = a.g;
  const unsigned imask = (unsigned)mt.x >> 24;
  const int nA = mt.x & 0xffffff, nB = mt.y;
  const float ux = g->fx_unit[0], uy = g->fx_unit[1], uz = g->fx_unit[2];
  float e_lj = 0.f, e_el = 0.f;
  for (int region = 0; region < 2; ++region) {
    const int n = region == 0 ? nA : nB;
    const unsigned* e = region == 0 ? a.ent : a.ent + a.mcap;
    for (int k = lane; k < n; k += 32) {
      const unsigned en = e[k];
      const int sj = (int)(en & 0xffffffu);
      if (sj >= a.slots) continue;
      const unsigned m = (region == 0 ? (unsigned)a.msk[k] : 0xffu) & imask;
      const int4 pj = a.xf[sj];
      for (int i = 0; i < CL; ++i) {
        if (!((m >> i) & 1u)) continue;
        const int si = a.c * CL + i;
        const int4 pi = a.xf[si];
        const float wx = fx_delta(pi.x, pj.x, ux), wy = fx_delta(pi.y, pj.y, uy), wz = fx_delta(pi.z, pj.z, uz);
        const float s = fmaf(wz, wz, fmaf(wy, wy, wx * wx));
        if (!(s < a.s_lo) && s <= a.s_hi) {
          const float4 ri = a.xq[si], rj = a.xq[sj];
          if (ref_inside(ri.x, ri.y, ri.z, rj.x, rj.y, rj.z, g->L[0], g->L[1], g->L[2], g->invL[0], g->invL[1], g->invL[2], a.s_max)) {
            float2 ab = make_float2(0.f, 0.f);
            if (a.terms & T_LJ) ab = a.AB[__float_as_int(a.xw[si].w) * a.ntypes + (int)(en >> 24)];
            ClTab tb;
            tb.ab = make_float4(ab.x, ab.x, ab.y, ab.y);
            tb.dab = make_float4(12.0f * ab.x, 12.0f * ab.x, 6.0f * ab.y, 6.0f * ab.y);
            const float nqq = (a.terms & T_ELEC) ? -(__int_as_float(pi.w) * __int_as_float(pj.w)) : 0.f;
            F2 elj, neel;
            const F2 nc = cl_coef2<ENERGY, EW>(sc, f2(s), f2(nqq), tb, elj, neel);
            red_add_f32x4(a.f + si, wx * nc.x, wy * nc.x, wz * nc.x);
            red_add_f32x4(a.f + sj, -wx * nc.x, -wy * nc.x, -wz * nc.x);
            if (ENERGY) {
              float wgt = 1.0f;
              if (!a.own_all) {
                const int ai = a.perm[si], aj = a.perm[sj];
                wgt = 0.5f * ((ai >= a.own_lo && ai < a.own_lo + a.own_n) ? 1.f : 0.f) + 0.5f * ((aj >= a.own_lo && aj < a.own_lo + a.own_n) ? 1.f : 0.f);
              }
              e_lj += wgt * elj.x;
              e_el -= wgt * neel.x;
            }
          }
        }
      }
    }
  }
  return make_float2(e_lj, e_el);
}
template <bool ENERGY>
__device__ __noinline__ float2 cl_exact_pass(ClExactArgs a, int2 mt, SwitchConsts sc) {
  return cl_exact_body<ENERGY, false>(a, mt, sc);
}
template <bool ENERGY>
__device__ __noinline__ float2 cl_exact_pass_ew(ClExactArgs a, int2 mt, SwitchConsts sc) {
  return cl_exact_body<ENERGY, true>(a, mt, sc);
}

// dynamic shared memory: per warp two entry buffers of (mcap + ecap) words, then per warp the LJ table (ntypes x CL_H)
template <bool ENERGY, bool PERIODIC, bool EW>
__device__ __forceinline__ void cpair_body(const DeviceState& S, const SwitchConsts& sc, double* __restrict__ energies) {
#if defined(TMD_SIMT_HOST)
  __shared__ __attribute__((aligned(128))) unsigned char cl_dyn[CL_SMEM_MAX];  // (interpreter build: no dynamic window)
#else
  extern __shared__ __align__(128) unsigned char cl_dyn[];
#endif
  __shared__ ClPairShared sh;
  const ClusterState& C = S.cl;
  const int r = blockIdx.y;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const size_t sb = cl_slot_base(C, r), cb = cl_cluster_base(C, r);
  const int stride_e = C.mcap + C.ecap;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    S.counters[0] += 1;              // next call: other flag
    S.counters[2] = S.counters[1];   // this step's Philox position, for k_cstep_boundary (which advances [1] while it reads)
  }
  const size_t buf_bytes_h = (size_t)stride_e * 4 + C.mcap;  // entry words + mask bytes of one buffer
  unsigned char* buf0 = cl_dyn + (size_t)w * 2 * buf_bytes_h;
  ClTab* tab = reinterpret_cast<ClTab*>(cl_dyn + (size_t)CL_WARPS * 2 * buf_bytes_h) + (size_t)w * S.ntypes * CL_H;
  const smem_addr buf_s = smem_address(buf0);
  const smem_addr bar_s = smem_address(&sh.bar[w][0]);
  if (lane == 0) {
    mbar_init(bar_s, 1);
    mbar_init(bar_s + 8, 1);
    fence_mbar_init();
  }
  __syncwarp();
  const float4* __restrict__ xq = C.xq + sb;
  const int4* __restrict__ xf = C.xf + sb;
  float4* __restrict__ fout = C.f + sb;
  const int ncl = C.nslots[r] / CL;
  // consecutive clusters per CTA: chunk of the cluster range, warps interleaved inside it
  const int per_cta = (ncl + gridDim.x - 1) / gridDim.x;
  const int c_begin = blockIdx.x * per_cta, c_end = min(ncl, c_begin + per_cta);
  F2 ELJ = f2(0.f), NEEL = f2(0.f);   // energies of the current cluster (fp32), folded into fp64 per cluster
  double acc_lj = 0.0, acc_el = 0.0;
  float ex_lj = 0.f, ex_el = 0.f;  // energies of the pairs decided by cl_exact_pass
  const bool lj_on = (S.pp.terms & T_LJ) != 0, el_on = (S.pp.terms & T_ELEC) != 0;
  // decision thresholds: without a box the reference's s <= s_max itself; in a periodic box the band around it
  float s_in = S.pp.s_max, s_hi = S.pp.s_max;
  F2 ux = f2(0.f), uy = f2(0.f), uz = f2(0.f);
  if (PERIODIC) {
    const Grid* g = S.grid + r;
    ux = f2(g->fx_unit[0]);
    uy = f2(g->fx_unit[1]);
    uz = f2(g->fx_unit[2]);
    // (a non-finite coordinate somewhere makes the margin infinite: every pair goes to the exact pass)
    const float margin = fmaf(g->fx_c1, __int_as_float(S.flags[r * F_COUNT + F_PMAX]), g->fx_c0);
    s_in = S.pp.s_max - margin;
    s_hi = S.pp.s_max + margin;
  }
  // s >= +0 always, so its bit pattern orders like its value: u = bits(s) - bits(s_in) wraps to >= 2^31 exactly for the
  // pairs inside (s < s_in), and the pairs in the band are those with u <= bits(s_hi) - bits(s_in)
  const unsigned b_in = __float_as_uint(fmaxf(s_in, 0.f)), b_band = __float_as_uint(fmaxf(s_hi, 0.f)) - b_in;

  // one buffer: (mcap + ecap) entry words, then mcap mask bytes
  const unsigned buf_bytes = (unsigned)stride_e * 4u + (unsigned)C.mcap;
  auto issue = [&](int c, int which, int2 mt) {  // lane 0: bulk copies of the cluster's regions into buffer `which`
    const int nA = mt.x & 0xffffff;
    const unsigned bytes = (unsigned)(nA + mt.y) * 4u + (unsigned)nA;
    const smem_addr dst = buf_s + (unsigned)which * buf_bytes, bar = bar_s + 8u * which;
    const unsigned* src = C.entries + (cb + c) * (size_t)stride_e;
    mbar_expect_tx(bar, bytes);
    if (nA) {
      bulk_g2s(dst, src, (unsigned)nA * 4u, bar);
      bulk_g2s(dst + (unsigned)stride_e * 4u, C.masks + (cb + c) * (size_t)C.mcap, (unsigned)nA, bar);
    }
    if (mt.y) bulk_g2s(dst + (unsigned)nA * 4u, src + C.mcap, (unsigned)mt.y * 4u, bar);
  };
  auto entries_of = [](int2 mt) { return (mt.x & 0xffffff) + mt.y; };

  int c = c_begin + w;
  int2 mt = make_int2(0, 0), mt_next = make_int2(0, 0);
  unsigned phase = 0;  // bit b: parity to wait for on buffer b
  int which = 0;
  if (c < c_end) {
    mt = C.meta[cb + c];
    if (lane == 0 && entries_of(mt)) issue(c, 0, mt);
    if (c + CL_WARPS < c_end) mt_next = C.meta[cb + c + CL_WARPS];
  }
  for (; c < c_end; c += CL_WARPS) {
    const int cn = c + CL_WARPS;
    // next cluster's list on its way while this one is evaluated
    const int2 mt_cur = mt;
    if (cn < c_end && lane == 0 && entries_of(mt_next)) issue(cn, which ^ 1, mt_next);
    mt = mt_next;
    if (cn + CL_WARPS < c_end) mt_next = C.meta[cb + cn + CL_WARPS];

    const int s0 = c * CL;
    const unsigned imask = (unsigned)mt_cur.x >> 24;
    if (entries_of(mt_cur) == 0) {  // (decomposed runs: most clusters far from the owned atoms have nothing to do)
      which ^= 1;
      continue;
    }
    // decomposed run, energies: a pair counts by the share of its atoms this rank owns (the other rank adds the rest)
    float own_i[CL];
#pragma unroll
    for (int k = 0; k < CL; ++k) own_i[k] = 1.0f;
    if (ENERGY && !S.own_all) {
#pragma unroll
      for (int k = 0; k < CL; ++k) {
        const int a = C.perm[sb + s0 + k];
        own_i[k] = (a >= S.own_lo && a < S.own_lo + S.own_n) ? 0.5f : 0.0f;
      }
    }
    // ---- the cluster's atoms, two by two: float records without a box, fixed-point records with one
    F2 XI[CL_H], YI[CL_H], ZI[CL_H], NQI[CL_H];
    int IX[CL], IY[CL], IZ[CL];
    int ti[CL];
#pragma unroll
    for (int p = 0; p < CL_H; ++p) {
      if (PERIODIC) {
        const int4 a = xf[s0 + 2 * p], b = xf[s0 + 2 * p + 1];
        IX[2 * p] = a.x; IY[2 * p] = a.y; IZ[2 * p] = a.z;
        IX[2 * p + 1] = b.x; IY[2 * p + 1] = b.y; IZ[2 * p + 1] = b.z;
        NQI[p] = el_on ? f2(-__int_as_float(a.w), -__int_as_float(b.w)) : f2(0.f);
      } else {
        const float4 a = xq[s0 + 2 * p], b = xq[s0 + 2 * p + 1];
        XI[p] = f2(a.x, b.x);
        YI[p] = f2(a.y, b.y);
        ZI[p] = f2(a.z, b.z);
        NQI[p] = el_on ? f2(-a.w, -b.w) : f2(0.f);
      }
      ti[2 * p] = __float_as_int(C.xw[sb + s0 + 2 * p].w);
      ti[2 * p + 1] = __float_as_int(C.xw[sb + s0 + 2 * p + 1].w);
    }
    __syncwarp();  // (the previous cluster's table reads are done)
    for (int e = lane; e < S.ntypes * CL_H; e += 32) {
      const int t = e / CL_H, p = e % CL_H;
      float2 v0 = make_float2(0.f, 0.f), v1 = v0;
      int t0 = 0, t1 = 0;  // (a register array cannot be indexed by p: select)
#pragma unroll
      for (int pp = 0; pp < CL_H; ++pp)
        if (pp == p) {
          t0 = ti[2 * pp];
          t1 = ti[2 * pp + 1];
        }
      if (lj_on) {
        v0 = S.AB[t0 * S.ntypes + t];
        v1 = S.AB[t1 * S.ntypes + t];
      }
      ClTab tb;
      tb.ab = make_float4(v0.x, v1.x, v0.y, v1.y);
      tb.dab = make_float4(12.0f * v0.x, 12.0f * v1.x, 6.0f * v0.y, 6.0f * v1.y);
      tab[t * CL_H + p] = tb;
    }
    F2 FX[CL_H], FY[CL_H], FZ[CL_H];
#pragma unroll
    for (int p = 0; p < CL_H; ++p) FX[p] = FY[p] = FZ[p] = f2(0.f);

    const int nbA = (mt_cur.x & 0xffffff) >> 5, nb = entries_of(mt_cur) >> 5;
    const smem_addr ebuf = buf_s + (unsigned)which * buf_bytes;
    const smem_addr mbuf = ebuf + (unsigned)stride_e * 4u;
    const unsigned char* __restrict__ mrow = C.masks + (cb + c) * (size_t)C.mcap;
    if (nb) mbar_wait(bar_s + 8u * which, (phase >> which) & 1u);
    __syncwarp();
    unsigned u_min = 0xffffffffu;  // smallest u of a pair not taken (see b_band)
    // base addresses the loop uses, kept in registers (otherwise re-derived from the parameter block per entry)
    unsigned long long rec_base = PERIODIC ? reinterpret_cast<unsigned long long>(xf) : reinterpret_cast<unsigned long long>(xq);
    unsigned long long f_base = reinterpret_cast<unsigned long long>(fout);
    TMD_PIN_L(rec_base);
    TMD_PIN_L(f_base);
    const unsigned nslots_cap = (unsigned)C.slots;

    // one partner (record rj: float x, y, z, q or fixed-point X, Y, Z, q bits) against the cluster
    auto body = [&](unsigned entry, unsigned mask, const int4 rj) {
      const unsigned tj = entry >> 24;
      const unsigned jslot = entry & 0xffffffu;
      const float qj = __int_as_float(rj.w);
      float own_j = 0.f;
      if (ENERGY && !S.own_all) {
        const int aj = jslot < nslots_cap ? C.perm[sb + jslot] : -1;
        own_j = (aj >= S.own_lo && aj < S.own_lo + S.own_n) ? 0.5f : 0.0f;
      }
      F2 GX = f2(0.f), GY = f2(0.f), GZ = f2(0.f);
#pragma unroll
      for (int p = 0; p < CL_H; ++p) {
        F2 dx, dy, dz;
        if (PERIODIC) {
          // two's-complement difference = minimum image, exact to L / 2^32
          dx = f2_mul(f2((float)(int)((unsigned)IX[2 * p] - (unsigned)rj.x), (float)(int)((unsigned)IX[2 * p + 1] - (unsigned)rj.x)), ux);
          dy = f2_mul(f2((float)(int)((unsigned)IY[2 * p] - (unsigned)rj.y), (float)(int)((unsigned)IY[2 * p + 1] - (unsigned)rj.y)), uy);
          dz = f2_mul(f2((float)(int)((unsigned)IZ[2 * p] - (unsigned)rj.z), (float)(int)((unsigned)IZ[2 * p + 1] - (unsigned)rj.z)), uz);
        } else {
          // the reference's rounded differences (forces.py:368-372)
          dx = f2_add(XI[p], f2(-__int_as_float(rj.x)));
          dy = f2_add(YI[p], f2(-__int_as_float(rj.y)));
          dz = f2_add(ZI[p], f2(-__int_as_float(rj.z)));
        }
        const F2 s = f2_fma(dz, dz, f2_fma(dy, dy, f2_mul(dx, dx)));
        const bool m0 = (mask >> (2 * p)) & 1u, m1 = (mask >> (2 * p + 1)) & 1u;
        bool in0, in1;
        if (PERIODIC) {
          const unsigned u0 = __float_as_uint(s.x) - b_in, u1 = __float_as_uint(s.y) - b_in;
          in0 = m0 && (int)u0 < 0;
          in1 = m1 && (int)u1 < 0;
          // (pairs a mask switches off are not filtered here: one of them inside the band only costs a pass that
          //  re-checks the masks)
          u_min = min(u_min, min(u0, u1));
        } else {
          in0 = m0 && s.x <= s_in;
          in1 = m1 && s.y <= s_in;
        }
        // every packed pair is evaluated (no per-pair branch), so the two pairs of a lane interleave
        const ClTab tb = tab[tj * CL_H + p];
        const F2 nqq = f2_mul(NQI[p], f2(qj));
        F2 elj, neel;
        F2 nc = cl_coef2<ENERGY, EW>(sc, s, nqq, tb, elj, neel);
        nc = f2(in0 ? nc.x : 0.f, in1 ? nc.y : 0.f);  // a select: the other half may hold inf / NaN
        FX[p] = f2_fma(dx, nc, FX[p]);
        FY[p] = f2_fma(dy, nc, FY[p]);
        FZ[p] = f2_fma(dz, nc, FZ[p]);
        GX = f2_fma(dx, nc, GX);
        GY = f2_fma(dy, nc, GY);
        GZ = f2_fma(dz, nc, GZ);
        if (ENERGY) {
          F2 e1 = f2(in0 ? elj.x : 0.f, in1 ? elj.y : 0.f), e2 = f2(in0 ? neel.x : 0.f, in1 ? neel.y : 0.f);
          if (!S.own_all) {
            const F2 wgt = f2(own_i[2 * p] + own_j, own_i[2 * p + 1] + own_j);
            e1 = f2_mul(e1, wgt);
            e2 = f2_mul(e2, wgt);
          }
          ELJ = f2_add(ELJ, e1);
          NEEL = f2_add(NEEL, e2);
        }
      }
      const float gx = -(GX.x + GX.y), gy = -(GY.x + GY.y), gz = -(GZ.x + GZ.y);
      if (gx != 0.f || gy != 0.f || gz != 0.f) red_add_f32x4(reinterpret_cast<float4*>(mad_wide_u32(jslot, 16u, f_base)), gx, gy, gz);
    };
    // (float4 and int4 records alike: 16 bytes at slot * 16)
    auto record_of = [&](unsigned en) { return ldg_s32x4(mad_wide_u32(en & 0xffffffu, 16u, rec_base)); };
    auto mask_of = [&](int e) { return (unsigned)lds_u8(mbuf + (unsigned)e); };

    // batches: entries from shared memory, partner records gathered one batch ahead
    if (nb) {
      unsigned en = lds_u32(ebuf + 4u * lane);
      unsigned mk = 0 < nbA ? mask_of(lane) : 0xffu;
      int4 rj = record_of(en);
#pragma unroll CL_UNROLL_N
      for (int b = 0; b < nb; ++b) {
        unsigned en_n = en, mk_n = 0xffu;
        int4 rj_n = rj;
        if (b + 1 < nb) {
          en_n = lds_u32(ebuf + 4u * ((b + 1) * 32 + lane));
          if (b + 1 < nbA) mk_n = mask_of((b + 1) * 32 + lane);
          rj_n = record_of(en_n);
        }
        unsigned m = mk & imask;
        if ((en & 0xffffffu) >= nslots_cap) m = 0;  // padding entry: the dummy record interacts with nothing
        body(en, m, rj);
        en = en_n;
        mk = mk_n;
        rj = rj_n;
      }
      phase ^= 1u << which;
    }
    // ---- forces on the cluster's atoms: reduce over the lanes, one reduction per atom
#pragma unroll
    for (int p = 0; p < CL_H; ++p) {
      const float ax = warp_sum(FX[p].x), ay = warp_sum(FY[p].x), az = warp_sum(FZ[p].x);
      const float bx = warp_sum(FX[p].y), by = warp_sum(FY[p].y), bz = warp_sum(FZ[p].y);
      if (lane == 0) {
        if ((imask >> (2 * p)) & 1u) red_add_f32x4(fout + s0 + 2 * p, ax, ay, az);
        if ((imask >> (2 * p + 1)) & 1u) red_add_f32x4(fout + s0 + 2 * p + 1, bx, by, bz);
      }
    }
    if (PERIODIC && __any_sync(0xffffffffu, u_min <= b_band)) {
      ClExactArgs a;
      a.xf = xf;
      a.xq = xq;
      a.xw = C.xw + sb;
      a.f = fout;
      a.ent = C.entries + (cb + c) * (size_t)stride_e;
      a.msk = mrow;
      a.g = S.grid + r;
      a.AB = S.AB;
      a.mcap = C.mcap;
      a.slots = C.slots;
      a.c = c;
      a.ntypes = S.ntypes;
      a.perm = C.perm + sb;
      a.own_lo = S.own_lo;
      a.own_n = S.own_n;
      a.own_all = S.own_all;
      a.terms = S.pp.terms;
      a.s_lo = s_in;
      a.s_hi = s_hi;
      a.s_max = S.pp.s_max;
      const float2 ee = EW ? cl_exact_pass_ew<ENERGY>(a, mt_cur, sc) : cl_exact_pass<ENERGY>(a, mt_cur, sc);
      ex_lj += ee.x;
      ex_el += ee.y;
    }
    if (ENERGY) {
      acc_lj += (double)(ELJ.x + ELJ.y) + (double)ex_lj;
      acc_el += (double)ex_el - (double)(NEEL.x + NEEL.y);
      ELJ = f2(0.f);
      NEEL = f2(0.f);
      ex_lj = 0.f;
      ex_el = 0.f;
    }
    which ^= 1;
  }
  if (ENERGY) {
    double* E = energies + (size_t)r * TMD_NUM_ENERGIES;
    __syncthreads();
    if (el_on) block_accumulate<CL_WARPS>(acc_el, E + TMD_E_ELECTROSTATICS, sh.red);
    if (lj_on) block_accumulate<CL_WARPS>(acc_lj, E + TMD_E_LJ, sh.red);
  }
}
template <bool ENERGY, bool PERIODIC>
__global__ void __launch_bounds__(CL_WARPS * 32, CL_MINBLOCKS)
k_cpair(DeviceState S, SwitchConsts sc, double* __restrict__ energies) {
  cpair_body<ENERGY, PERIODIC, false>(S, sc, energies);
}
// particle-mesh Ewald contexts (periodic only): real-space Ewald electrostatics (sc from make_switch_consts_ewald)
template <bool ENERGY>
__global__ void __launch_bounds__(CL_WARPS * 32, CL_MINBLOCKS)
k_cpair_ew(DeviceState S, SwitchConsts sc, double* __restrict__ energies) {
  cpair_body<ENERGY, true, true>(S, sc, energies);
}

// forces[i] = pair force of the atom's slot  (systems without bonded terms; otherwise k_bonded_sum adds on the way)
__global__ void k_cunsort(DeviceState S, float* __restrict__ forces) {
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.natoms) return;
  const size_t a = (size_t)r * S.natoms + i;
  const float4 f = S.cl.f[cl_slot_base(S.cl, r) + S.cl.inv[a]];
  forces[a * 3 + 0] = f.x;
  forces[a * 3 + 1] = f.y;
  forces[a * 3 + 2] = f.z;
}

// ---- the reference's neighbour list from the cluster lists (tmd_export_pairs) ------------------------
__global__ void k_cexport_pairs(DeviceState S, int r, int* __restrict__ pairs, long long capacity, unsigned long long* count) {
  const ClusterState& C = S.cl;
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int ncl = C.nslots[r] / CL;
  if (c >= ncl) return;
  const size_t sb = cl_slot_base(C, r), cb = cl_cluster_base(C, r);
  const Grid* g = S.grid + r;
  const int2 mt = C.meta[cb + c];
  const unsigned imask = (unsigned)mt.x >> 24;
  const unsigned* ent = C.entries + (cb + c) * (size_t)(C.mcap + C.ecap);
  const unsigned char* msk = C.masks + (cb + c) * (size_t)C.mcap;
  for (int region = 0; region < 2; ++region) {
    const int n = region == 0 ? (mt.x & 0xffffff) : mt.y;
    const unsigned* e = region == 0 ? ent : ent + C.mcap;
    for (int k = lane; k < n; k += 32) {
      const unsigned en = e[k];
      const int sj = (int)(en & 0xffffffu);
      if (sj >= C.slots) continue;
      const unsigned m = (region == 0 ? (unsigned)msk[k] : 0xffu) & imask;
      const float4 pj = C.xq[sb + sj];
      const int aj = C.perm[sb + sj];
      for (int i = 0; i < CL; ++i) {
        if (!((m >> i) & 1u)) continue;
        const float4 pi = C.xq[sb + c * CL + i];
        bool in;
        if (g->periodic)
          in = ref_inside(pi.x, pi.y, pi.z, pj.x, pj.y, pj.z, g->L[0], g->L[1], g->L[2], g->invL[0], g->invL[1], g->invL[2], S.pp.s_max);
        else
          in = norm2_ref(sub_rn(pi.x, pj.x), sub_rn(pi.y, pj.y), sub_rn(pi.z, pj.z)) <= S.pp.s_max;
        if (in) {
          const int ai = C.perm[sb + c * CL + i];
          const unsigned long long slot = atomicAdd(count, 1ull);
          if ((long long)slot < capacity) {
            pairs[2 * slot] = min(ai, aj);
            pairs[2 * slot + 1] = max(ai, aj);
          }
        }
      }
    }
  }
}

}  // namespace tmd
