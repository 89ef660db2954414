// neighbor.cuh -- cell list + Verlet neighbour list, built on the device.
//
// The reference has no neighbour search: it evaluates every pair of its static
// all-pairs table and masks with dist <= cutoff each step (forces.py:264-269;
// torchmd/neighbourlist.py is an unused stub whose fixed-width binning would
// miss cross-boundary pairs, SURVEY.md section 8a-19).  Here:
//
//   k_prepare     every call: displacement test against the positions of the
//                 last build (sets the rebuild flag) + refresh of the sorted
//                 position/charge records the pair kernel gathers from.
//   k_bounds/k_grid  (non-periodic only) bounding box -> cell grid.
//   k_bin         cell index per atom + counting pass.
//   k_scan        exclusive scan of the cell counts (one CTA per replica).
//   k_place       counting-sort scatter.
//   k_sort_pack   order every cell by original atom index (deterministic),
//                 write the sorted records and the inverse permutation.
//   k_build_list  full Verlet list: one CTA per cell stages the surrounding cells in
//                 shared memory (already shifted by their periodic image) and writes,
//                 for every atom of the cell, all partners within cutoff+skin that are
//                 not excluded into one 128-byte-aligned row per atom.
//
// Every rebuild kernel returns immediately unless the replica's rebuild flag is
// set, so the host can enqueue them unconditionally (no host round trip).  The
// flag, its parity and every counter live on the device: a captured CUDA graph of
// one step is replayable.
#pragma once
#include "context.cuh"
#include "ptx.cuh"

namespace tmd {

__device__ __forceinline__ int enc_float(float f) {
  int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7fffffff;
}
__device__ __forceinline__ float dec_float(int i) {
  return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff);
}

__device__ __forceinline__ int cell_of_point(const Grid& g, float x, float y, float z) {
  float p[3] = {x, y, z};
  int c[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    int ci;
    if (g.periodic) {
      float f = p[d] * g.invL[d];
      f -= floorf(f);  // [0,1]
      ci = (int)(f * (float)g.n[d]);
    } else {
      ci = (int)floorf((p[d] - g.origin[d]) * g.inv_w[d]);
    }
    c[d] = max(0, min(ci, g.n[d] - 1));
  }
  return (c[2] * g.n[1] + c[1]) * g.n[0] + c[0];
}

// ---- every call ---------------------------------------------------------------
// One atom of the per-call preparation: displacement trigger against the positions of the last
// rebuild, far-position check, refresh of the sorted records (float and fixed-point), largest
// |coordinate|.  (x, y, z) is the atom's current position.
__device__ __forceinline__ void prepare_atom(const DeviceState& S, int r, int i, int parity, float x, float y, float z) {
  int* fl = S.flags + r * F_COUNT;
  const size_t a = (size_t)r * S.natoms + i;
  const float4 ref = S.pos_ref[a];
  const float dx = x - ref.x, dy = y - ref.y, dz = z - ref.z;
  const float d2 = dx * dx + dy * dy + dz * dz;
  if (!(d2 <= S.trigger2)) {  // also true for NaN (= no list yet)
    if (fl[F_REBUILD0 + parity] == 0) {
      fl[F_REBUILD0 + parity] = 1;
      // inside a CUDA graph the rebuild kernels sit in the body of a conditional node: switch it on
      // (cudaGraphSetConditional is a driver-resolved builtin, bound when the module loads)
      if (S.cond) cudaGraphSetConditional((cudaGraphConditionalHandle)S.cond, 1u);
    }
  }
  if (S.check_far) {
    const Grid* g = S.grid + r;
    if (!(fabsf(x) < 2000.f * g->L[0]) || !(fabsf(y) < 2000.f * g->L[1]) || !(fabsf(z) < 2000.f * g->L[2]))
      fl[F_FARPOS] = 1;
  }
  if (S.cl.on) {  // cluster path (cluster.cuh): slot record refreshed, force accumulator of the slot cleared
    const size_t s = (size_t)r * (S.cl.slots + 1) + S.cl.inv[a];
    S.cl.xq[s] = make_float4(x, y, z, S.q[i]);
    S.cl.f[s] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (S.cl.xf) {  // periodic box: fixed-point record + largest |coordinate| for the decision band
      const Grid* g = S.grid + r;
      S.cl.xf[s] = make_int4(fx_encode(x, g->fx_inv[0]), fx_encode(y, g->fx_inv[1]), fx_encode(z, g->fx_inv[2]), __float_as_int(S.q[i]));
      float m = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
      if (!(fabsf(x) < INFINITY) || !(fabsf(y) < INFINITY) || !(fabsf(z) < INFINITY)) m = INFINITY;
      const unsigned am = __activemask();
      const int mb = __reduce_max_sync(am, __float_as_int(m));
      if ((threadIdx.x & 31) == __ffs(am) - 1 && mb > fl[F_PMAX]) atomicMax(fl + F_PMAX, mb);
    }
    return;
  }
  const int k = S.inv[a];
  S.xq_s[(size_t)r * (S.natoms + 1) + k] = make_float4(x, y, z, S.q[i]);
  if (S.xf_s) {  // fixed-point records of the periodic pair kernel (physics.cuh, fx_encode)
    const Grid* g = S.grid + r;
    S.xf_s[(size_t)r * (S.natoms + 1) + k] =
        make_int4(fx_encode(x, g->fx_inv[0]), fx_encode(y, g->fx_inv[1]), fx_encode(z, g->fx_inv[2]),
                  __float_as_int(S.q[i]));
    float m = fmaxf(fabsf(x), fmaxf(fabsf(y), fabsf(z)));
    if (!(fabsf(x) < INFINITY) || !(fabsf(y) < INFINITY) || !(fabsf(z) < INFINITY)) m = INFINITY;
    const unsigned am = __activemask();
    const int mb = __reduce_max_sync(am, __float_as_int(m));  // non-negative floats order like ints
    if ((threadIdx.x & 31) == __ffs(am) - 1 && mb > fl[F_PMAX]) atomicMax(fl + F_PMAX, mb);
  }
}

__global__ void k_prepare(DeviceState S, const float* __restrict__ pos) {
  const int parity = (int)(S.counters[0] & 1ull);  // device-resident: the launch sequence is CUDA-graph replayable
  const int r = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) S.flags[r * F_COUNT + F_REBUILD0 + (parity ^ 1)] = 0;  // nobody reads or sets that one now
  if (i >= S.natoms) return;
  const size_t a = (size_t)r * S.natoms + i;
  prepare_atom(S, r, i, parity, pos[a * 3 + 0], pos[a * 3 + 1], pos[a * 3 + 2]);
}

// ---- rebuild phases -----------------------------------------------------------------
// Each phase is a device function over a (bx of nbx blocks) slice of the grid with
// grid-stride loops; the gated kernels below run one phase each.

// non-periodic bounding box
__device__ __forceinline__ void phase_bounds(const DeviceState& S, int r, int bx, int nbx,
                                             const float* __restrict__ pos) {
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (int i = bx * blockDim.x + threadIdx.x; i < S.natoms; i += nbx * blockDim.x) {
    const size_t a = ((size_t)r * S.natoms + i) * 3;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], pos[a + d]);
      hi[d] = fmaxf(hi[d], pos[a + d]);
    }
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    for (int o = 16; o; o >>= 1) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
  }
  if ((threadIdx.x & 31) == 0) {
    int* b = reinterpret_cast<int*>(S.bounds) + r * 6;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      atomicMin(b + d, enc_float(lo[d]));
      atomicMax(b + 3 + d, enc_float(hi[d]));
    }
  }
}

// cell grid from the bounding box (one thread per replica)
__device__ __forceinline__ void phase_grid(const DeviceState& S, int r) {
  int* b = reinterpret_cast<int*>(S.bounds) + r * 6;
  Grid g;
  g.periodic = 0;
  int cap = 1;
  while ((cap + 1) * (cap + 1) * (cap + 1) <= S.max_cells) ++cap;
  const float w0 = S.rlist / (float)S.nsub;  // +inf without cutoff
  g.ncells = 1;
  for (int d = 0; d < 3; ++d) {
    const float lo = dec_float(b[d]), hi = dec_float(b[3 + d]);
    const float ext = fmaxf(hi - lo, 0.0f);
    float w = fmaxf(w0, ext / (float)cap * 1.0001f);
    int n = isinf(w) ? 1 : min(cap, (int)(ext / w) + 1);
    g.n[d] = n;
    g.reach[d] = (n > 1) ? S.nsub : 0;
    g.L[d] = 0.0f;
    g.invL[d] = 0.0f;
    g.origin[d] = lo;
    g.inv_w[d] = isinf(w) ? 0.0f : 1.0f / w;
    g.ncells *= n;
    b[d] = enc_float(INFINITY);  // re-arm for the next build
    b[3 + d] = enc_float(-INFINITY);
  }
  S.grid[r] = g;
}

// counting sort by cell, pass 1: cell index per atom + slot in the cell
__device__ __forceinline__ void phase_bin(const DeviceState& S, int r, int bx, int nbx,
                                          const float* __restrict__ pos) {
  const int ncells = S.grid[r].ncells;
  for (int i = bx * blockDim.x + threadIdx.x; i < S.natoms; i += nbx * blockDim.x) {
    const size_t a = (size_t)r * S.natoms + i;
    const float x = pos[a * 3 + 0], y = pos[a * 3 + 1], z = pos[a * 3 + 2];
    int c = cell_of_point(S.grid[r], x, y, z);
    if (!isfinite(x + y + z)) {  // blown-up coordinates: report, and spread them so no cell degenerates
      S.flags[r * F_COUNT + F_FARPOS] = 1;
      c = i % ncells;
    }
    S.cell_of[a] = c;
    const int slot = atomicAdd(S.cell_count + (size_t)r * (S.max_cells + 1) + c, 1);
    S.rank[a] = ncells == 1 ? i : slot;  // one cell (small box / no cutoff): already in index order
    S.pos_ref[a] = make_float4(x, y, z, 0.0f);
  }
}

// exclusive scan of the cell counts by ONE block (any multiple of 32 threads up to 1024)
__device__ __forceinline__ void phase_scan(const DeviceState& S, int r, int* warp_tot /*32 ints shared*/) {
  const int n = S.grid[r].ncells;
  const int nt = blockDim.x;
  const int* cnt = S.cell_count + (size_t)r * (S.max_cells + 1);
  int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  const int chunk = (n + nt - 1) / nt;
  const int b = threadIdx.x * chunk, e = min(n, b + chunk);
  int sum = 0;
  for (int c = b; c < e; ++c) sum += cnt[c];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = nt >> 5;
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
    warp_tot[lane] = ti - t;  // exclusive offset of each warp
  }
  __syncthreads();
  int run = warp_tot[wid] + incl - sum;
  for (int c = b; c < e; ++c) {
    start[c] = run;
    run += cnt[c];
  }
  if (threadIdx.x == nt - 1) start[n] = run;  // inclusive prefix of the last thread = total
  __syncthreads();
}

// counting sort, pass 2: scatter
__device__ __forceinline__ void phase_place(const DeviceState& S, int r, int bx, int nbx) {
  const int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  for (int i = bx * blockDim.x + threadIdx.x; i < S.natoms; i += nbx * blockDim.x) {
    const size_t a = (size_t)r * S.natoms + i;
    S.perm[(size_t)r * S.natoms + start[S.cell_of[a]] + S.rank[a]] = i;
  }
}

// One warp per cell: sort the cell's atoms by original index, then emit the sorted
// records.  Cells are small (a few to a few tens of atoms); rank-by-counting.
__device__ __forceinline__ void phase_sort_pack(const DeviceState& S, int r, int bx, int nbx) {
  const int lane = threadIdx.x & 31;
  const int warps_per_grid = nbx * (blockDim.x >> 5);
  const int ncells = S.grid[r].ncells;
  const int gper = S.grid[r].periodic;
  const float gL0 = S.grid[r].L[0], gL1 = S.grid[r].L[1], gL2 = S.grid[r].L[2];
  const float giL0 = S.grid[r].invL[0], giL1 = S.grid[r].invL[1], giL2 = S.grid[r].invL[2];
  const size_t base = (size_t)r * S.natoms;
  int* perm = S.perm + base;
  int* tmp = S.rank + base;  // free after the scatter
  int* cnt = S.cell_count + (size_t)r * (S.max_cells + 1);
  const int* start = S.cell_start + (size_t)r * (S.max_cells + 1);
  for (int c = bx * (blockDim.x >> 5) + (threadIdx.x >> 5); c < ncells; c += warps_per_grid) {
    const int b = start[c], n = start[c + 1] - b;
    if (lane == 0) cnt[c] = 0;  // leave the counters clean for the next build
    if (ncells == 1) {
      // single cell: phase_bin placed the atoms in index order already
    } else if (n <= 32) {
      const int v = lane < n ? perm[b + lane] : 0x7fffffff;
      int rk = 0;
      for (int m = 0; m < n; ++m) rk += (__shfl_sync(0xffffffffu, v, m) < v);
      __syncwarp();
      if (lane < n) perm[b + rk] = v;
    } else {
      for (int e = lane; e < n; e += 32) {
        const int v = perm[b + e];
        int rk = 0;
        for (int m = 0; m < n; ++m) rk += (perm[b + m] < v);
        tmp[b + rk] = v;
      }
      __syncwarp();
      __threadfence_block();
      for (int e = lane; e < n; e += 32) perm[b + e] = tmp[b + e];
    }
    __syncwarp();
    __threadfence_block();
    for (int e = lane; e < n; e += 32) {
      const int i = perm[b + e];
      const float4 p = S.pos_ref[base + i];
      S.inv[base + i] = b + e;
      S.xq_s[(size_t)r * (S.natoms + 1) + b + e] = make_float4(p.x, p.y, p.z, S.q[i]);
      if (S.xf_s) {
        const Grid* g = S.grid + r;
        S.xf_s[(size_t)r * (S.natoms + 1) + b + e] =
            make_int4(fx_encode(p.x, g->fx_inv[0]), fx_encode(p.y, g->fx_inv[1]), fx_encode(p.z, g->fx_inv[2]),
                      __float_as_int(S.q[i]));
      }
      S.type_s[base + b + e] = S.type[i];
      float wx = p.x, wy = p.y, wz = p.z;  // coordinates folded into [0, L] for the list build
      if (gper) {
        wx -= gL0 * floorf(wx * giL0);
        wy -= gL1 * floorf(wy * giL1);
        wz -= gL2 * floorf(wz * giL2);
      }
      S.xw_s[base + b + e] = make_float4(wx, wy, wz, 0.f);
    }
  }
}

// gated kernels: a replica without a pending rebuild returns at once
#define TMD_GATE                                                                    \
  const int parity = (int)(S.counters[0] & 1ull); /* device-resident: replayable */ \
  if (!S.flags[blockIdx.y * F_COUNT + F_REBUILD0 + parity]) return;
__global__ void k_bounds(DeviceState S, const float* __restrict__ pos) {
  TMD_GATE
  phase_bounds(S, blockIdx.y, blockIdx.x, gridDim.x, pos);
}
__global__ void k_grid(DeviceState S) {
  const int parity = (int)(S.counters[0] & 1ull);
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < S.nrep && S.flags[r * F_COUNT + F_REBUILD0 + parity]) phase_grid(S, r);
}
__global__ void k_bin(DeviceState S, const float* __restrict__ pos) {
  TMD_GATE
  phase_bin(S, blockIdx.y, blockIdx.x, gridDim.x, pos);
}
__global__ void __launch_bounds__(1024) k_scan(DeviceState S) {
  const int parity = (int)(S.counters[0] & 1ull);
  if (!S.flags[blockIdx.x * F_COUNT + F_REBUILD0 + parity]) return;
  __shared__ int warp_tot[32];
  phase_scan(S, blockIdx.x, warp_tot);
}
__global__ void k_place(DeviceState S) {
  TMD_GATE
  phase_place(S, blockIdx.y, blockIdx.x, gridDim.x);
}
__global__ void k_sort_pack(DeviceState S) {
  TMD_GATE
  phase_sort_pack(S, blockIdx.y, blockIdx.x, gridDim.x);
}

// ---- rebuild: Verlet list ---------------------------------------------------------------
// One CTA per cell.  The atoms of the (2*reach+1)^3 surrounding cells are staged in
// shared memory once per cell, already shifted by the periodic image of their cell, so
// the inner loop is a bare distance test on shared-memory operands: no per-pair minimum
// image, no per-atom cell arithmetic, no global gathers.  Cells adjacent in x are
// adjacent in memory, so every (dz,dy) row is one or two contiguous runs copied with
// coalesced 16-byte loads.  Each warp then takes atoms of the cell in turn and appends
// the accepted partners (sorted indices) to the atom's 128-byte-aligned row.  The test
// is generous (rlist carries a safety margin); the exact reference predicate is applied
// by the pair kernel.  Row order is fixed by the run order: deterministic.
#ifndef BT_WARPS_N
#define BT_WARPS_N 4
#endif
#ifndef BT_MINBLOCKS
#define BT_MINBLOCKS 6
#endif
constexpr int BT_WARPS = BT_WARPS_N;
#ifndef BT_TILE_N
#define BT_TILE_N 2048
#endif
constexpr int BT_TILE = BT_TILE_N;   // candidates staged per pass (16 B each)
constexpr int BT_MAXRUN = 64;   // (2*2+1)^2 rows x 2 segments = 50
constexpr int BT_MAXI = 256;    // atoms of the cell handled per pass

struct Run {
  int a0, len;
  float sx, sy, sz;
};

// Every 32-candidate chunk of the tile gets a bounding box; an atom only walks the chunks
// whose box comes within the list radius (the sweep volume is ~5x the list sphere, so most
// chunks cannot contribute).  Skipped chunks hold no accepted candidate, so the rows are
// the same as those of a walk over every chunk.
constexpr int BT_CHUNKS = BT_TILE / 32;
static_assert(BT_CHUNKS <= 64, "the per-atom chunk mask is 64 bits");

struct BuildShared {
  float4 tile[BT_TILE];
  Run runs[BT_MAXRUN];
  int roff[BT_MAXRUN + 1];  // exclusive prefix of the run lengths
  int counts[BT_MAXI];
  float bb[BT_CHUNKS][6];   // per chunk: min x,y,z, max x,y,z over its finite records
  int jr[BT_CHUNKS][2];     // per chunk: smallest / largest sorted atom index among its records
  float2 pp[BT_WARPS][4];   // per warp, the x / y / z of its two atoms side by side (read back as register pairs)
};

// bounding boxes of the staged chunks (one warp per chunk; NaN records are left out: they
// fail every distance test anyway)
__device__ __forceinline__ void build_chunk_boxes(BuildShared& sh, int fill) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nchunks = (fill + 31) >> 5;
  for (int c = warp; c < nchunks; c += BT_WARPS) {
    const float4 p = sh.tile[c * 32 + lane];
    const float v[3] = {p.x, p.y, p.z};
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const bool ok = v[d] == v[d];
      const int lo = __reduce_min_sync(0xffffffffu, enc_float(ok ? v[d] : INFINITY));
      const int hi = __reduce_max_sync(0xffffffffu, enc_float(ok ? v[d] : -INFINITY));
      if (lane == 0) {
        sh.bb[c][d] = dec_float(lo);
        sh.bb[c][3 + d] = dec_float(hi);
      }
    }
    const int j = __float_as_int(p.w) & 0xffffff;  // (padding records carry 0xffffff: they only widen the range)
    const int jlo = __reduce_min_sync(0xffffffffu, j), jhi = __reduce_max_sync(0xffffffffu, j);
    if (lane == 0) {
      sh.jr[c][0] = jlo;
      sh.jr[c][1] = jhi;
    }
  }
}

// A warp takes TWO atoms of the cell through the staged chunks at a time.  The candidate record is loaded once for
// both, the two separations and squared distances are packed fp32x2 operations (physics.cuh F2: same rounding per
// half as the scalar expressions), and a chunk is visited if either atom's bounding-box test asks for it -- a chunk
// that an atom's own test had culled holds no candidate within its list radius, so visiting it adds nothing to that
// atom's row.
struct BuildAtom {
  int k;                        // sorted index
  float4 pi;                    // folded position
  int ne, e0, my_excl;          // exclusions: count, CSR offset, this lane's (first 32) as a sorted index
  int exlo, exhi;               // index range that holds the atom and its exclusions
  unsigned long long row_addr;  // its row
  int count;
  unsigned store;               // all ones if rows are written for this atom, 0 for a stand-in
};

template <bool WRAP>
__device__ __forceinline__ void build_process_tile_paired(const DeviceState& S, const Grid& g, size_t base,
                                                          BuildShared& sh, int fill, int b0, int nib, bool w0,
                                                          bool w1, bool w2) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  float rl2 = S.rlist2;
  int cap = S.row_cap;
  TMD_PIN_F(rl2);
  TMD_PIN_R(cap);
  const int nchunks = (fill + 31) >> 5;

  auto owned = [&](int k) {
    if (S.own_all) return true;
    const int io = S.perm[base + k];
    return io >= S.own_lo && io < S.own_lo + S.own_n;
  };
  auto load_atom = [&](int k, int ii, bool store) {
    BuildAtom a;
    a.k = k;
    a.pi = S.xw_s[base + k];
    a.ne = 0; a.e0 = 0; a.my_excl = -1;
    a.exlo = 0x7fffffff; a.exhi = -1;
    if (S.excl_ptr) {
      const int io = S.perm[base + k];
      a.e0 = S.excl_ptr[io];
      a.ne = S.excl_ptr[io + 1] - a.e0;
      for (int eb = 0; eb < a.ne; eb += 32) {
        const int v = (eb + lane < a.ne) ? S.inv[base + S.excl_idx[a.e0 + eb + lane]] : -1;
        if (eb == 0) a.my_excl = v;
        if (v >= 0) { a.exlo = min(a.exlo, v); a.exhi = max(a.exhi, v); }
      }
      for (int o = 16; o; o >>= 1) {
        a.exlo = min(a.exlo, __shfl_xor_sync(0xffffffffu, a.exlo, o));
        a.exhi = max(a.exhi, __shfl_xor_sync(0xffffffffu, a.exhi, o));
      }
    }
    a.exlo = min(a.exlo, k);
    a.exhi = max(a.exhi, k);
    a.row_addr = reinterpret_cast<unsigned long long>(S.nbr + (base + k) * (size_t)cap);
    a.count = sh.counts[ii];
    a.store = store ? 0xffffffffu : 0u;
    return a;
  };
  // chunks within the list radius of the atom (lane c tests chunks c and c+32) and, of those, the ones
  // whose index range can hold the atom or one of its exclusions
  auto chunk_masks = [&](const BuildAtom& a, unsigned mh[2], unsigned sp[2]) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = lane + 32 * h;
      bool v = false;
      if (c < nchunks) {
        const float* bb = sh.bb[c];
        float dx = fmaxf(fmaxf(bb[0] - a.pi.x, a.pi.x - bb[3]), 0.f);
        float dy = fmaxf(fmaxf(bb[1] - a.pi.y, a.pi.y - bb[4]), 0.f);
        float dz = fmaxf(fmaxf(bb[2] - a.pi.z, a.pi.z - bb[5]), 0.f);
        if (WRAP) {
          if (w0) dx = 0.f;
          if (w1) dy = 0.f;
          if (w2) dz = 0.f;
        }
        v = (dx * dx + dy * dy + dz * dz) * 0.99999f <= rl2;
      }
      mh[h] = __ballot_sync(0xffffffffu, v);
      sp[h] = __ballot_sync(0xffffffffu, v && sh.jr[c][0] <= a.exhi && sh.jr[c][1] >= a.exlo);
    }
  };
  // lanes whose candidate j is the atom itself or one of its exclusions
  auto excluded = [&](const BuildAtom& a, int j) {
    bool excl = (j == a.k);
    const int nfast = min(a.ne, 32);
#pragma unroll 1
    for (int e = 0; e < nfast; ++e) excl |= (__shfl_sync(0xffffffffu, a.my_excl, e) == j);
#pragma unroll 1
    for (int e = 32; e < a.ne; ++e) excl |= (S.inv[base + S.excl_idx[a.e0 + e]] == j);
    return __ballot_sync(0xffffffffu, excl);
  };
  // keep the row padded to a multiple of 32 entries with the sentinel (record natoms holds NaN coordinates and fails
  // every cutoff test).  Later tiles overwrite the padding as the row grows.
  auto finish = [&](const BuildAtom& a, int ii) {
    if (!a.store) return;
    int* row = reinterpret_cast<int*>(a.row_addr);
    const int end = min((a.count + 31) & ~31, cap);
    for (int e = a.count + lane; e < end; e += 32) row[e] = S.natoms;
    if (lane == 0) sh.counts[ii] = a.count;
  };

  for (int ii = 2 * warp; ii < nib; ii += 2 * BT_WARPS) {
    const bool have1 = ii + 1 < nib;
    const bool s0 = owned(b0 + ii), s1 = have1 && owned(b0 + ii + 1);
    if (!s0 && !s1) continue;
    // a missing or foreign partner is replaced by a stand-in (the atom itself once more) that writes nothing
    const int i0 = s0 ? ii : ii + 1, i1 = (s0 && s1) ? ii + 1 : i0;
    BuildAtom A = load_atom(b0 + i0, i0, true);
    BuildAtom B = load_atom(b0 + i1, i1, s0 && s1);
    unsigned mhA[2], spA[2], mhB[2], spB[2];
    chunk_masks(A, mhA, spA);
    chunk_masks(B, mhB, spB);
    // values the chunk loop needs on every pass stay in registers (otherwise re-derived from the constant bank,
    // the row address with a dozen integer operations per store).  The two atoms' coordinates go through shared
    // memory once and come back as 64-bit loads: that is what makes them adjacent register PAIRS, the operand form
    // of the packed instructions (assembled from the two float4 records they cost two moves per use).
    __syncwarp();
    if (lane == 0) {
      sh.pp[warp][0] = make_float2(A.pi.x, B.pi.x);
      sh.pp[warp][1] = make_float2(A.pi.y, B.pi.y);
      sh.pp[warp][2] = make_float2(A.pi.z, B.pi.z);
    }
    __syncwarp();
    const float2 PX = sh.pp[warp][0], PY = sh.pp[warp][1], PZ = sh.pp[warp][2];
    unsigned lt_r = lt, lb_r = 1u << lane;
    smem_addr tile_lane = smem_address(sh.tile) + 16u * (unsigned)lane;  // this lane's record of chunk 0
    TMD_PIN_R(tile_lane);
    TMD_PIN_L(A.row_addr);
    TMD_PIN_L(B.row_addr);
    TMD_PIN_R(lt_r);
    TMD_PIN_R(lb_r);
    TMD_PIN_F(rl2);
    TMD_PIN_R(cap);
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
      unsigned visit = mhA[h] | mhB[h];
      const unsigned special = spA[h] | spB[h];
#pragma unroll 1
      while (visit) {
        const int cbit = __ffs((int)visit) - 1;
        visit &= visit - 1;
        const float4 pj = lds_f32x4(tile_lane + 512u * (unsigned)(cbit + 32 * h));  // a chunk is 32 records of 16 bytes
        const int entry = __float_as_int(pj.w);
        const int j = entry & 0xffffff;
        F2 s;
        if (WRAP) {  // a dimension too short for cells: one cell spans it, fold per pair (scalar: rare small boxes)
          float d[2][3] = {{A.pi.x - pj.x, A.pi.y - pj.y, A.pi.z - pj.z}, {B.pi.x - pj.x, B.pi.y - pj.y, B.pi.z - pj.z}};
          float q[2];
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            if (w0) d[t][0] -= g.L[0] * rintf(d[t][0] * g.invL[0]);
            if (w1) d[t][1] -= g.L[1] * rintf(d[t][1] * g.invL[1]);
            if (w2) d[t][2] -= g.L[2] * rintf(d[t][2] * g.invL[2]);
            q[t] = d[t][0] * d[t][0] + d[t][1] * d[t][1] + d[t][2] * d[t][2];
          }
          s = f2(q[0], q[1]);
        } else {
          const F2 px = f2(PX.x, PX.y), py = f2(PY.x, PY.y), pz = f2(PZ.x, PZ.y);
          const F2 dx = f2_add(px, f2(-pj.x)), dy = f2_add(py, f2(-pj.y)), dz = f2_add(pz, f2(-pj.z));
          s = f2_fma(dz, dz, f2_fma(dy, dy, f2_mul(dx, dx)));
        }
        unsigned mA = __ballot_sync(0xffffffffu, s.x <= rl2);
        unsigned mB = __ballot_sync(0xffffffffu, s.y <= rl2) & B.store;
        if ((special >> cbit) & 1u) {  // rare, warp-uniform: an atom itself or an exclusion may be in this chunk
          mA &= ~excluded(A, j);
          mB &= ~excluded(B, j);
        }
        const int slotA = A.count + __popc(mA & lt_r), slotB = B.count + __popc(mB & lt_r);
        if ((mA & lb_r) && slotA < cap) stg_u32(A.row_addr + 4ull * (unsigned)slotA, entry);
        if ((mB & lb_r) && slotB < cap) stg_u32(B.row_addr + 4ull * (unsigned)slotB, entry);
        A.count += __popc(mA);
        B.count += __popc(mB);
      }
    }
    finish(A, i0);
    finish(B, i1);
  }
}

__device__ __forceinline__ void phase_build(const DeviceState& S, int r, int bx, int nbx, BuildShared& sh) {
  int* fl = S.flags + r * F_COUNT;
  if (bx == 0 && threadIdx.x == 0) atomicAdd(fl + F_NREBUILD, 1);
  float4* const tile = sh.tile;
  Run* const runs = sh.runs;
  int* const roff = sh.roff;
  int* const counts = sh.counts;
  const Grid g = S.grid[r];
  const size_t base = (size_t)r * S.natoms;
  const float4* __restrict__ xw = S.xw_s + base;
  const int* __restrict__ start = S.cell_start + (size_t)r * (S.max_cells + 1);
  const bool w0 = g.periodic && g.n[0] == 1, w1 = g.periodic && g.n[1] == 1, w2 = g.periodic && g.n[2] == 1;
  const int tid = threadIdx.x, nthr = BT_WARPS * 32;
  const int ny = 2 * g.reach[1] + 1, nz = 2 * g.reach[2] + 1;
  const int nrows = ny * nz;  // <= 25, two run slots each

  // Grids of a few cells (small boxes, no cutoff): `split` CTAs share a cell, each taking every split-th pass of 64 of
  // its atoms, so that a 688-atom single-cell system is built by eleven CTAs instead of one.
  const int split = max(1, S.build_split);
  const int pass = split > 1 ? 64 : BT_MAXI;
  for (int wi = bx; wi < g.ncells * split; wi += nbx) {
    const int c = wi / split, sub = wi % split;
    const int b0c = start[c], ni = start[c + 1] - b0c;
    if (ni == 0 || sub * pass >= ni) continue;  // block-uniform
    if (!S.own_all) {       // decomposed run: skip cells without an owned atom
      int mine = 0;
      for (int t = tid; t < ni; t += nthr) {
        const int io = S.perm[base + b0c + t];
        mine |= (io >= S.own_lo && io < S.own_lo + S.own_n);
      }
      if (!__syncthreads_or(mine)) continue;
    }
    __syncthreads();        // previous cell's shared state no longer in use
    // ---- run table: one thread per (dz,dy) row of neighbour cells, all loads in flight together
    if (tid < BT_MAXRUN / 2) {
      Run ra = {0, 0, 0.f, 0.f, 0.f}, rb = {0, 0, 0.f, 0.f, 0.f};
      if (tid < nrows) {
        const int cx = c % g.n[0], cy = (c / g.n[0]) % g.n[1], cz = c / (g.n[0] * g.n[1]);
        int z2 = cz + tid / ny - g.reach[2], y2 = cy + tid % ny - g.reach[1];
        float sz = 0.f, sy = 0.f;
        bool valid = true;
        if (g.periodic) {
          if (z2 < 0) { z2 += g.n[2]; sz = -g.L[2]; } else if (z2 >= g.n[2]) { z2 -= g.n[2]; sz = g.L[2]; }
          if (y2 < 0) { y2 += g.n[1]; sy = -g.L[1]; } else if (y2 >= g.n[1]) { y2 -= g.n[1]; sy = g.L[1]; }
        } else {
          valid = z2 >= 0 && z2 < g.n[2] && y2 >= 0 && y2 < g.n[1];
        }
        if (valid) {
          const int rowbase = (z2 * g.n[1] + y2) * g.n[0];
          const int lo = cx - g.reach[0], hi = cx + g.reach[0];
          int alo = lo, ahi = hi, blo = 0, bhi = -1;
          float asx = 0.f, bsx = 0.f;
          if (g.periodic) {
            if (lo < 0) { alo = lo + g.n[0]; ahi = g.n[0] - 1; asx = -g.L[0]; blo = 0; bhi = hi; }
            else if (hi >= g.n[0]) { alo = lo; ahi = g.n[0] - 1; blo = 0; bhi = hi - g.n[0]; bsx = g.L[0]; }
          } else {
            alo = max(lo, 0);
            ahi = min(hi, g.n[0] - 1);
          }
          const int a0 = start[rowbase + alo], a1 = start[rowbase + ahi + 1];
          ra = {a0, a1 - a0, asx, sy, sz};
          if (bhi >= blo) {
            const int c0 = start[rowbase + blo], c1 = start[rowbase + bhi + 1];
            rb = {c0, c1 - c0, bsx, sy, sz};
          }
        }
      }
      runs[2 * tid] = ra;
      runs[2 * tid + 1] = rb;
      // exclusive scan of the 64 lengths by the first warp (two per lane)
      const int l0 = ra.len, l1 = rb.len;
      int incl = l0 + l1;
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (tid >= o) incl += v;
      }
      roff[2 * tid] = incl - l0 - l1;
      roff[2 * tid + 1] = incl - l1;
      if (tid == 31) roff[BT_MAXRUN] = incl;
    }
    __syncthreads();
    const int M = roff[BT_MAXRUN];
    for (int i0 = sub * pass; i0 < ni; i0 += split * pass) {
      const int nib = min(pass, ni - i0);
      const int b0 = b0c + i0;
      for (int t = tid; t < nib; t += nthr) counts[t] = 0;
      for (int t0 = 0; t0 < M; t0 += BT_TILE) {
        const int fill = min(BT_TILE, M - t0);
        __syncthreads();  // tile free, counts initialised
        // one warp per run, lanes stride its records (tile slot = run offset + position in the run).
        // The list entry: sorted index (24 bits) + atom type (8 bits), see pair.cuh
        for (int q = tid >> 5; q < BT_MAXRUN; q += BT_WARPS) {
          const Run rn = runs[q];
          const int first = roff[q] - t0;  // tile position of the run's first record (the run may straddle tiles)
          for (int u = (tid & 31); u < rn.len; u += 32) {
            const int at = first + u;
            if (at < 0 || at >= fill) continue;
            const int j = rn.a0 + u;
            const float4 p = xw[j];
            tile[at] = make_float4(p.x + rn.sx, p.y + rn.sy, p.z + rn.sz, __int_as_float(j | (S.type_s[base + j] << 24)));
          }
        }
        // pad the last 32-candidate chunk with records that pass no distance test
        for (int u = fill + tid; u < ((fill + 31) & ~31); u += nthr)
          tile[u] = make_float4(NAN, NAN, NAN, __int_as_float(0xffffff));  // NaN: fails `<= rlist2` even when that is +inf
        __syncthreads();
        build_chunk_boxes(sh, fill);
        __syncthreads();
        if (w0 || w1 || w2) build_process_tile_paired<true>(S, g, base, sh, fill, b0, nib, w0, w1, w2);
        else build_process_tile_paired<false>(S, g, base, sh, fill, b0, nib, w0, w1, w2);
      }
      __syncthreads();
      for (int t = tid; t < nib; t += nthr) {
        const int cnt = counts[t];
        S.nnbr[base + b0 + t] = min(cnt, S.row_cap);
        if (cnt > S.row_cap) fl[F_OVERFLOW] = 1;
        if (cnt > fl[F_MAXNBR]) atomicMax(fl + F_MAXNBR, cnt);
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(BT_WARPS * 32, BT_MINBLOCKS) k_build_list(DeviceState S) {
  TMD_GATE
  __shared__ BuildShared sh;
  phase_build(S, blockIdx.y, blockIdx.x, gridDim.x, sh);
}

// ---- inspection: the reference's neighbour list ----------------------------------------
// Applies the exact reference predicate to every listed pair and emits (i<j) in
// original atom indices.  Used by the bit-exact index test.
__global__ void k_export_pairs(DeviceState S, int r, int* __restrict__ out, long long capacity,
                               unsigned long long* __restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (k >= S.natoms) return;
  const Grid g = S.grid[r];
  const size_t base = (size_t)r * S.natoms;
  const float4* xq = S.xq_s + (size_t)r * (S.natoms + 1);
  const int* perm = S.perm + base;
  const int* row = S.nbr + (base + k) * (size_t)S.row_cap;
  const int n = S.nnbr[base + k];
  const float4 pi = xq[k];
  const int oi = perm[k];
  if (!S.own_all && (oi < S.own_lo || oi >= S.own_lo + S.own_n)) return;  // rows of other ranks are not built here
  const unsigned lt = (1u << lane) - 1u;
  for (int e0 = 0; e0 < n; e0 += 32) {
    const int e = e0 + lane;
    bool ok = false;
    int oj = 0;
    if (e < n) {
      const int j = row[e] & 0xffffff;  // e < nnbr: never a padding entry
      const float4 pj = xq[j];
      float dx = sub_rn(pi.x, pj.x), dy = sub_rn(pi.y, pj.y), dz = sub_rn(pi.z, pj.z);
      if (g.periodic) {  // always the guarded (exact) form here
        dx = min_image(dx, g.L[0], g.invL[0]);
        dy = min_image(dy, g.L[1], g.invL[1]);
        dz = min_image(dz, g.L[2], g.invL[2]);
      }
      oj = perm[j];
      ok = (norm2_ref(dx, dy, dz) <= S.pp.s_max) &&
           (oi < oj || (!S.own_all && (oj < S.own_lo || oj >= S.own_lo + S.own_n)));  // each pair once per owner set
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    unsigned long long b = 0;
    if (lane == 0 && m) b = atomicAdd(count, (unsigned long long)__popc(m));
    b = __shfl_sync(0xffffffffu, b, 0);
    if (ok) {
      const unsigned long long slot = b + __popc(m & lt);
      if ((long long)slot < capacity) {
        out[slot * 2 + 0] = oi;
        out[slot * 2 + 1] = oj;
      }
    }
  }
}

}  // namespace tmd
