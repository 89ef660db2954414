// context.cuh -- device-resident state of one tmd_ctx and small helpers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/tmd_b200.h"
#include "physics.cuh"

namespace tmd {

// Cell grid of one replica.  Filled on the host for periodic boxes
// (tmd_set_box) and by k_bounds_grid on the device for non-periodic systems.
struct Grid {
  int n[3];         // cells per dimension
  int reach[3];     // neighbour-cell reach per dimension (0 when n == 1)
  int ncells;       // n[0]*n[1]*n[2]
  int periodic;     // wrap cell indices / minimum image
  float L[3];       // box lengths (periodic) -- 0 otherwise
  float invL[3];    // 1/L
  float origin[3];  // lower corner (non-periodic); 0 for periodic
  float inv_w[3];   // 1 / cell width
  // fixed-point coordinates of the periodic pair kernel (physics.cuh, fx_encode)
  float fx_unit[3];     // L / 2^32
  float fx_c0, fx_c1;   // |s_fx - s_ref| <= fx_c0 + fx_c1 * max|coordinate|
  double fx_inv[3];     // 2^32 / L
};

// Flags/counters per replica (device ints).
enum {
  F_REBUILD0 = 0,  // rebuild request, even calls
  F_REBUILD1 = 1,  // rebuild request, odd calls
  F_OVERFLOW = 2,
  F_NREBUILD = 3,
  F_MAXNBR = 4,
  F_FARPOS = 5,    // a position was further than 2000 box lengths from the origin
  F_PMAX = 6,      // bits of the largest |coordinate| seen since the box was set (+inf if one was not finite)
  F_PEERWAIT = 7,  // (replica 0) the wait for the peers' position stores timed out
  F_CLFAIL = 8,    // cluster path: a cluster grew past the size the single image count per (cluster, partner) allows,
                   // or an exclusion set / segment table overflowed -> the host falls back to the full Verlet rows
  F_CLMAXA = 9,    // cluster path: most masked / plain entries any cluster wanted at the last builds
  F_CLMAXB = 10,
  F_COUNT = 12
};

// Cluster half-list path (cluster.cuh).  Slots: atoms sorted by cell row and x, rows padded to whole clusters.
struct ClusterState {
  int on;              // cluster path in use
  int slots;           // slot capacity per replica (a multiple of the cluster size); record `slots` is the dummy
  int nclusters_cap;   // slots / cluster size
  int ecap, mcap;      // plain / masked entries reserved per cluster (multiples of 32)
  float max_extent;    // largest bounding-box edge a cluster may have (periodic boxes)
  float4* xq;          // [rep*(slots+1) + s] raw x, y, z + scaled charge (every step)
  float4* f;           // [rep*(slots+1) + s] force accumulators (zeroed every step)
  float4* xw;          // coordinates folded into the box at the last build; .w = atom type (bits)
  int4* xf;            // fixed-point records (physics.cuh, fx_encode) of a periodic box: X, Y, Z + charge bits (every step)
  int* perm;           // slot -> atom (-1: padding)
  int* bucket;         // [(rep*max_cells + cell) * CL_BUCKET + k] atoms of a cell in arrival order (rebuild scratch)
  int* row_tot;        // [rep*(max_rows+1) + row] scan scratch: padded atoms of a cell row, then its first slot
  int max_rows;
  int* cell_owned;     // decomposed runs: owned atoms per cell (rebuild scratch), and
  int* owned_pre;      //   their running count inside each cell row
  int* inv;            // [rep*natoms + i] atom -> slot
  int* nslots;         // [rep] slots in use after the last build
  int2* meta;          // [rep*nclusters_cap + c] (masked entries | mask of real atoms << 24, plain entries), counts padded to 32
  unsigned* entries;   // [(rep*nclusters_cap + c) * (mcap + ecap)] masked region, then plain region
  unsigned char* masks;  // [(rep*nclusters_cap + c) * mcap] which atoms of the cluster a masked entry interacts with
};

struct DeviceState {
  // sizes
  int natoms, nrep;
  int row_cap;      // neighbour entries reserved per atom
  int max_cells;    // capacity of the cell arrays per replica
  int nsub;         // cells per list radius
  int build_split;  // full-row list build: CTAs that share one cell (grids of a few cells)
  int own_lo, own_n, own_all;  // atoms (original indices) whose forces this context computes; all by default
  unsigned long long* counters;  // [0] force calls (parity of the rebuild flag), [1] vv_first calls (Philox position), [2] copy of [1] taken by the cluster pair kernel
  unsigned long long cond;       // cudaGraphConditionalHandle of the rebuild body when this launch is a graph node; 0 otherwise
  int check_far;    // flag positions beyond 2000 box lengths (guard-free minimum image in use)
  // per-atom static data (original order)
  const float* q;        // charge * sqrt(coulomb constant)
  const int* type;       // atom type id
  const int* excl_ptr;   // CSR exclusions, original indices
  const int* excl_idx;
  // LJ tables
  const float2* AB;      // (T*T) {A,B}
  int ntypes;
  // per replica dynamic data (index [rep*natoms + k])
  float4* xq_s;          // sorted: raw x,y,z + scaled charge
  int4* xf_s;            // sorted: fixed-point x,y,z (fx_encode) + bits of the scaled charge; null = not in use
  int* type_s;           // sorted atom type
  float4* xw_s;          // sorted: coordinates folded into the box at the last build (list build only)
  int* perm;             // sorted slot -> original atom
  int* inv;              // original atom -> sorted slot
  float4* pos_ref;       // positions at the last rebuild (original order)
  int* cell_of;          // original atom -> cell
  int* rank;             // slot inside the cell handed out by the counting pass
  int* cell_count;       // [rep*(max_cells+1) + c]   zero outside rebuilds
  int* cell_start;       // exclusive scan of the counts (ncells+1 entries)
  int* nbr;              // [(rep*natoms + k)*row_cap + e]
  int* nnbr;             // neighbours of sorted atom k
  int* flags;            // [rep*F_COUNT + f]
  Grid* grid;            // [rep]
  float* bounds;         // [rep*6] min xyz, max xyz (non-periodic), as ordered ints
  // list parameters
  float rlist2;          // (cutoff+skin)^2 * (1+eps); +inf without cutoff
  float rlist;           // cutoff + skin
  float trigger2;        // (skin/2 - margin)^2 ; +inf without cutoff
  PairParams pp;
  ClusterState cl;
};

// P: type of the parameter rows, float ("precision: single") or double ("precision: double")
template <typename P>
struct BondedSetT {
  int n = 0;
  int* idx = nullptr;    // (n,k)
  P* prm = nullptr;      // (n,p)
  int* term_ptr = nullptr;  // torsions only
  P* terms = nullptr;
  int amber = 1;
};
using BondedSet = BondedSetT<float>;

// ---- "precision: double" (tmd_set_precision(ctx, 64)): full Verlet rows, fp64 state ------------
// The list build is the fp32 one, run on an fp32 shadow of the positions (the list is a superset
// of the pairs and decides nothing); the decision and every value are fp64.
struct alignas(32) Rec64 {
  double x, y, z, q;  // position + charge * sqrt(coulomb constant)
};
struct PairParams64 {
  uint32_t terms;
  int has_cutoff, has_switch, rfa, true_gradient;
  double s_max;        // largest double s with sqrt_rn(s) <= cutoff; +inf without cutoff
  double cutoff, switch_dist, inv_sw_width;  // 1 / (cutoff - switch_dist)
  // reaction-field constants (forces.py:466-468), or with particle-mesh Ewald alpha and 2 alpha / sqrt(pi)
  union { double krf; double ew_alpha; };
  union { double crf; double ew_beta; };
};
struct DeviceState64 {
  Rec64* xq_s;         // [rep*(natoms+1) + k] sorted records; record natoms is the NaN sentinel
  float* shadow;       // (R,N,3) positions rounded to fp32: what the list build reads
  const double* q;     // charge * sqrt(coulomb constant)
  const double* AB;    // (T*T) {A,B} interleaved
  const double* L;     // (R,3) box lengths
  double pos_limit;    // |coordinate| from which F_FARPOS is raised (the shadow's rounding must stay inside the list margin)
  PairParams64 pp;
};

}  // namespace tmd

struct tmd_ctx {
  int device = 0;
  int nsm = 1;  // SMs of the device: caps the grids of the grid-stride list-build kernels
  int natoms = 0, nrep = 0;
  tmd::DeviceState d{};
  // owned device buffers behind the const pointers in d
  float* q = nullptr;
  int* type = nullptr;
  int* excl_ptr = nullptr;
  int* excl_idx = nullptr;
  float2* AB = nullptr;
  tmd::BondedSet bonds, angles, torsions[2], pairs14;
  std::vector<int32_t> bonds_idx_h, angles_idx_h, torsions_idx_h[2], pairs14_idx_h;  // host copies for the atom CSR
  int* bonded_atom_ptr = nullptr;    // device CSR: atom -> bonded term entries (see bonded.cuh)
  int* bonded_entries = nullptr;
  int bonded_nentries = 0;
  uint32_t bonded_mask = 0;   // which bonded energy terms are enabled
  uint32_t pair_mask = 0;
  double coulomb = 0.0, cutoff = -1.0, switch_dist = -1.0, skin = 0.0;
  int rfa = 0;
  bool have_atoms = false, have_nonbonded = false, have_box = false, have_excl = false;
  bool excl_is_set = true;           // the exclusion CSR lists every pair in both rows, once, and no atom with itself
  bool periodic = false;
  bool safe_image = false;           // guard-free minimum image valid (see min_image_fast)
  int coop_blocks = 0;               // CTAs per replica of the cooperative rebuild kernel (0: separate kernels)
  int pair_mode = 0;                 // 1: LJ+switch + reaction-field Coulomb specialisation
  int exact_gradient = 0;            // tmd_set_force_convention: switched-LJ force as the true gradient
  int last_pair_kernel = 0;          // tmd_pair_kernel(): 0 float (k_pair), 1 k_pair_fx, 2 k_pair_fx2, 3 k_pair2_open
  bool fx_packed = false;            // TMD_B200_FX=2: k_pair_fx2 (fp32x2 arithmetic) where it applies
  int4* xf_buf = nullptr;            // fixed-point records (periodic pair kernel), owned; d.xf_s points here when in use
  bool cluster_failed = false;       // the cluster path reported F_CLFAIL: full rows until cluster_retry_at force calls
  int64_t cluster_retry_at = 0, cluster_retry_after = 0;
  int64_t rebuilds_before = 0;  // list builds counted before the last (re-)finalisation cleared the device flags
  // peer-to-peer position exchange (tmd_dd_*): one cudaMalloc holding [pos0 | pos1 | flags | sync]
  int dd_rank = -1, dd_world = 0;
  bool dd_connected = false;
  void* dd_base = nullptr;                    // this rank's allocation
  void* dd_peer_base[TMD_MAX_PEERS] = {};     // the peers' allocations as mapped here (own entry = dd_base)
  size_t dd_pos_bytes = 0;                    // bytes of one position buffer (offset of the second)
  unsigned* dd_sync = nullptr;                // local: [0] block ticket, [1] push epoch, [2] wait epoch
  std::vector<float> box_host;       // (nrep,3)
  std::vector<float> charges_host;   // unscaled charges
  int64_t launches = 0;
  int64_t force_calls = 0;
  double* ke_scratch = nullptr;      // (nrep) doubles for the host entry
  double* e_scratch = nullptr;       // (nrep, TMD_NUM_ENERGIES)
  // "precision: double" (tmd_set_precision)
  int precision = 32;
  bool touched = false;              // a setter has run: the precision is fixed
  tmd::DeviceState64 d64{};
  tmd::Rec64* xq64 = nullptr;        // owned buffers behind d64
  float* shadow = nullptr;
  double* q64 = nullptr;
  double* AB64 = nullptr;
  double* L64 = nullptr;
  std::vector<double> charges64_host, box64_host;
  tmd::BondedSetT<double> bonds64, angles64, torsions64[2], pairs1464;
};
