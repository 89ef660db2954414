// tmd_b200.cu -- C ABI (include/tmd_b200.h) over the sm_90a kernels.
// Host side only enqueues: no synchronisation and no allocation in the per-step
// entry points once the context is finalised.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "bonded.cuh"
#include "context.cuh"
#include "integrate.cuh"
#include "wrap.cuh"
#include "neighbor.cuh"
#include "pair.cuh"
#include "cluster.cuh"
#include "fused.cuh"
#include "double.cuh"
#include "constrain.cuh"
#include "pme.cuh"
#include "barostat.cuh"

using namespace tmd;

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define TMD_CUDA(call)                                                                          \
  do {                                                                                          \
    cudaError_t e__ = (call);                                                                   \
    if (e__ != cudaSuccess)                                                                     \
      return fail(TMD_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__));           \
  } while (0)

#define TMD_LAUNCHED(ctx, name)                                                                 \
  do {                                                                                          \
    (ctx)->launches++;                                                                          \
    cudaError_t e__ = cudaGetLastError();                                                       \
    if (e__ != cudaSuccess)                                                                     \
      return fail(TMD_ERR_CUDA, std::string("launch ") + name + ": " + cudaGetErrorString(e__)); \
  } while (0)

// Run-time switches: the environment decides ("0" off, "1"/"2" on), otherwise the default below
// (-DTMD_DEFAULT_<NAME>=... for an A/B build).
#ifndef TMD_DEFAULT_FX
#define TMD_DEFAULT_FX 2        // TMD_B200_FX: 1 fixed-point pair kernel, 2 + fp32x2 arithmetic
#endif
#ifndef TMD_DEFAULT_COOP
#define TMD_DEFAULT_COOP 0      // TMD_B200_COOP: rebuild as one cooperative launch
#endif
#ifndef TMD_DEFAULT_OVERLAP
#define TMD_DEFAULT_OVERLAP 1   // TMD_B200_OVERLAP: bonded kernel on a second stream
#endif
#ifndef TMD_DEFAULT_COND
#define TMD_DEFAULT_COND 0      // TMD_B200_COND: rebuild as a conditional node when captured (needs TMD_COND_NODE)
#endif
#ifndef TMD_DEFAULT_GRAPH
#define TMD_DEFAULT_GRAPH 1     // TMD_B200_GRAPH: tmd_md_steps replays a captured step
#endif
#ifndef TMD_DEFAULT_FUSESTEP
#define TMD_DEFAULT_FUSESTEP 1  // TMD_B200_FUSESTEP: second half of a step and first half of the next one in one kernel
#endif
#ifndef TMD_DEFAULT_FUSEPREP
#define TMD_DEFAULT_FUSEPREP 1  // TMD_B200_FUSEPREP: integrate + prepare in one kernel, bonded fold in the second kick
#endif
#ifndef TMD_DEFAULT_CLUSTER
#define TMD_DEFAULT_CLUSTER 1   // TMD_B200_CLUSTER: cluster half-list pair path (cluster.cuh) where it applies
#endif
static int env_switch(const char* name, int def) {
  const char* e = getenv(name);
  return (e && e[0] >= '0' && e[0] <= '9') ? (e[0] - '0') : def;
}

// Every kernel launch goes through here.  The product enqueues on the stream; the SIMT interpreter
// build of tests/simt (TMD_SIMT_HOST: the same kernels compiled for the CPU to check their logic
// without a GPU) runs the grid on the spot.
template <typename... KArgs, typename... Args>
inline void launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args&&... args) {
#if defined(TMD_SIMT_HOST)
  // (a capturing stream records the launch -- arguments by value, like a kernel node -- and the graph replays it)
  auto run = [kernel, grid, block, held = std::make_tuple(std::decay_t<Args>(args)...)]() {
    simt::run_grid(grid, block, [&]() { std::apply(kernel, held); });
  };
  if (simt_stub::capturing(st)) simt_stub::record(st, run);
  else run();
#else
  kernel<<<grid, block, 0, st>>>(std::forward<Args>(args)...);
#endif
}

template <typename... KArgs, typename... Args>
inline void launch_smem(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
#if defined(TMD_SIMT_HOST)
  (void)smem;
  launch(kernel, grid, block, st, std::forward<Args>(args)...);
#else
  kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
#endif
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

template <typename T>
int upload(T** dst, const T* src, size_t n) {
  if (*dst) {
    cudaFree(*dst);
    *dst = nullptr;
  }
  if (n == 0) return TMD_OK;
  TMD_CUDA(cudaMalloc((void**)dst, n * sizeof(T)));
  TMD_CUDA(cudaMemcpy(*dst, src, n * sizeof(T), cudaMemcpyHostToDevice));
  return TMD_OK;
}

template <typename T>
int device_alloc(T** dst, size_t n) {
  if (*dst) {
    cudaFree(*dst);
    *dst = nullptr;
  }
  if (n == 0) return TMD_OK;
  TMD_CUDA(cudaMalloc((void**)dst, n * sizeof(T)));
  return TMD_OK;
}

// page-locked host memory, so that a cudaMemcpyAsync from it neither stages nor waits (plain memory in the interpreter)
static void* stage_alloc(size_t bytes) {
#if defined(TMD_SIMT_HOST)
  return malloc(bytes);
#else
  void* p = nullptr;
  return cudaMallocHost(&p, bytes) == cudaSuccess ? p : nullptr;
#endif
}
static void stage_free(void* p) {
  if (!p) return;
#if defined(TMD_SIMT_HOST)
  free(p);
#else
  cudaFreeHost(p);
#endif
}


struct CtxPriv {
  // TMD_B200_OVERLAP=1: bonded kernel on a second stream, concurrent with the pair kernel
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  double* bonded_scratch = nullptr;  // (R,N,3) fp64
  // TMD_B200_COND=1: when a force call is being captured into a CUDA graph, the rebuild kernels go
  // into the body of a conditional node that k_prepare switches on (nothing is launched on the
  // steps that keep their list) instead of five kernels that return at once
  bool use_cond = false;
  cudaStream_t helper = nullptr;     // captures the body of the conditional node
  // TMD_B200_GRAPH=1: tmd_md_steps replays one captured step (two variants: with / without energies)
  bool use_graph = false;
  cudaStream_t gstream = nullptr;    // capture + replay stream (the caller's may be the legacy default stream)
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  // [0] a whole step, [1] a whole step with the energy outputs (the last, or only, step of a call);
  // TMD_B200_FUSESTEP=1 (cluster path): [2] the first step of a call without its second half-kick, [3] a middle
  // step that opens with k_cstep_boundary (second half of the step before + first half of this one), [4] the last
  // step: boundary, force call with energies, second half-kick with the kinetic energy
  static constexpr int NGRAPH = 5;
  cudaGraphExec_t exec[NGRAPH] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaGraph_t graph[NGRAPH] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  struct StepKey {
    float *pos, *vel, *forces;
    const float *masses, *vcoeff;
    double dt, gamma;
    uint64_t seed, first_step;
    double *energies, *ke;
  } step_key{};
  DeviceState step_state{};          // the kernel arguments baked into the captured steps
  bool steps_valid = false;
  int64_t step_launches[5] = {0, 0, 0, 0, 0};  // kernels of one captured step (rebuild body included)
  // TMD_B200_FUSEPREP=1: tmd_md_steps moves the atoms and prepares the force call in one kernel
  // (k_vv_first_prepare); the handle of the rebuild's conditional node is then made before that launch
  bool fuse_prepare = false;
  double* term_forces = nullptr;  // k_bonded_terms -> k_bonded_sum: force of every (term, slot), fp64 (R x slots x 3)
  size_t term_forces_len = 0;
  bool bonded_terms = true;       // TMD_B200_BONDED_TERMS=0: the one-kernel atom-centric k_bonded
  bool flags_live = false;  // the device flags hold counts of this context (set by the first finalisation)
  bool fuse_step = false;   // TMD_B200_FUSESTEP=1: k_cstep_boundary between the steps of one tmd_md_steps call
  bool fold_next = false;                       // tmd_md_steps: the vv_second that follows folds the bonded sums in (k_vv_second_fold)
  bool fold_pending = false;                    // set by enqueue_forces when it left them in the scratch buffer
  bool prepared = false;                        // the next enqueue_forces finds k_prepare's work done
  cudaGraphConditionalHandle prepared_cond = 0; // and this handle already handed to the kernel
  bool dirty = true;
  size_t nbr_entries = 0;
  // cluster path inside tmd_md_steps: the bonded kernel is folded into the second half-kick (fused.cuh)
  int64_t last_body_launches = 0; // kernels the last captured force call put into the rebuild's conditional body
  bool defer_bonded = false;      // set by tmd_md_steps for the force call it is about to make
  bool bonded_deferred = false;   // enqueue_forces left the bonded terms (and the unsort) to enqueue_vv_second
  double* deferred_energies = nullptr;
  BondedTables deferred_tables{};
  const float* deferred_pos = nullptr;
  // cluster path: owned buffers behind ctx->d.cl
  std::vector<void*> cl_bufs;
  int cl_blocks = 0;        // CTAs of k_cpair per replica
  size_t cl_smem = 0;       // its dynamic shared memory
  std::vector<cudaEvent_t> ev;  // pair-kernel timing samples (begin,end interleaved)
  int ev_used = 0;
  bool profiling = false;
  // tmd_set_constraints: rigid waters and X-H clusters (constrain.cuh); con_ngroups == 0 means none
  int con_ngroups = 0, con_nfree = 0;
  CGroup* con_groups = nullptr;
  int* con_free = nullptr;
  double* con_L = nullptr;   // (R,3) box lengths, 0 without a box
  void* con_ref = nullptr;   // (R,N,3) positions before the drift, in the context's precision
  int* con_fail = nullptr;   // a group's SHAKE iteration did not converge (tmd_get_stats reports it)
  const void* con_pos = nullptr;  // positions of the last tmd_vv_first[_f64]: what tmd_vv_second[_f64] constrains against
  // tmd_set_pme: particle-mesh Ewald (pme.cuh); pme_tol <= 0 means off.  alpha and the grid are chosen by pme_choose.
  double pme_tol = 0.0, pme_alpha = 0.0;
  int pme_K[3] = {0, 0, 0};
  PmeArgs pme{};  // the reciprocal kernels' arguments (buffers below, owned)
  double *pme_q = nullptr, *pme_L = nullptr, *pme_tw = nullptr, *pme_econst = nullptr;
  unsigned long long* pme_qgrid = nullptr;
  void *pme_cgrid = nullptr, *pme_infl = nullptr;
  cudaStream_t pme_side = nullptr;  // fp32: the reciprocal chain runs here, beside the pair kernel
  cudaEvent_t pme_fork = nullptr, pme_join = nullptr;
  double* pme_mod = nullptr;        // B-spline moduli |b(m)|^2 of the grid, K[0] + K[1] + K[2] (k_pme_influence)
  double pme_q2 = 0.0, pme_qsum = 0.0;  // sum q^2 and sum q (scaled charges): the self and background energies
  bool pme_pinned = false;          // tmd_rescale_box keeps alpha and the grid; tmd_set_box / tmd_set_pme choose again
  int64_t step_captures = 0;        // tmd_step_captures: captures of a tmd_md_steps step graph
  // tmd_rescale_box: the cell grids of the boxes held (host copy), the choices finalize made that a rescale must keep
  std::vector<Grid> grids;
  bool grid_fx = false;             // the grids carry fixed-point units (k_pair_fx, cluster path)
  bool rescaled = false;            // cl.max_extent has been set to the bound every fast-path box keeps
  double cl_bound = 0.0;            // that bound (A)
  double* box_dev = nullptr;        // (R,3) box lengths on the device, for tmd_scale_molecules
  void* rs_stage = nullptr;         // page-locked staging of the per-box tables a rescale copies
  size_t rs_stage_bytes = 0;
  cudaEvent_t rs_done = nullptr;    // recorded after the staging was read
  // tmd_set_molecules: molecule CSR (barostat.cuh)
  int mol_n = 0;
  int *mol_ptr = nullptr, *mol_atoms = nullptr, *mol_parent = nullptr;
  double* mol_u = nullptr;
};

}  // namespace

// private per-context bookkeeping kept out of the public struct layout
struct tmd_ctx_full : tmd_ctx {
  CtxPriv priv;
};
static inline CtxPriv& priv(tmd_ctx* c) { return static_cast<tmd_ctx_full*>(c)->priv; }
// An fp32 entry point on an fp64 context (or the reverse) is a call-order error.
static int need_precision(tmd_ctx* ctx, int bits, const char* name) {
  if (ctx->precision == bits) return TMD_OK;
  return fail(TMD_ERR_STATE, std::string(name) + ": this context runs in " + (ctx->precision == 64 ? "fp64" : "fp32") +
                                 " (tmd_set_precision); use the " + (ctx->precision == 64 ? "_f64" : "fp32") + " entry point");
}
#define TMD_PRECISION(ctx, bits, name) \
  if (int rc__ = need_precision((ctx), (bits), (name))) return rc__;

// ---- particle-mesh Ewald: parameter choice (the one place it is made) ------------------------
static inline bool pme_on(tmd_ctx* ctx) { return priv(ctx).pme_tol > 0.0; }
// MODE of the full-row pair kernels (physics.cuh, pair_terms): a PME context never runs another
static int pair_mode_of(tmd_ctx* ctx) {
  if (pme_on(ctx)) return 2;
  return (ctx->pair_mask == (T_LJ | T_ELEC) && ctx->d.pp.has_switch && ctx->d.pp.rfa && !ctx->exact_gradient) ? 1 : 0;
}
static int smallest_235(int n) {
  for (int m = std::max(n, 1);; ++m) {
    int k = m;
    for (int p : {2, 3, 5})
      while (k % p == 0) k /= p;
    if (k == 1) return m;
  }
}
// alpha = sqrt(-ln 2 tol) / rc; n_d = smallest 2^a 3^b 5^c >= max(2 alpha L_d / (3 tol^(1/5)), 10), the largest over
// the replicas (OpenMM's choice).  The real-space sum is a minimum-image sum, so every box must be at least two
// cutoffs long on every axis; the line kernels hold at most PME_MAX_N points.
static int pme_choose(tmd_ctx* ctx, double tol, const double* box, double* alpha, int K[3]) {
  if (ctx->cutoff < 0) return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald needs a cutoff");
  const double rc = ctx->cutoff;
  *alpha = sqrt(-log(2.0 * tol)) / rc;
  for (int d = 0; d < 3; ++d) {
    double lmax = 0.0;
    for (int r = 0; r < ctx->nrep; ++r) {
      const double L = box[3 * r + d];
      if (!(L > 0.0)) return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald needs a periodic box on every replica");
      if (rc > 0.5 * L)
        return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald needs cutoff <= half of every box length (the real-space "
                                         "sum takes the minimum image only)");
      lmax = std::max(lmax, L);
    }
    const double want = std::max(2.0 * *alpha * lmax / (3.0 * pow(tol, 0.2)), 10.0);
    K[d] = smallest_235((int)std::min(ceil(want), 1e6));
    if (K[d] > PME_MAX_N)
      return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald grid of " + std::to_string(K[d]) + " points along an axis: the FFT "
                                       "kernels take at most " + std::to_string(PME_MAX_N) + " (a larger tolerance or smaller box)");
  }
  return TMD_OK;
}
// ---- peer-to-peer position exchange --------------------------------------------------------
static inline float* dd_pos_of(tmd_ctx* ctx, int peer, int which) {
  return reinterpret_cast<float*>(static_cast<char*>(ctx->dd_peer_base[peer]) + (size_t)which * ctx->dd_pos_bytes);
}
static inline unsigned* dd_flags_of(tmd_ctx* ctx, int peer) {
  return reinterpret_cast<unsigned*>(static_cast<char*>(ctx->dd_peer_base[peer]) + 2 * ctx->dd_pos_bytes);
}
static void dd_release(tmd_ctx* ctx) {
  for (int p = 0; p < ctx->dd_world; ++p)
    if (p != ctx->dd_rank && ctx->dd_peer_base[p]) cudaIpcCloseMemHandle(ctx->dd_peer_base[p]);
  if (ctx->dd_base) cudaFree(ctx->dd_base);
  ctx->dd_base = nullptr;
  for (void*& b : ctx->dd_peer_base) b = nullptr;
  ctx->dd_connected = false;
  ctx->dd_world = 0;
  ctx->dd_rank = -1;
}


extern "C" {

const char* tmd_last_error(void) { return g_err.c_str(); }
#if defined(TMD_SIMT_HOST)
int tmd_version(void) { return -100; }  // host SIMT interpreter build (tests/simt): torchmd_b200/_lib.py refuses it
#else
int tmd_version(void) { return 104; }  // 101: the "precision: double" entry points (tmd_set_precision, *_f64); 102: constraints; 103: PME; 104: box rescale + molecule scaling
#endif

int tmd_create(tmd_ctx** out, int device, int natoms, int nreplicas) {
  if (!out || natoms <= 0 || nreplicas <= 0) return fail(TMD_ERR_ARG, "tmd_create: bad arguments");
  if (nreplicas > 65535) return fail(TMD_ERR_ARG, "tmd_create: at most 65535 replicas");
  int ndev = 0;
  TMD_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(TMD_ERR_ARG, "tmd_create: no such CUDA device");
  DeviceGuard guard(device);
  int nsm = 0;
  TMD_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
  tmd_ctx_full* c = new tmd_ctx_full();
  c->device = device;
  c->nsm = std::max(1, nsm);
  c->natoms = natoms;
  c->nrep = nreplicas;
  DeviceState& d = c->d;
  d.natoms = natoms;
  d.nrep = nreplicas;
  d.nsub = 2;
  const size_t RN = (size_t)natoms * nreplicas;
  int rc = TMD_OK;
  if ((rc = device_alloc(&d.xq_s, RN + nreplicas))) return rc;  // +1 sentinel record per replica
  if ((rc = device_alloc(&d.type_s, RN))) return rc;
  if ((rc = device_alloc(&d.xw_s, RN))) return rc;
  if ((rc = device_alloc(&d.perm, RN))) return rc;
  if ((rc = device_alloc(&d.inv, RN))) return rc;
  if ((rc = device_alloc(&d.pos_ref, RN))) return rc;
  if ((rc = device_alloc(&d.cell_of, RN))) return rc;
  if ((rc = device_alloc(&d.rank, RN))) return rc;
  if ((rc = device_alloc(&d.nnbr, RN))) return rc;
  if ((rc = device_alloc(&d.flags, (size_t)nreplicas * F_COUNT))) return rc;
  if ((rc = device_alloc(&d.grid, (size_t)nreplicas))) return rc;
  if ((rc = device_alloc(&d.bounds, (size_t)nreplicas * 6))) return rc;
  if ((rc = device_alloc(&d.counters, (size_t)4))) return rc;
  TMD_CUDA(cudaMemset(d.counters, 0, 4 * sizeof(unsigned long long)));
  d.own_lo = 0;
  d.own_n = natoms;
  d.own_all = 1;
  if ((rc = device_alloc(&c->ke_scratch, (size_t)nreplicas))) return rc;
  if ((rc = device_alloc(&c->e_scratch, (size_t)nreplicas * TMD_NUM_ENERGIES))) return rc;
  TMD_CUDA(cudaMemset(d.xq_s, 0xFF, (RN + nreplicas) * sizeof(float4)));  // NaN everywhere, incl. the sentinels
  TMD_CUDA(cudaMemset(d.type_s, 0, RN * sizeof(int)));
  TMD_CUDA(cudaMemset(d.nnbr, 0, RN * sizeof(int)));
  *out = c;
  return TMD_OK;
}

int tmd_destroy(tmd_ctx* ctx) {
  if (!ctx) return TMD_OK;
  DeviceGuard guard(ctx->device);
  DeviceState& d = ctx->d;
  void* bufs[] = {d.xq_s, d.xw_s, d.type_s, d.perm, d.inv, d.pos_ref, d.cell_of, d.rank, d.nnbr, d.flags,
                  d.grid, d.bounds, d.counters, d.cell_count, d.cell_start, d.nbr, ctx->q, ctx->type,
                  ctx->excl_ptr, ctx->excl_idx, ctx->AB, ctx->ke_scratch, ctx->e_scratch,
                  ctx->bonds.idx, ctx->bonds.prm, ctx->angles.idx, ctx->angles.prm,
                  ctx->torsions[0].idx, ctx->torsions[0].term_ptr, ctx->torsions[0].terms,
                  ctx->torsions[1].idx, ctx->torsions[1].term_ptr, ctx->torsions[1].terms,
                  ctx->pairs14.idx, ctx->pairs14.prm, ctx->bonded_atom_ptr, ctx->bonded_entries, ctx->xf_buf,
                  ctx->xq64, ctx->shadow, ctx->q64, ctx->AB64, ctx->L64,
                  ctx->bonds64.idx, ctx->bonds64.prm, ctx->angles64.idx, ctx->angles64.prm,
                  ctx->torsions64[0].idx, ctx->torsions64[0].term_ptr, ctx->torsions64[0].terms,
                  ctx->torsions64[1].idx, ctx->torsions64[1].term_ptr, ctx->torsions64[1].terms,
                  ctx->pairs1464.idx, ctx->pairs1464.prm};
  for (void* b : bufs)
    if (b) cudaFree(b);
  dd_release(ctx);
  for (void* b : priv(ctx).cl_bufs) cudaFree(b);
  if (priv(ctx).term_forces) cudaFree(priv(ctx).term_forces);
  for (cudaEvent_t e : priv(ctx).ev) cudaEventDestroy(e);
  for (int k = 0; k < CtxPriv::NGRAPH; ++k) {
    if (priv(ctx).exec[k]) cudaGraphExecDestroy(priv(ctx).exec[k]);
    if (priv(ctx).graph[k]) cudaGraphDestroy(priv(ctx).graph[k]);
  }
  if (priv(ctx).helper) cudaStreamDestroy(priv(ctx).helper);
  if (priv(ctx).gstream) cudaStreamDestroy(priv(ctx).gstream);
  if (priv(ctx).ev_in) cudaEventDestroy(priv(ctx).ev_in);
  if (priv(ctx).ev_out) cudaEventDestroy(priv(ctx).ev_out);
  if (priv(ctx).side) cudaStreamDestroy(priv(ctx).side);
  if (priv(ctx).ev_fork) cudaEventDestroy(priv(ctx).ev_fork);
  if (priv(ctx).ev_join) cudaEventDestroy(priv(ctx).ev_join);
  if (priv(ctx).bonded_scratch) cudaFree(priv(ctx).bonded_scratch);
  for (void* b : {(void*)priv(ctx).con_groups, (void*)priv(ctx).con_free, (void*)priv(ctx).con_L, priv(ctx).con_ref, (void*)priv(ctx).con_fail})
    if (b) cudaFree(b);
  {
    CtxPriv& p = priv(ctx);
    for (void* b : {(void*)p.pme_q, (void*)p.pme_L, (void*)p.pme_tw, (void*)p.pme_econst, (void*)p.pme_qgrid, p.pme_cgrid, p.pme_infl,
                    (void*)p.pme_mod, (void*)p.box_dev, (void*)p.mol_ptr, (void*)p.mol_atoms, (void*)p.mol_parent, (void*)p.mol_u})
      if (b) cudaFree(b);
    if (p.pme_side) cudaStreamDestroy(p.pme_side);
    if (p.pme_fork) cudaEventDestroy(p.pme_fork);
    if (p.pme_join) cudaEventDestroy(p.pme_join);
    if (p.rs_done) cudaEventDestroy(p.rs_done);
    stage_free(p.rs_stage);
  }
  delete static_cast<tmd_ctx_full*>(ctx);
  return TMD_OK;
}

int tmd_set_atoms(tmd_ctx* ctx, const float* charges, const int32_t* types, int ntypes,
                  const float* A, const float* B) {
  if (!ctx || !charges || !types || ntypes <= 0) return fail(TMD_ERR_ARG, "tmd_set_atoms: bad arguments");
  TMD_PRECISION(ctx, 32, "tmd_set_atoms")
  DeviceGuard guard(ctx->device);
  for (int i = 0; i < ctx->natoms; ++i)
    if (types[i] < 0 || types[i] >= ntypes) return fail(TMD_ERR_ARG, "tmd_set_atoms: atom type out of range");
  ctx->charges_host.assign(charges, charges + ctx->natoms);
  int rc;
  if ((rc = upload(&ctx->type, types, (size_t)ctx->natoms))) return rc;
  std::vector<float2> ab((size_t)ntypes * ntypes, make_float2(0.f, 0.f));
  if (A && B)
    for (size_t t = 0; t < ab.size(); ++t) ab[t] = make_float2(A[t], B[t]);
  if ((rc = upload(&ctx->AB, ab.data(), ab.size()))) return rc;
  ctx->d.ntypes = ntypes;
  ctx->have_atoms = true;
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}

int tmd_set_exclusions(tmd_ctx* ctx, const int64_t* row_ptr, const int32_t* cols) {
  if (!ctx || !row_ptr) return fail(TMD_ERR_ARG, "tmd_set_exclusions: bad arguments");
  DeviceGuard guard(ctx->device);
  const int n = ctx->natoms;
  if (row_ptr[n] >= (1ll << 31)) return fail(TMD_ERR_ARG, "tmd_set_exclusions: too many entries");
  std::vector<int> rp(n + 1);
  for (int i = 0; i <= n; ++i) rp[i] = (int)row_ptr[i];
  for (int64_t e = 0; e < row_ptr[n]; ++e)
    if (cols[e] < 0 || cols[e] >= n) return fail(TMD_ERR_ARG, "tmd_set_exclusions: index out of range");
  int rc;
  if ((rc = upload(&ctx->excl_ptr, rp.data(), rp.size()))) return rc;
  if ((rc = upload(&ctx->excl_idx, cols, (size_t)row_ptr[n]))) return rc;
  ctx->have_excl = row_ptr[n] > 0;
  {  // particle-mesh Ewald reads the rows as the set of excluded pairs (pme_finalize refuses anything else)
    std::vector<std::pair<int, int>> e;
    e.reserve((size_t)row_ptr[n]);
    for (int i = 0; i < n; ++i)
      for (int64_t k = row_ptr[i]; k < row_ptr[i + 1]; ++k) e.emplace_back(i, cols[k]);
    std::sort(e.begin(), e.end());
    bool ok = std::adjacent_find(e.begin(), e.end()) == e.end();
    for (size_t k = 0; ok && k < e.size(); ++k)
      ok = e[k].first != e[k].second && std::binary_search(e.begin(), e.end(), std::make_pair(e[k].second, e[k].first));
    ctx->excl_is_set = ok;
  }
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}

int tmd_set_nonbonded(tmd_ctx* ctx, uint32_t term_mask, double cutoff, double switch_dist, int rfa,
                      double solvent_dielectric, double coulomb_constant, double skin) {
  if (!ctx) return fail(TMD_ERR_ARG, "tmd_set_nonbonded: null context");
  if (rfa && cutoff < 0) return fail(TMD_ERR_ARG, "tmd_set_nonbonded: reaction field needs a cutoff");
  if (skin < 0) return fail(TMD_ERR_ARG, "tmd_set_nonbonded: negative skin");
  if (switch_dist >= 0 && cutoff >= 0 && switch_dist >= cutoff)
    return fail(TMD_ERR_ARG, "tmd_set_nonbonded: switch_dist must be below cutoff");
  const uint32_t pair_bits = T_ELEC | T_LJ | T_REP | T_REPCG;
  ctx->pair_mask = term_mask & pair_bits;
  ctx->bonded_mask = term_mask & ~pair_bits;
  ctx->cutoff = cutoff;
  ctx->switch_dist = switch_dist;
  ctx->rfa = rfa;
  ctx->coulomb = coulomb_constant;
  ctx->skin = cutoff >= 0 ? skin : 0.0;
  PairParams& pp = ctx->d.pp;
  memset(&pp, 0, sizeof(pp));
  pp.terms = ctx->pair_mask;
  pp.has_cutoff = cutoff >= 0;
  pp.cutoff = pp.has_cutoff ? (float)cutoff : INFINITY;
  pp.s_max = pp.has_cutoff ? squared_threshold(pp.cutoff) : INFINITY;
  // the reference switches only when both are given (forces.py:403)
  pp.has_switch = (switch_dist >= 0 && cutoff >= 0);
  pp.switch_dist = pp.has_switch ? (float)switch_dist : 0.f;
  pp.inv_sw_width = pp.has_switch ? (float)(1.0 / (cutoff - switch_dist)) : 0.f;
  pp.rfa = rfa ? 1 : 0;
  if (rfa) {  // forces.py:466-468
    const double denom = 2.0 * solvent_dielectric + 1.0;
    const double krf = (1.0 / (cutoff * cutoff * cutoff)) * (solvent_dielectric - 1.0) / denom;
    const double crf = (1.0 / cutoff) * (3.0 * solvent_dielectric) / denom;
    pp.krf = (float)krf;
    pp.crf = (float)crf;
    pp.two_krf = (float)(2.0 * krf);
  }
  {  // the same set-up for the fp64 kernels (contexts of tmd_set_precision(ctx, 64))
    PairParams64& p = ctx->d64.pp;
    memset(&p, 0, sizeof(p));
    p.terms = ctx->pair_mask;
    p.has_cutoff = cutoff >= 0;
    p.cutoff = p.has_cutoff ? cutoff : INFINITY;
    p.s_max = p.has_cutoff ? squared_threshold64(cutoff) : INFINITY;
    p.has_switch = pp.has_switch;
    p.switch_dist = p.has_switch ? switch_dist : 0.0;
    p.inv_sw_width = p.has_switch ? 1.0 / (cutoff - switch_dist) : 1.0;
    p.rfa = pp.rfa;
    if (rfa) {
      const double denom = 2.0 * solvent_dielectric + 1.0;
      p.krf = (1.0 / (cutoff * cutoff * cutoff)) * (solvent_dielectric - 1.0) / denom;
      p.crf = (1.0 / cutoff) * (3.0 * solvent_dielectric) / denom;
    }
    p.true_gradient = ctx->exact_gradient;
  }
  ctx->have_nonbonded = true;
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}

extern "C++" {  // (templates inside the C-linkage block)
template <typename P>
static int set_bonded(tmd_ctx* ctx, BondedSetT<P>& s, std::vector<int32_t>& idx_h, int n, int k, int p,
                      const int32_t* idx, const P* prm) {
  DeviceGuard guard(ctx->device);
  if (n < 0 || (n > 0 && (!idx || !prm))) return fail(TMD_ERR_ARG, "bonded set: bad arguments");
  for (long long e = 0; e < (long long)n * k; ++e)
    if (idx[e] < 0 || idx[e] >= ctx->natoms) return fail(TMD_ERR_ARG, "bonded set: atom index out of range");
  int rc;
  if ((rc = upload(&s.idx, idx, (size_t)n * k))) return rc;
  if ((rc = upload(&s.prm, prm, (size_t)n * p))) return rc;
  s.n = n;
  idx_h.assign(idx, idx + (size_t)n * k);
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}
}  // extern "C++"

int tmd_set_bonds(tmd_ctx* ctx, int n, const int32_t* idx, const float* prm) {
  if (!ctx) return fail(TMD_ERR_ARG, "null context");
  TMD_PRECISION(ctx, 32, "tmd_set_bonds")
  return set_bonded(ctx, ctx->bonds, ctx->bonds_idx_h, n, 2, 2, idx, prm);
}
int tmd_set_angles(tmd_ctx* ctx, int n, const int32_t* idx, const float* prm) {
  if (!ctx) return fail(TMD_ERR_ARG, "null context");
  TMD_PRECISION(ctx, 32, "tmd_set_angles")
  return set_bonded(ctx, ctx->angles, ctx->angles_idx_h, n, 3, 2, idx, prm);
}
int tmd_set_pairs14(tmd_ctx* ctx, int n, const int32_t* idx, const float* prm) {
  if (!ctx) return fail(TMD_ERR_ARG, "null context");
  TMD_PRECISION(ctx, 32, "tmd_set_pairs14")
  return set_bonded(ctx, ctx->pairs14, ctx->pairs14_idx_h, n, 2, 4, idx, prm);
}
extern "C++" {  // (templates inside the C-linkage block)
template <typename P>
static int set_torsions(tmd_ctx* ctx, BondedSetT<P>& s, int which, int n, const int32_t* idx, const int32_t* term_ptr,
                        const P* terms, int amber_form) {
  DeviceGuard guard(ctx->device);
  if (n < 0 || (n > 0 && (!idx || !term_ptr || !terms))) return fail(TMD_ERR_ARG, "tmd_set_torsions: bad arguments");
  for (long long e = 0; e < (long long)n * 4; ++e)
    if (idx[e] < 0 || idx[e] >= ctx->natoms) return fail(TMD_ERR_ARG, "tmd_set_torsions: atom index out of range");
  int rc;
  if ((rc = upload(&s.idx, idx, (size_t)n * 4))) return rc;
  if ((rc = upload(&s.term_ptr, term_ptr, (size_t)(n ? n + 1 : 0)))) return rc;
  if ((rc = upload(&s.terms, terms, (size_t)(n ? term_ptr[n] : 0) * 3))) return rc;
  s.n = n;
  s.amber = amber_form ? 1 : 0;
  ctx->torsions_idx_h[which].assign(idx, idx + (size_t)n * 4);
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}
}  // extern "C++"
int tmd_set_torsions(tmd_ctx* ctx, int which, int n, const int32_t* idx, const int32_t* term_ptr,
                     const float* terms, int amber_form) {
  if (!ctx || which < 0 || which > 1) return fail(TMD_ERR_ARG, "tmd_set_torsions: bad arguments");
  TMD_PRECISION(ctx, 32, "tmd_set_torsions")
  return set_torsions(ctx, ctx->torsions[which], which, n, idx, term_ptr, terms, amber_form);
}

// ---- "precision: double" --------------------------------------------------------------------
int tmd_set_precision(tmd_ctx* ctx, int bits) {
  if (!ctx || (bits != 32 && bits != 64)) return fail(TMD_ERR_ARG, "tmd_set_precision: 32 or 64");
  if (ctx->touched || ctx->force_calls || ctx->launches)
    return fail(TMD_ERR_STATE, "tmd_set_precision: call it right after tmd_create, before any setter");
  ctx->precision = bits;
  return TMD_OK;
}

int tmd_set_atoms_f64(tmd_ctx* ctx, const double* charges, const int32_t* types, int ntypes, const double* A,
                      const double* B) {
  if (!ctx || !charges || !types || ntypes <= 0) return fail(TMD_ERR_ARG, "tmd_set_atoms_f64: bad arguments");
  TMD_PRECISION(ctx, 64, "tmd_set_atoms_f64")
  DeviceGuard guard(ctx->device);
  for (int i = 0; i < ctx->natoms; ++i)
    if (types[i] < 0 || types[i] >= ntypes) return fail(TMD_ERR_ARG, "tmd_set_atoms_f64: atom type out of range");
  ctx->charges64_host.assign(charges, charges + ctx->natoms);
  ctx->charges_host.assign(charges, charges + ctx->natoms);  // (the fp32 records of the list build)
  int rc;
  if ((rc = upload(&ctx->type, types, (size_t)ctx->natoms))) return rc;
  std::vector<float2> ab((size_t)ntypes * ntypes, make_float2(0.f, 0.f));
  std::vector<double> ab64(2 * ab.size(), 0.0);
  if (A && B)
    for (size_t t = 0; t < ab.size(); ++t) {
      ab64[2 * t] = A[t];
      ab64[2 * t + 1] = B[t];
    }
  if ((rc = upload(&ctx->AB, ab.data(), ab.size()))) return rc;
  if ((rc = upload(&ctx->AB64, ab64.data(), ab64.size()))) return rc;
  ctx->d.ntypes = ntypes;
  ctx->have_atoms = true;
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}
int tmd_set_bonds_f64(tmd_ctx* ctx, int n, const int32_t* idx, const double* prm) {
  if (!ctx) return fail(TMD_ERR_ARG, "null context");
  TMD_PRECISION(ctx, 64, "tmd_set_bonds_f64")
  return set_bonded(ctx, ctx->bonds64, ctx->bonds_idx_h, n, 2, 2, idx, prm);
}
int tmd_set_angles_f64(tmd_ctx* ctx, int n, const int32_t* idx, const double* prm) {
  if (!ctx) return fail(TMD_ERR_ARG, "null context");
  TMD_PRECISION(ctx, 64, "tmd_set_angles_f64")
  return set_bonded(ctx, ctx->angles64, ctx->angles_idx_h, n, 3, 2, idx, prm);
}
int tmd_set_pairs14_f64(tmd_ctx* ctx, int n, const int32_t* idx, const double* prm) {
  if (!ctx) return fail(TMD_ERR_ARG, "null context");
  TMD_PRECISION(ctx, 64, "tmd_set_pairs14_f64")
  return set_bonded(ctx, ctx->pairs1464, ctx->pairs14_idx_h, n, 2, 4, idx, prm);
}
int tmd_set_torsions_f64(tmd_ctx* ctx, int which, int n, const int32_t* idx, const int32_t* term_ptr,
                         const double* terms, int amber_form) {
  if (!ctx || which < 0 || which > 1) return fail(TMD_ERR_ARG, "tmd_set_torsions_f64: bad arguments");
  TMD_PRECISION(ctx, 64, "tmd_set_torsions_f64")
  return set_torsions(ctx, ctx->torsions64[which], which, n, idx, term_ptr, terms, amber_form);
}

extern "C++" {  // (templates inside the C-linkage block)
template <typename T>
static int set_box(tmd_ctx* ctx, const T* box_diag) {
  int nzero = 0;
  for (int e = 0; e < ctx->nrep * 3; ++e) {
    if (!(box_diag[e] >= T(0))) return fail(TMD_ERR_ARG, "tmd_set_box: negative or NaN box length");
    nzero += (box_diag[e] == T(0));
  }
  if (nzero != 0 && nzero != ctx->nrep * 3)
    return fail(TMD_ERR_UNSUPPORTED, "tmd_set_box: box must be all zero (no wrapping) or all positive");
  if (pme_on(ctx)) {  // alpha and the grid follow the box
    std::vector<double> b(box_diag, box_diag + ctx->nrep * 3);
    double alpha;
    int K[3];
    if (int rc = pme_choose(ctx, priv(ctx).pme_tol, b.data(), &alpha, K)) return fail(rc, "tmd_set_box: " + g_err);
    priv(ctx).pme_alpha = alpha;
    for (int d = 0; d < 3; ++d) priv(ctx).pme_K[d] = K[d];
  }
  priv(ctx).pme_pinned = false;
  ctx->periodic = (nzero == 0);
  ctx->box_host.assign(box_diag, box_diag + ctx->nrep * 3);
  ctx->box64_host.assign(box_diag, box_diag + ctx->nrep * 3);
  if (priv(ctx).con_L) TMD_CUDA(cudaMemcpy(priv(ctx).con_L, ctx->box64_host.data(), ctx->nrep * 3 * sizeof(double), cudaMemcpyHostToDevice));
  if (priv(ctx).box_dev) TMD_CUDA(cudaMemcpy(priv(ctx).box_dev, ctx->box64_host.data(), ctx->nrep * 3 * sizeof(double), cudaMemcpyHostToDevice));
  ctx->have_box = true;
  ctx->touched = true;
  priv(ctx).dirty = true;
  return TMD_OK;
}
}  // extern "C++"
int tmd_set_box(tmd_ctx* ctx, const float* box_diag) {
  if (!ctx || !box_diag) return fail(TMD_ERR_ARG, "tmd_set_box: bad arguments");
  TMD_PRECISION(ctx, 32, "tmd_set_box")
  return set_box(ctx, box_diag);
}
int tmd_set_box_f64(tmd_ctx* ctx, const double* box_diag) {
  if (!ctx || !box_diag) return fail(TMD_ERR_ARG, "tmd_set_box_f64: bad arguments");
  TMD_PRECISION(ctx, 64, "tmd_set_box_f64")
  return set_box(ctx, box_diag);
}

// ---- particle-mesh Ewald ----------------------------------------------------------------------
int tmd_set_pme(tmd_ctx* ctx, double tolerance) {
  if (!ctx) return fail(TMD_ERR_ARG, "tmd_set_pme: null context");
  CtxPriv& pv = priv(ctx);
  if (!(tolerance > 0.0)) {
    if (pme_on(ctx)) {
      pv.pme_tol = 0.0;
      if (!ctx->rfa) {  // (the reaction-field words held the Ewald constants)
        ctx->d.pp.krf = ctx->d.pp.crf = 0.f;
        ctx->d64.pp.krf = ctx->d64.pp.crf = 0.0;
      }
      pv.dirty = true;
    }
    return TMD_OK;
  }
  if (!(tolerance < 0.5)) return fail(TMD_ERR_ARG, "tmd_set_pme: the tolerance must be below 0.5");
  if (ctx->dd_base || !ctx->d.own_all)
    return fail(TMD_ERR_UNSUPPORTED, "tmd_set_pme: decomposed runs cannot use particle-mesh Ewald");
  if (!ctx->have_nonbonded) return fail(TMD_ERR_STATE, "tmd_set_pme: call tmd_set_nonbonded first");
  if (ctx->cutoff < 0) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_pme: particle-mesh Ewald needs a cutoff");
  if (ctx->rfa) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_pme: particle-mesh Ewald and the reaction field exclude each other");
  if (!(ctx->pair_mask & T_ELEC)) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_pme: particle-mesh Ewald needs the electrostatics term");
  if (ctx->have_box) {
    double alpha;
    int K[3];
    if (!ctx->periodic) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_pme: particle-mesh Ewald needs a periodic box on every replica");
    if (int rc = pme_choose(ctx, tolerance, ctx->box64_host.data(), &alpha, K)) return fail(rc, "tmd_set_pme: " + g_err);
    pv.pme_alpha = alpha;
    for (int d = 0; d < 3; ++d) pv.pme_K[d] = K[d];
  }
  pv.pme_tol = tolerance;
  pv.pme_pinned = false;
  ctx->touched = true;
  pv.dirty = true;
  return TMD_OK;
}

int tmd_get_pme(tmd_ctx* ctx, double* alpha, int32_t grid[3]) {
  if (!ctx || !alpha || !grid) return fail(TMD_ERR_ARG, "tmd_get_pme: bad arguments");
  if (!pme_on(ctx)) return fail(TMD_ERR_STATE, "tmd_get_pme: particle-mesh Ewald is off (tmd_set_pme)");
  if (!ctx->have_box) return fail(TMD_ERR_STATE, "tmd_get_pme: the grid follows the box: call tmd_set_box first");
  *alpha = priv(ctx).pme_alpha;
  for (int d = 0; d < 3; ++d) grid[d] = priv(ctx).pme_K[d];
  return TMD_OK;
}

}  // extern "C"

// ---- finalise: host-side sizing, allocation, uploads (first use / after changes) ----------
static constexpr double F64_POS_LIMIT = 8192.0;  // A: fp64 contexts flag coordinates from here on (margin, finalize)

// Particle-mesh Ewald tables of the context's boxes: the pair kernels' Ewald constants, twiddles, the influence function
// G(m) with the B-spline moduli, the self + background energies, and the grids.
static double pme_econst(double alpha, double q2, double qsum, const double* L) {
  const double V = L[0] * L[1] * L[2];
  return -alpha / sqrt(M_PI) * q2 - M_PI * qsum * qsum / (2.0 * V * alpha * alpha);
}
template <typename T>
static void launch_pme_influence(tmd_ctx* ctx, cudaStream_t st) {
  const CtxPriv& pv = priv(ctx);
  const long long blocks = std::min<long long>((pv.pme.ktot + PME_THREADS - 1) / PME_THREADS, 4 * (long long)ctx->nsm);
  launch(k_pme_influence<T>, dim3((unsigned)std::max<long long>(blocks, 1), ctx->nrep), PME_THREADS, st, pv.pme, (const double*)pv.pme_mod);
}

// A rescaled box (tmd_rescale_box) keeps alpha and the grid the context had (pme_pinned): a re-finalisation on the
// way (grown lists) keeps them too.  Otherwise both are chosen from the boxes held.
static int pme_finalize(tmd_ctx* ctx, cudaStream_t stream) {
  CtxPriv& pv = priv(ctx);
  if (!ctx->periodic) return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald needs a periodic box on every replica");
  if (ctx->rfa) return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald and the reaction field exclude each other");
  if (!(ctx->pair_mask & T_ELEC)) return fail(TMD_ERR_UNSUPPORTED, "particle-mesh Ewald needs the electrostatics term");
  if (!ctx->excl_is_set)
    return fail(TMD_ERR_ARG, "particle-mesh Ewald: tmd_set_exclusions must list every excluded pair in both rows, once, "
                             "and no atom with itself (the exclusion correction sums each row)");
  double alpha;
  int K[3];
  if (pv.pme_pinned) {
    alpha = pv.pme_alpha;
    for (int d = 0; d < 3; ++d) K[d] = pv.pme_K[d];
  } else if (int rc = pme_choose(ctx, pv.pme_tol, ctx->box64_host.data(), &alpha, K)) {
    return rc;
  }
  pv.pme_alpha = alpha;
  for (int d = 0; d < 3; ++d) pv.pme_K[d] = K[d];
  const double beta = 2.0 * alpha / sqrt(M_PI);
  ctx->d.pp.ew_alpha = (float)alpha;
  ctx->d.pp.ew_beta = (float)beta;
  ctx->d64.pp.ew_alpha = alpha;
  ctx->d64.pp.ew_beta = beta;
  const int N = ctx->natoms, R = ctx->nrep;
  const bool f64 = ctx->precision == 64;
  const size_t ktot = (size_t)K[0] * K[1] * K[2];
  int rc;
  // charges carry sqrt(coulomb constant), as in the pair kernels
  std::vector<double> q(N);
  const double sk = sqrt(ctx->coulomb > 0 ? ctx->coulomb : 0.0);
  double qabs = 0.0, qsum = 0.0, q2 = 0.0;
  for (int i = 0; i < N; ++i) {
    q[i] = (f64 ? ctx->charges64_host[i] : (double)ctx->charges_host[i]) * sk;
    qabs += fabs(q[i]);
    qsum += q[i];
    q2 += q[i] * q[i];
  }
  // Fixed point of the charge grid: a point receives q th_x th_y th_z from at most every atom, and the weights of one
  // atom sum to 1, so |value| <= sum |q| over the whole grid.  scale = 2^e with e the largest integer such that
  // scale * sum|q| <= 2^61; each contribution rounds by at most 1/2 unit, 125 per atom, so the integer sum stays below
  // 2^61 + 63 N < 2^63 for any N < 2^55.  Resolution 2^-e, e.g. 2^-40 e for 10^5 TIP3P atoms.
  const double e = qabs > 0.0 ? floor(61.0 - log2(qabs)) : 40.0;
  const double scale = ldexp(1.0, (int)std::min(e, 1000.0));
  std::vector<double> tw(2 * (size_t)(K[0] + K[1] + K[2]));
  {
    size_t o = 0;
    for (int d = 0; d < 3; ++d)
      for (int t = 0; t < K[d]; ++t, ++o) {
        tw[2 * o] = cos(2.0 * M_PI * t / K[d]);
        tw[2 * o + 1] = -sin(2.0 * M_PI * t / K[d]);
      }
  }
  // |b(m)|^2 of order-5 B-splines (zeros at m = K/2 take their neighbours' mean, as OpenMM does)
  double th[PME_ORDER], dth[PME_ORDER];
  pme_bspline(0.0, th, dth);
  std::vector<double> mod[3];
  for (int d = 0; d < 3; ++d) {
    mod[d].resize(K[d]);
    for (int m = 0; m < K[d]; ++m) {
      double re = 0.0, im = 0.0;
      for (int k = 0; k < PME_ORDER; ++k) {
        re += th[k] * cos(2.0 * M_PI * m * k / K[d]);
        im += th[k] * sin(2.0 * M_PI * m * k / K[d]);
      }
      mod[d][m] = re * re + im * im;
    }
    for (int m = 0; m < K[d]; ++m)
      if (mod[d][m] < 1e-7) mod[d][m] = 0.5 * (mod[d][(m + K[d] - 1) % K[d]] + mod[d][(m + 1) % K[d]]);
  }
  std::vector<double> econst(R), mods;
  for (int r = 0; r < R; ++r) econst[r] = pme_econst(alpha, q2, qsum, &ctx->box64_host[3 * r]);
  for (int d = 0; d < 3; ++d) mods.insert(mods.end(), mod[d].begin(), mod[d].end());
  pv.pme_q2 = q2;
  pv.pme_qsum = qsum;
  for (void* b : {(void*)pv.pme_qgrid, pv.pme_cgrid, pv.pme_infl})
    if (b) cudaFree(b);
  pv.pme_qgrid = nullptr;
  pv.pme_cgrid = nullptr;
  pv.pme_infl = nullptr;
  if ((rc = upload(&pv.pme_q, q.data(), q.size()))) return rc;
  if ((rc = upload(&pv.pme_L, ctx->box64_host.data(), ctx->box64_host.size()))) return rc;
  if ((rc = upload(&pv.pme_tw, tw.data(), tw.size()))) return rc;
  if ((rc = upload(&pv.pme_econst, econst.data(), econst.size()))) return rc;
  if ((rc = upload(&pv.pme_mod, mods.data(), mods.size()))) return rc;
  if ((rc = device_alloc(&pv.pme_qgrid, (size_t)R * ktot))) return rc;
  TMD_CUDA(cudaMemset(pv.pme_qgrid, 0, (size_t)R * ktot * sizeof(unsigned long long)));
  if (f64) {
    if ((rc = device_alloc(reinterpret_cast<double**>(&pv.pme_infl), (size_t)R * ktot))) return rc;
    if ((rc = device_alloc(reinterpret_cast<Cplx<double>**>(&pv.pme_cgrid), (size_t)R * ktot))) return rc;
  } else {
    if ((rc = device_alloc(reinterpret_cast<float**>(&pv.pme_infl), (size_t)R * ktot))) return rc;
    if ((rc = device_alloc(reinterpret_cast<Cplx<float>**>(&pv.pme_cgrid), (size_t)R * ktot))) return rc;
    if (!pv.pme_side) {
      TMD_CUDA(cudaStreamCreateWithFlags(&pv.pme_side, cudaStreamNonBlocking));
      TMD_CUDA(cudaEventCreateWithFlags(&pv.pme_fork, cudaEventDisableTiming));
      TMD_CUDA(cudaEventCreateWithFlags(&pv.pme_join, cudaEventDisableTiming));
    }
  }
  PmeArgs& a = pv.pme;
  a.natoms = N;
  for (int d = 0; d < 3; ++d) a.K[d] = K[d];
  a.ktot = (long long)ktot;
  a.scale = scale;
  a.inv_scale = 1.0 / scale;
  a.q = pv.pme_q;
  a.L = pv.pme_L;
  a.qgrid = pv.pme_qgrid;
  a.cgrid = pv.pme_cgrid;
  a.tw = pv.pme_tw;
  a.infl = pv.pme_infl;
  a.econst = pv.pme_econst;
  a.excl_ptr = ctx->have_excl ? ctx->excl_ptr : nullptr;
  a.excl_idx = ctx->have_excl ? ctx->excl_idx : nullptr;
  a.alpha = alpha;
  a.beta = beta;
  const ClusterState& cl = ctx->d.cl;
  a.cl_f = cl.on ? cl.f : nullptr;
  a.cl_inv = cl.on ? cl.inv : nullptr;
  a.cl_stride = (long long)cl.slots + 1;
  if (f64) launch_pme_influence<double>(ctx, stream);
  else launch_pme_influence<float>(ctx, stream);
  TMD_CUDA(cudaGetLastError());  // (set-up work: not counted with the force calls' launches)
  return TMD_OK;
}

// Cell grid of one replica's box L (list radius rl, ctx->d.nsub cells per radius), and the fixed-point units of the
// pair kernels when priv(ctx).grid_fx.  keep: the cell counts the replica's grid had, which a rescale keeps while the
// cells stay at least rl / nsub wide (a growing box only widens them) and otherwise lowers to floor(L nsub / rl) --
// never above the counts the cell arrays were sized for.  null: chosen from the box.  Returns false when a kept grid
// would fall below 2 nsub + 1 cells along an axis.
static bool box_grid(tmd_ctx* ctx, Grid& g, const float* L3, double rl, double margin, const int* keep) {
  const int nsub = ctx->d.nsub;
  const bool cells = ctx->periodic && ctx->cutoff >= 0;
  bool ok = true;
  memset(&g, 0, sizeof(g));
  g.periodic = ctx->periodic ? 1 : 0;
  g.ncells = 1;
  double lmax = 0.0;
  for (int k = 0; k < 3; ++k) {
    const float L = L3[k];
    g.L[k] = L;
    g.invL[k] = ctx->periodic ? 1.0f / L : 0.f;
    g.n[k] = 1;
    if (cells) {
      int n = std::min((int)floor((double)L * nsub / rl), 128);
      if (keep) {
        if (keep[k] > 1) {
          n = std::min(n, keep[k]);
          ok = ok && n >= 2 * nsub + 1;
        } else {
          n = 1;
        }
      }
      if (n >= 2 * nsub + 1) {
        g.n[k] = n;
        g.reach[k] = nsub;
        g.inv_w[k] = (float)(n / (double)L);
      }
    }
    g.ncells *= g.n[k];
    lmax = std::max(lmax, (double)L);
  }
  if (priv(ctx).grid_fx) {
    for (int k = 0; k < 3; ++k) {
      g.fx_unit[k] = (float)((double)g.L[k] / 4294967296.0);
      g.fx_inv[k] = 4294967296.0 / (double)g.L[k];
    }
    const double rmax = ctx->cutoff + 2.0 * ctx->skin + 2.0 * margin;  // no listed pair is further apart
    double c0, c1;
    fx_margin(rmax, lmax, &c0, &c1);
    g.fx_c0 = (float)(c0 * 1.0000002);  // never round the bound down
    g.fx_c1 = (float)(c1 * 1.0000002);
  }
  return ok;
}

// list radius margin (A) over cutoff + skin: see finalize
static double list_margin(const tmd_ctx* ctx) { return 0.004 + (ctx->precision == 64 ? 36.0 / 4096.0 : 0.0); }

static int finalize(tmd_ctx* ctx, cudaStream_t stream) {
  if (!ctx->have_atoms) return fail(TMD_ERR_STATE, "tmd_set_atoms has not been called");
  if (!ctx->have_box) return fail(TMD_ERR_STATE, "tmd_set_box has not been called");
  if (!ctx->have_nonbonded) return fail(TMD_ERR_STATE, "tmd_set_nonbonded has not been called");
  TMD_CUDA(cudaStreamSynchronize(stream));
  DeviceState& d = ctx->d;
  const int N = ctx->natoms, R = ctx->nrep;
  int rc;

  // charges carry sqrt(coulomb constant) so q_i*q_j is the full prefactor
  {
    std::vector<float> qs(N);
    const double sk = sqrt(ctx->coulomb > 0 ? ctx->coulomb : 0.0);
    for (int i = 0; i < N; ++i) qs[i] = (float)((double)ctx->charges_host[i] * sk);
    if ((rc = upload(&ctx->q, qs.data(), (size_t)N))) return rc;
  }
  d.q = ctx->q;
  d.type = ctx->type;
  d.AB = ctx->AB;
  d.excl_ptr = ctx->have_excl ? ctx->excl_ptr : nullptr;
  d.excl_idx = ctx->have_excl ? ctx->excl_idx : nullptr;

  const bool has_cut = ctx->cutoff >= 0;
  const bool f64 = ctx->precision == 64;
  // fp64 contexts build the list from an fp32 shadow of the positions (double.cuh), so the list radius also covers
  // what that shadow can be off by.  Conditions: every |coordinate| < P = F64_POS_LIMIT = 2^13 A (else k_prepare_f64
  // raises F_FARPOS, which tmd_get_stats reports) and every box length L <= 2^12 A (else refused below).  Below 2^13 an
  // fp32 ulp is at most 2^-11 A; h = 2^-12 A is half of it.  Per coordinate of one atom, against the exact fp64 geometry,
  // the build sees at most:
  //   the shadow's rounding                                                    h
  //   the fold x - L*floor(x/L) of phase_sort_pack, product and subtraction
  //   rounded separately (no contraction assumed): |L*floor(x/L)| < P + L
  //   <= 1.5 * 2^13, half an ulp 2h; the result is below 2L <= 2^13:           2h + h
  //   fp32 box length against the fp64 one, |floor(x/L)| * |L32 - L64|
  //   <= (P/L + 1) * L * 2^-24 = (P + L) * 2^-24 <= 1.5 * 2^-11:               3h
  // so 7h per atom, and per component of a pair 14h plus h for the one image shift the build adds with L32 (|L32 - L64|
  // <= h): 15h, sqrt(3) * 15h < 26h on a distance.  The displacement trigger compares shadows with shadows; an atom's
  // true displacement exceeds its shadow displacement by at most 2 sqrt(3) h, a pair's distance by 4 sqrt(3) h < 7h.
  // With the fp32 slack of the build arithmetic and binning (0.004 A) the radius needs 26h + 7h = 33h more; 36h =
  // 0.0088 A is added.
  const double margin = list_margin(ctx);  // A
  if (f64 && ctx->periodic)
    for (int e = 0; e < R * 3; ++e)
      if (ctx->box_host[e] > 4096.f)
        return fail(TMD_ERR_UNSUPPORTED, "fp64 contexts take box lengths up to 4096 A (the fp32 shadow of the list build)");
  const double rl = has_cut ? ctx->cutoff + ctx->skin + margin : INFINITY;
  d.rlist = (float)rl;
  d.rlist2 = has_cut ? (float)(rl * rl) : INFINITY;
  d.trigger2 = has_cut ? (float)(0.25 * ctx->skin * ctx->skin) : INFINITY;

  // Cluster half-list path (cluster.cuh): a cutoff, pair terms out of {lj, electrostatics}, explicit-force
  // convention, few atom types, the whole system on this context; in a periodic box additionally every pair a list
  // can hold must have ONE image within reach (size condition below).  Otherwise: full Verlet rows.
  ClusterState& cl = d.cl;
  const double cl_extent = 8.0;  // a periodic box must leave room for clusters at least this long (A)
  bool use_cluster = env_switch("TMD_B200_CLUSTER", TMD_DEFAULT_CLUSTER) == 1 && !f64 && !ctx->cluster_failed && has_cut &&
                     ctx->pair_mask != 0 && (ctx->pair_mask & ~(T_LJ | T_ELEC)) == 0 && !ctx->exact_gradient &&
                     d.ntypes <= CL_MAXT && N < (1 << 24) - 4096 * CL;
  double cl_max_extent = INFINITY;
  if (use_cluster && ctx->periodic) {
    // pair (i, j) of a list: |x_i - x_j| <= rl + (cluster extent) + skin along every axis, and that must stay below
    // half a box length (cluster.cuh)
    float lmin = INFINITY;
    for (int e = 0; e < R * 3; ++e) lmin = std::min(lmin, ctx->box_host[e]);
    // (the fixed-point separations wrap to the minimum image by themselves: a listed pair only has to stay below
    //  half a box length, rl + extent + skin < L / 2)
    cl_max_extent = 0.5 * (double)lmin - rl - ctx->skin - 0.05;
    use_cluster = cl_max_extent >= cl_extent;
  }
  {
    double cellw = 4.0;
    if (const char* e = getenv("TMD_B200_CELLW")) cellw = std::max(1.0, atof(e));
    d.nsub = use_cluster ? std::max(1, (int)floor(rl / cellw + 0.5)) : 2;
  }

  // guard-free minimum image is valid iff no listed pair can be further than 0.45 L apart
  ctx->safe_image = false;
  if (ctx->periodic && has_cut) {
    float lmin = INFINITY;
    for (int e = 0; e < R * 3; ++e) lmin = std::min(lmin, ctx->box_host[e]);
    ctx->safe_image = (ctx->cutoff + 2.0 * ctx->skin + 2.0 * margin) < 0.45 * (double)lmin;
  }
  d.check_far = ctx->safe_image ? 1 : 0;
  d.pp.true_gradient = ctx->exact_gradient;
  ctx->pair_mode = pair_mode_of(ctx);
  // Fixed-point separations in the pair kernel (k_pair_fx): periodic box with the guard-free
  // image condition (TMD_B200_FX=1 or 2).
  const int fx = env_switch("TMD_B200_FX", TMD_DEFAULT_FX);
  ctx->fx_packed = fx == 2;
  priv(ctx).grid_fx = (((fx == 1 || fx == 2) && ctx->safe_image) || (use_cluster && ctx->periodic)) && ctx->pair_mask && !f64;

  // cell grid per replica
  std::vector<Grid> grids(R);
  long long max_cells = 1;
  double max_density = 0.0;
  for (int r = 0; r < R; ++r) {
    Grid& g = grids[r];
    box_grid(ctx, g, &ctx->box_host[r * 3], rl, margin, nullptr);
    max_cells = std::max<long long>(max_cells, g.ncells);
    if (ctx->periodic) max_density = std::max(max_density, N / ((double)g.L[0] * g.L[1] * g.L[2]));
  }
  if (!ctx->periodic && has_cut) max_cells = use_cluster ? 40 * 40 * 40 : 64 * 64 * 64;  // (cluster path: a bucket per cell)
  d.max_cells = (int)max_cells;
  // full-row list build: a grid of a few cells is shared out over more CTAs than cells
  d.build_split = (ctx->periodic && max_cells < ctx->nsm) ? (int)std::min<long long>(64, (ctx->nsm + max_cells - 1) / max_cells) : 1;

  d.xf_s = nullptr;
  if (priv(ctx).grid_fx && !use_cluster) {
    const size_t n = (size_t)R * N + R;
    if ((rc = device_alloc(&ctx->xf_buf, n))) return rc;
    TMD_CUDA(cudaMemset(ctx->xf_buf, 0, n * sizeof(int4)));
    d.xf_s = ctx->xf_buf;
  }

  // neighbour row capacity
  long long cap;
  if (!has_cut) cap = N;
  else if (ctx->periodic) cap = (long long)(4.0 / 3.0 * M_PI * rl * rl * rl * max_density * 1.3) + 48;
  else cap = 512;
  cap = std::min<long long>(cap, N);
  if (d.row_cap > cap) cap = d.row_cap;  // keep a capacity grown after an overflow
  d.row_cap = (int)(((std::max<long long>(cap, 64) + 63) / 64) * 64);  // rows are padded to 64-entry chunks

  if (ctx->pair_mask) {
    if (N >= (1 << 24) || d.ntypes > 128)
      return fail(TMD_ERR_UNSUPPORTED, "neighbour entries pack a 24-bit atom index and a 7-bit atom type: "
                                       "at most 16,777,216 atoms per replica and 128 atom types");
    const size_t need = use_cluster ? 256 : (size_t)R * N * d.row_cap + 256;  // slack: the pair loop prefetches past a row's end
    if (need * sizeof(int) > (size_t)64 << 30)  // (an H100 has 80 GB)
      return fail(TMD_ERR_UNSUPPORTED, "neighbour list would exceed 64 GiB (no cutoff on a large system?)");
    if (need != priv(ctx).nbr_entries) {
      if ((rc = device_alloc(&d.nbr, need))) return rc;
      priv(ctx).nbr_entries = need;
    }
    if ((rc = device_alloc(&d.cell_count, (size_t)R * (max_cells + 1)))) return rc;
    if ((rc = device_alloc(&d.cell_start, (size_t)R * (max_cells + 1)))) return rc;
    TMD_CUDA(cudaMemset(d.cell_count, 0, (size_t)R * (max_cells + 1) * sizeof(int)));
    TMD_CUDA(cudaMemset(d.cell_start, 0, (size_t)R * (max_cells + 1) * sizeof(int)));
  }
  // cluster path: slot arrays and lists
  {
    CtxPriv& pv = priv(ctx);
    const int keep_ecap = cl.ecap, keep_mcap = cl.mcap;
    for (void* b : pv.cl_bufs) cudaFree(b);
    pv.cl_bufs.clear();
    memset(&cl, 0, sizeof(cl));
    if (use_cluster) {
      long long rows = 1;
      for (int r = 0; r < R; ++r) rows = std::max<long long>(rows, (long long)grids[r].n[1] * grids[r].n[2]);
      if (!ctx->periodic) rows = 40 * 40;  // the device sizes that grid
      const long long slots = ((long long)N + rows * (CL - 1) + CL - 1) / CL * CL;
      cl.on = 1;
      cl.max_rows = (int)rows;
      cl.slots = (int)slots;
      cl.nclusters_cap = (int)(slots / CL);
      cl.max_extent = (float)cl_max_extent;
      // entries per cluster: half of the atoms within rl of a box of about (2.5, w, w) A, with head room
      const double w = rl / d.nsub, a = 2.5, rho = std::max(max_density, 0.11);
      const double vol = a * w * w + 2.0 * (a * w + w * w + a * w) * rl + M_PI * (a + 2 * w) * rl * rl + 4.0 / 3.0 * M_PI * rl * rl * rl;
      long long ecap = (long long)(0.5 * rho * vol * 1.6) + 128;
      if (const char* e = getenv("TMD_B200_CLUSTER_ECAP")) ecap = std::max(32, atoi(e));  // (tests: start too small, grow)
      ecap = std::max<long long>(ecap, keep_ecap);
      ecap = std::min<long long>((ecap + 31) / 32 * 32, ((long long)N + 31) / 32 * 32);
      cl.ecap = (int)std::max<long long>(ecap, 32);
      cl.mcap = std::max(64, keep_mcap);
      auto grab = [&](auto** ptr, size_t n) {
        void* b = nullptr;
        if (cudaMalloc(&b, n * sizeof(**ptr)) != cudaSuccess) return false;
        pv.cl_bufs.push_back(b);
        *ptr = reinterpret_cast<std::remove_reference_t<decltype(**ptr)>*>(b);
        return true;
      };
      const size_t S1 = (size_t)R * (slots + 1), C1 = (size_t)R * cl.nclusters_cap;
      const size_t ne = C1 * (size_t)(cl.mcap + cl.ecap);
      if (ne * 4 > ((size_t)64 << 30)) return fail(TMD_ERR_UNSUPPORTED, "cluster lists would exceed 64 GiB");
      bool ok = grab(&cl.xq, S1) && grab(&cl.f, S1) && grab(&cl.xw, S1) && (!ctx->periodic || grab(&cl.xf, S1)) &&
                grab(&cl.perm, S1) && grab(&cl.bucket, (size_t)R * d.max_cells * CL_BUCKET) &&
                grab(&cl.row_tot, (size_t)R * (rows + 1)) && grab(&cl.cell_owned, (size_t)R * (d.max_cells + 1)) && grab(&cl.owned_pre, (size_t)R * (d.max_cells + 1)) && grab(&cl.inv, (size_t)R * N) && grab(&cl.nslots, (size_t)R) &&
                grab(&cl.meta, C1) && grab(&cl.entries, ne + 64) && grab(&cl.masks, C1 * (size_t)cl.mcap + 64);
      if (!ok) return fail(TMD_ERR_CUDA, "cudaMalloc of the cluster lists failed");
      TMD_CUDA(cudaMemset(cl.xq, 0, S1 * sizeof(float4)));
      TMD_CUDA(cudaMemset(cl.f, 0, S1 * sizeof(float4)));
      if (cl.xf) TMD_CUDA(cudaMemset(cl.xf, 0, S1 * sizeof(int4)));
      TMD_CUDA(cudaMemset(cl.perm, 0xFF, S1 * sizeof(int)));
      TMD_CUDA(cudaMemset(cl.nslots, 0, (size_t)R * sizeof(int)));
      TMD_CUDA(cudaMemset(cl.cell_owned, 0, (size_t)R * (d.max_cells + 1) * sizeof(int)));
      TMD_CUDA(cudaMemset(cl.row_tot, 0, (size_t)R * (rows + 1) * sizeof(int)));
      TMD_CUDA(cudaMemset(cl.owned_pre, 0, (size_t)R * (d.max_cells + 1) * sizeof(int)));
      TMD_CUDA(cudaMemset(cl.meta, 0, C1 * sizeof(int2)));
      {
        std::vector<int> ident((size_t)R * N);
        for (int r = 0; r < R; ++r)
          for (int i = 0; i < N; ++i) ident[(size_t)r * N + i] = i;
        TMD_CUDA(cudaMemcpy(cl.inv, ident.data(), ident.size() * sizeof(int), cudaMemcpyHostToDevice));
      }
      // launch shape of k_cpair: persistent CTAs, as many as fit
      pv.cl_smem = (size_t)CL_WARPS * 2 * ((size_t)(cl.mcap + cl.ecap) * sizeof(unsigned) + cl.mcap) + (size_t)CL_WARPS * d.ntypes * CL_H * sizeof(ClTab);
#if !defined(TMD_SIMT_HOST)
      if (pv.cl_smem > (size_t)180 * 1024) return fail(TMD_ERR_UNSUPPORTED, "cluster lists too long for the shared-memory staging");
      int per_sm = 0;
      const void* kernels[6] = {(const void*)k_cpair<false, false>, (const void*)k_cpair<false, true>,
                                (const void*)k_cpair<true, false>, (const void*)k_cpair<true, true>,
                                (const void*)k_cpair_ew<false>, (const void*)k_cpair_ew<true>};
      for (const void* k : kernels) TMD_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pv.cl_smem));
      TMD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_cpair<false, true>, CL_WARPS * 32, pv.cl_smem));
      pv.cl_blocks = std::max(1, std::min(ctx->nsm * std::max(per_sm, 1), (cl.nclusters_cap + CL_WARPS - 1) / CL_WARPS));
#else
      if (cl.mcap + cl.ecap > CL_SIMT_MAX_ENTRIES || d.ntypes > CL_SIMT_MAX_TYPES) return fail(TMD_ERR_UNSUPPORTED, "interpreter build: cluster list too long");
      pv.cl_blocks = std::max(1, std::min(16, (cl.nclusters_cap + CL_WARPS - 1) / CL_WARPS));
#endif
    }
  }
  TMD_CUDA(cudaMemcpy(d.grid, grids.data(), (size_t)R * sizeof(Grid), cudaMemcpyHostToDevice));
  TMD_CUDA(cudaMemset(d.pos_ref, 0xFF, (size_t)R * N * sizeof(float4)));  // NaN: forces a build
  if (priv(ctx).flags_live) {  // a re-finalisation (grown lists, another pair path): the build count carries over
    std::vector<int> fl((size_t)R * F_COUNT);
    TMD_CUDA(cudaMemcpy(fl.data(), d.flags, fl.size() * sizeof(int), cudaMemcpyDeviceToHost));
    for (int r = 0; r < R; ++r) ctx->rebuilds_before += fl[r * F_COUNT + F_NREBUILD];
  }
  priv(ctx).flags_live = true;
  TMD_CUDA(cudaMemset(d.flags, 0, (size_t)R * F_COUNT * sizeof(int)));
  TMD_CUDA(cudaMemset(d.counters, 0, sizeof(unsigned long long)));  // flag parity restarts with the flags
  {
    std::vector<int> ident((size_t)R * N);
    for (int r = 0; r < R; ++r)
      for (int i = 0; i < N; ++i) ident[(size_t)r * N + i] = i;
    TMD_CUDA(cudaMemcpy(d.inv, ident.data(), ident.size() * sizeof(int), cudaMemcpyHostToDevice));
    TMD_CUDA(cudaMemcpy(d.perm, ident.data(), ident.size() * sizeof(int), cudaMemcpyHostToDevice));
    std::vector<int> b((size_t)R * 6);
    const float pinf = INFINITY, ninf = -INFINITY;
    int ep, en;
    memcpy(&ep, &pinf, 4);  // enc(+inf) = bits of +inf
    memcpy(&en, &ninf, 4);
    en ^= 0x7fffffff;       // enc of a negative float
    for (int r = 0; r < R; ++r)
      for (int k = 0; k < 3; ++k) {
        b[r * 6 + k] = ep;
        b[r * 6 + 3 + k] = en;
      }
    TMD_CUDA(cudaMemcpy(d.bounds, b.data(), b.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  // atom -> bonded term entries (kind | slot | term), fixed order: deterministic bonded forces
  {
    const uint32_t bm = ctx->bonded_mask;
    struct Src { int kind, k; const std::vector<int32_t>* idx; bool on; };
    const Src src[5] = {
        {BK_BOND, 2, &ctx->bonds_idx_h, (bm & TMD_TERM(TMD_E_BONDS)) != 0},
        {BK_ANGLE, 3, &ctx->angles_idx_h, (bm & TMD_TERM(TMD_E_ANGLES)) != 0},
        {BK_DIHEDRAL, 4, &ctx->torsions_idx_h[0], (bm & TMD_TERM(TMD_E_DIHEDRALS)) != 0},
        {BK_PAIR14, 2, &ctx->pairs14_idx_h, (bm & TMD_TERM(TMD_E_14)) != 0},
        {BK_IMPROPER, 4, &ctx->torsions_idx_h[1], (bm & TMD_TERM(TMD_E_IMPROPERS)) != 0}};
    std::vector<int> ptr(N + 1, 0);
    for (const Src& sc : src)
      if (sc.on)
        for (int32_t a : *sc.idx) ptr[a + 1]++;
    for (int i = 0; i < N; ++i) ptr[i + 1] += ptr[i];
    std::vector<int> fill(ptr.begin(), ptr.end() - 1), ent(ptr[N]);
    for (const Src& sc : src) {
      if (!sc.on) continue;
      const size_t nt = sc.idx->size() / sc.k;
      if (nt >= (1u << 27)) return fail(TMD_ERR_UNSUPPORTED, "more than 2^27 bonded terms of one kind");
      for (size_t t = 0; t < nt; ++t)
        for (int sl = 0; sl < sc.k; ++sl)
          ent[fill[(*sc.idx)[t * sc.k + sl]]++] = (int)(((unsigned)sc.kind << 29) | ((unsigned)sl << 27) | (unsigned)t);
    }
    ctx->bonded_nentries = ptr[N];
    if ((rc = upload(&ctx->bonded_atom_ptr, ptr.data(), ptr.size()))) return rc;
    if ((rc = upload(&ctx->bonded_entries, ent.data(), ent.size()))) return rc;
    CtxPriv& pv = priv(ctx);
    pv.bonded_terms = env_switch("TMD_B200_BONDED_TERMS", 1) == 1 || f64;  // (fp64: the two-pass kernels only)
    const size_t need = pv.bonded_terms ? (size_t)R * ptr[N] * 3 : 0;  // one slot per (term, atom of the term) = per entry
    if (need > pv.term_forces_len) {
      if (pv.term_forces) cudaFree(pv.term_forces);
      pv.term_forces = nullptr;
      pv.term_forces_len = 0;
      if ((rc = device_alloc(&pv.term_forces, need))) return rc;
      pv.term_forces_len = need;
    }
  }
  // cooperative rebuild kernel: as many CTAs as can be co-resident, split over the replicas
  ctx->coop_blocks = 0;
  {
    const bool want_coop = env_switch("TMD_B200_COOP", TMD_DEFAULT_COOP) == 1;
    int coop = 0, per_sm = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, ctx->device);
    // opt-in (TMD_B200_COOP=1): a grid-wide barrier can only deadlock, never fail, if co-residency
    // is ever violated -- the separate gated kernels are the default
    if (coop && want_coop &&
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_rebuild, BT_WARPS * 32, 0) == cudaSuccess) {
      const int total = per_sm * ctx->nsm;
      if (total >= R) ctx->coop_blocks = std::max(1, total / R);
    }
  }
  // bonded kernel concurrent with the pair kernel (TMD_B200_OVERLAP)
  {
    CtxPriv& pv = priv(ctx);
    const bool want = env_switch("TMD_B200_OVERLAP", TMD_DEFAULT_OVERLAP) == 1 && ctx->bonded_nentries > 0 && ctx->pair_mask && !f64;
    if (want && !pv.side) {
      TMD_CUDA(cudaStreamCreateWithFlags(&pv.side, cudaStreamNonBlocking));
      TMD_CUDA(cudaEventCreateWithFlags(&pv.ev_fork, cudaEventDisableTiming));
      TMD_CUDA(cudaEventCreateWithFlags(&pv.ev_join, cudaEventDisableTiming));
      if ((rc = device_alloc(&pv.bonded_scratch, (size_t)R * N * 3))) return rc;
      TMD_CUDA(cudaMemset(pv.bonded_scratch, 0, (size_t)R * N * 3 * sizeof(double)));
    }
    if (!want && pv.side) {
      cudaStreamDestroy(pv.side);
      pv.side = nullptr;
    }
  }
  {
    CtxPriv& pv = priv(ctx);
    pv.use_graph = env_switch("TMD_B200_GRAPH", TMD_DEFAULT_GRAPH) == 1;
    // (without the compiled-in node: five gated kernels, as in stream order)
    pv.use_cond = TMD_COND_NODE && (env_switch("TMD_B200_COND", TMD_DEFAULT_COND) == 1 || pv.use_graph);
    if (pv.use_cond && !pv.helper) TMD_CUDA(cudaStreamCreateWithFlags(&pv.helper, cudaStreamNonBlocking));
    if (pv.use_graph && !pv.gstream) {
      TMD_CUDA(cudaStreamCreateWithFlags(&pv.gstream, cudaStreamNonBlocking));
      TMD_CUDA(cudaEventCreateWithFlags(&pv.ev_in, cudaEventDisableTiming));
      TMD_CUDA(cudaEventCreateWithFlags(&pv.ev_out, cudaEventDisableTiming));
    }
    pv.fuse_prepare = env_switch("TMD_B200_FUSEPREP", TMD_DEFAULT_FUSEPREP) == 1;
    pv.fuse_step = env_switch("TMD_B200_FUSESTEP", TMD_DEFAULT_FUSESTEP) == 1;
    pv.steps_valid = false;  // buffers may have moved: captured steps are rebuilt
  }
  if (f64) {
    DeviceState64& D = ctx->d64;
    std::vector<double> qs(N);
    const double sk = sqrt(ctx->coulomb > 0 ? ctx->coulomb : 0.0);
    for (int i = 0; i < N; ++i) qs[i] = ctx->charges64_host[i] * sk;
    if ((rc = upload(&ctx->q64, qs.data(), (size_t)N))) return rc;
    if ((rc = upload(&ctx->L64, ctx->box64_host.data(), ctx->box64_host.size()))) return rc;
    if ((rc = device_alloc(&ctx->xq64, (size_t)R * (N + 1)))) return rc;
    TMD_CUDA(cudaMemset(ctx->xq64, 0xFF, (size_t)R * (N + 1) * sizeof(Rec64)));  // NaN, incl. the sentinels
    if ((rc = device_alloc(&ctx->shadow, (size_t)R * N * 3))) return rc;
    D.xq_s = ctx->xq64;
    D.shadow = ctx->shadow;
    D.q = ctx->q64;
    D.AB = ctx->AB64;
    D.L = ctx->L64;
    D.pos_limit = has_cut ? F64_POS_LIMIT : INFINITY;  // without a cutoff every pair is listed: nothing to bound
    D.pp.true_gradient = ctx->exact_gradient;
  }
  if (pme_on(ctx) && (rc = pme_finalize(ctx, stream))) return rc;
  if (!priv(ctx).box_dev && (rc = device_alloc(&priv(ctx).box_dev, (size_t)R * 3))) return rc;
  TMD_CUDA(cudaMemcpy(priv(ctx).box_dev, ctx->box64_host.data(), (size_t)R * 3 * sizeof(double), cudaMemcpyHostToDevice));
  priv(ctx).grids = grids;
  priv(ctx).rescaled = false;
  priv(ctx).dirty = false;
  return TMD_OK;
}

// Particle-mesh Ewald (a periodic box) on the full rows: the real-space Ewald instantiations of the same kernels the
// context would run without it, and nothing else.  tmd_pair_kernel(): 6 k_pair<MODE 2>, 7 k_pair_fx<MODE 2>,
// 9 k_pair_fx2_ew (the cluster path: 10 k_cpair_ew).
static void launch_pair_ewald(tmd_ctx* ctx, dim3 pg, cudaStream_t st, float* forces, double* energies) {
  const bool e = energies != nullptr, small = ctx->d.ntypes <= FX_SMALLT_MAX;
  const int th = PAIR_WARPS * 32;
  const bool lj_el_only = ctx->pair_mask != 0 && (ctx->pair_mask & ~(T_LJ | T_ELEC)) == 0;
  if (ctx->d.xf_s && ctx->fx_packed && lj_el_only && !ctx->exact_gradient && ctx->d.ntypes <= 128) {
    ctx->last_pair_kernel = 9;
    const SwitchConsts sc = make_switch_consts_ewald(ctx->d.pp);
    if (e && small) launch(k_pair_fx2_ew<true, true>, pg, th, st, ctx->d, sc, forces, energies);
    else if (e) launch(k_pair_fx2_ew<true, false>, pg, th, st, ctx->d, sc, forces, energies);
    else if (small) launch(k_pair_fx2_ew<false, true>, pg, th, st, ctx->d, sc, forces, energies);
    else launch(k_pair_fx2_ew<false, false>, pg, th, st, ctx->d, sc, forces, energies);
    return;
  }
  if (ctx->d.xf_s) {
    ctx->last_pair_kernel = 7;
    if (e && small) launch(k_pair_fx<true, 2, true>, pg, th, st, ctx->d, forces, energies);
    else if (e) launch(k_pair_fx<true, 2, false>, pg, th, st, ctx->d, forces, energies);
    else if (small) launch(k_pair_fx<false, 2, true>, pg, th, st, ctx->d, forces, energies);
    else launch(k_pair_fx<false, 2, false>, pg, th, st, ctx->d, forces, energies);
    return;
  }
  ctx->last_pair_kernel = 6;
  if (ctx->safe_image) {
    if (e) launch(k_pair<true, true, true, 2>, pg, th, st, ctx->d, forces, energies);
    else launch(k_pair<false, true, true, 2>, pg, th, st, ctx->d, forces, energies);
  } else {
    if (e) launch(k_pair<true, true, false, 2>, pg, th, st, ctx->d, forces, energies);
    else launch(k_pair<false, true, false, 2>, pg, th, st, ctx->d, forces, energies);
  }
}
template <bool E, bool P, bool SAFE>
static void launch_pair_mode(tmd_ctx* ctx, dim3 pg, cudaStream_t st, float* forces, double* energies) {
  if (ctx->pair_mode == 1) launch(k_pair<E, P, SAFE, 1>, pg, PAIR_WARPS * 32, st, ctx->d, forces, energies);
  else launch(k_pair<E, P, SAFE, 0>, pg, PAIR_WARPS * 32, st, ctx->d, forces, energies);
}
template <bool E>
static void launch_pair_fx(tmd_ctx* ctx, dim3 pg, cudaStream_t st, float* forces, double* energies) {
  const bool small = ctx->d.ntypes <= FX_SMALLT_MAX;
  const int th = PAIR_WARPS * 32;
  // TMD_B200_FX=2: fp32x2 arithmetic for the term sets made of "lj" and "electrostatics"
  const bool lj_el_only = ctx->pair_mask != 0 && (ctx->pair_mask & ~(T_LJ | T_ELEC)) == 0;
  if (ctx->fx_packed && lj_el_only && !ctx->exact_gradient && ctx->d.ntypes <= 128) {
    ctx->last_pair_kernel = 2;
    const SwitchConsts sc = make_switch_consts(ctx->d.pp);
    if (small) launch(k_pair_fx2<E, true>, pg, th, st, ctx->d, sc, forces, energies);
    else launch(k_pair_fx2<E, false>, pg, th, st, ctx->d, sc, forces, energies);
    return;
  }
  ctx->last_pair_kernel = 1;
  if (ctx->pair_mode == 1) {
    if (small) launch(k_pair_fx<E, 1, true>, pg, th, st, ctx->d, forces, energies);
    else launch(k_pair_fx<E, 1, false>, pg, th, st, ctx->d, forces, energies);
  } else {
    if (small) launch(k_pair_fx<E, 0, true>, pg, th, st, ctx->d, forces, energies);
    else launch(k_pair_fx<E, 0, false>, pg, th, st, ctx->d, forces, energies);
  }
}
static void launch_pair(tmd_ctx* ctx, dim3 pg, cudaStream_t st, float* forces, double* energies) {
  const bool e = energies != nullptr;
  ctx->last_pair_kernel = 0;
  if (pme_on(ctx)) {
    launch_pair_ewald(ctx, pg, st, forces, energies);
  } else if (ctx->d.xf_s) {
    if (e) launch_pair_fx<true>(ctx, pg, st, forces, energies);
    else launch_pair_fx<false>(ctx, pg, st, forces, energies);
  } else if (!ctx->periodic && ctx->fx_packed && ctx->pair_mask != 0 && (ctx->pair_mask & ~(T_LJ | T_ELEC)) == 0 &&
             !ctx->exact_gradient) {
    // TMD_B200_FX=2 without a box: fp32x2 arithmetic on the float records
    ctx->last_pair_kernel = 3;
    const SwitchConsts sc = make_switch_consts(ctx->d.pp);
    const bool small = ctx->d.ntypes <= FX_SMALLT_MAX;
    const int th = PAIR_WARPS * 32;
    if (e && small) launch(k_pair2_open<true, true>, pg, th, st, ctx->d, sc, forces, energies);
    else if (e) launch(k_pair2_open<true, false>, pg, th, st, ctx->d, sc, forces, energies);
    else if (small) launch(k_pair2_open<false, true>, pg, th, st, ctx->d, sc, forces, energies);
    else launch(k_pair2_open<false, false>, pg, th, st, ctx->d, sc, forces, energies);
  } else if (!ctx->periodic) {
    if (e) launch_pair_mode<true, false, false>(ctx, pg, st, forces, energies);
    else launch_pair_mode<false, false, false>(ctx, pg, st, forces, energies);
  } else if (ctx->safe_image) {
    if (e) launch_pair_mode<true, true, true>(ctx, pg, st, forces, energies);
    else launch_pair_mode<false, true, true>(ctx, pg, st, forces, energies);
  } else {
    if (e) launch_pair_mode<true, true, false>(ctx, pg, st, forces, energies);
    else launch_pair_mode<false, true, false>(ctx, pg, st, forces, energies);
  }
}

static inline dim3 atoms_grid(const tmd_ctx* ctx, int threads) {
  return dim3((unsigned)((ctx->natoms + threads - 1) / threads), (unsigned)ctx->nrep);
}
static inline dim3 owned_grid(const tmd_ctx* ctx, int threads) {
  return dim3((unsigned)((std::max(ctx->d.own_n, 1) + threads - 1) / threads), (unsigned)ctx->nrep);
}

// The kernels' bonded table (BondedTables or BondedTables64) from the context's sets, disabled terms emptied.
template <typename Tables, typename Set>
static Tables bonded_tables(const tmd_ctx* ctx, const Set& bonds, const Set& angles, const Set* torsions, const Set& pairs14) {
  const uint32_t bm = ctx->bonded_mask;
  Tables T;
  T.atom_ptr = ctx->bonded_atom_ptr;
  T.entries = ctx->bonded_entries;
  T.bonds = bonds;
  T.angles = angles;
  T.torsions[0] = torsions[0];
  T.torsions[1] = torsions[1];
  T.pairs14 = pairs14;
  if (!(bm & TMD_TERM(TMD_E_BONDS))) T.bonds.n = 0;
  if (!(bm & TMD_TERM(TMD_E_ANGLES))) T.angles.n = 0;
  if (!(bm & TMD_TERM(TMD_E_DIHEDRALS))) T.torsions[0].n = 0;
  if (!(bm & TMD_TERM(TMD_E_IMPROPERS))) T.torsions[1].n = 0;
  if (!(bm & TMD_TERM(TMD_E_14))) T.pairs14.n = 0;
  return T;
}
// Where each (kind, term, slot) force sits in the per-term buffer of k_bonded_terms / k_bonded_sum.
template <typename Tables>
static TermLayout term_layout(const Tables& T) {
  TermLayout lay;
  const int cnt[5] = {T.bonds.n, T.angles.n, T.torsions[0].n, T.torsions[1].n, T.pairs14.n};
  int nt = 0, ns = 0;
  for (int k = 0; k < 5; ++k) {
    lay.first[k] = nt;
    lay.slot0[k] = ns;
    nt += cnt[k];
    ns += cnt[k] * term_arity(k);
  }
  lay.nterms = nt;
  lay.nslots = ns;
  return lay;
}

// The gated full-row rebuild (neighbor.cuh) from the fp32 positions `pos`: every kernel returns at once unless
// k_prepare raised the replica's rebuild flag.
static int enqueue_rebuild_rows(tmd_ctx* ctx, const float* pos, int need_bounds, cudaStream_t rs) {
  const DeviceState& d = ctx->d;
  const int R = ctx->nrep;
  if (need_bounds) {
    launch(k_bounds, atoms_grid(ctx, 256), 256, rs, d, pos);
    TMD_LAUNCHED(ctx, "k_bounds");
    launch(k_grid, (R + 63) / 64, 64, rs, d);
    TMD_LAUNCHED(ctx, "k_grid");
  }
  launch(k_bin, atoms_grid(ctx, 256), 256, rs, d, pos);
  TMD_LAUNCHED(ctx, "k_bin");
  launch(k_scan, R, 1024, rs, d);
  TMD_LAUNCHED(ctx, "k_scan");
  launch(k_place, atoms_grid(ctx, 256), 256, rs, d);
  TMD_LAUNCHED(ctx, "k_place");
  {
    const int blocks = std::max(1, std::min((d.max_cells + 7) / 8, ctx->nsm * 8));
    launch(k_sort_pack, dim3(blocks, R), 256, rs, d);
    TMD_LAUNCHED(ctx, "k_sort_pack");
  }
  launch(k_build_list, dim3(std::max(1, std::min(d.max_cells * std::max(1, d.build_split), ctx->nsm * 12)), R), BT_WARPS * 32, rs, d);
  TMD_LAUNCHED(ctx, "k_build_list");
  return TMD_OK;
}

// Particle-mesh Ewald reciprocal chain (pme.cuh) up to phi on the grid: spread, then the 3D DFT as lines along z, y,
// x (with the influence function), y, z.  Six kernels; k_pme_gather follows once the forces buffer holds the pair forces.
template <typename T>
static int enqueue_pme_chain(tmd_ctx* ctx, const T* pos, double* energies, cudaStream_t s) {
  const PmeArgs& a = priv(ctx).pme;
  const unsigned R = (unsigned)ctx->nrep;
  launch(k_pme_spread<T>, atoms_grid(ctx, PME_THREADS), PME_THREADS, s, a, pos);
  TMD_LAUNCHED(ctx, "k_pme_spread");
  auto nl = [&](int axis) { return pme_lines_log2<T>(a.K[axis], axis); };
  auto blocks = [&](int axis) {
    const long long lines = a.ktot / a.K[axis], per = 1ll << nl(axis);
    return dim3((unsigned)((lines + per - 1) / per), R);
  };
  launch(k_pme_fft<T, PME_FIRST>, blocks(2), PME_THREADS, s, a, 2, nl(2), (double*)nullptr);
  TMD_LAUNCHED(ctx, "k_pme_fft");
  launch(k_pme_fft<T, PME_FWD>, blocks(1), PME_THREADS, s, a, 1, nl(1), (double*)nullptr);
  TMD_LAUNCHED(ctx, "k_pme_fft");
  launch(k_pme_fft<T, PME_CONV>, blocks(0), PME_THREADS, s, a, 0, nl(0), energies);
  TMD_LAUNCHED(ctx, "k_pme_fft");
  launch(k_pme_fft<T, PME_INV>, blocks(1), PME_THREADS, s, a, 1, nl(1), (double*)nullptr);
  TMD_LAUNCHED(ctx, "k_pme_fft");
  launch(k_pme_fft<T, PME_INV>, blocks(2), PME_THREADS, s, a, 2, nl(2), (double*)nullptr);
  TMD_LAUNCHED(ctx, "k_pme_fft");
  return TMD_OK;
}
template <typename T>
static int enqueue_pme_gather(tmd_ctx* ctx, const T* pos, T* forces, double* energies, cudaStream_t s) {
  launch(k_pme_gather<T>, atoms_grid(ctx, PME_THREADS), PME_THREADS, s, priv(ctx).pme, pos, forces, energies);
  TMD_LAUNCHED(ctx, "k_pme_gather");
  return TMD_OK;
}

// Forces.compute on an fp64 context: preparation (fp32 shadow), the gated fp32 list build on the shadow, the fp64
// records in the new order, k_pair_f64, then the two bonded passes in stream order.
static int enqueue_forces_f64(tmd_ctx* ctx, const double* pos, double* forces, double* energies, cudaStream_t st) {
  const DeviceState& d = ctx->d;
  const DeviceState64& D = ctx->d64;
  const int N = ctx->natoms, R = ctx->nrep;
  ctx->force_calls++;
  if (energies) TMD_CUDA(cudaMemsetAsync(energies, 0, (size_t)R * TMD_NUM_ENERGIES * sizeof(double), st));
  if (ctx->pair_mask) {
    launch(k_prepare_f64, atoms_grid(ctx, 256), 256, st, d, D, pos);
    TMD_LAUNCHED(ctx, "k_prepare_f64");
    if (int rc = enqueue_rebuild_rows(ctx, D.shadow, (!ctx->periodic && ctx->cutoff >= 0) ? 1 : 0, st)) return rc;
    launch(k_pack_f64, atoms_grid(ctx, 256), 256, st, d, D, pos);
    TMD_LAUNCHED(ctx, "k_pack_f64");
    const bool pme = pme_on(ctx);
    if (pme)
      if (int rc = enqueue_pme_chain<double>(ctx, pos, energies, st)) return rc;
    CtxPriv& pv = priv(ctx);
    const bool sample = pv.profiling && (size_t)(pv.ev_used + 2) <= pv.ev.size();
    if (sample) TMD_CUDA(cudaEventRecord(pv.ev[pv.ev_used], st));
    const dim3 pg((N + PAIR_WARPS - 1) / PAIR_WARPS, R);
    const int th = PAIR_WARPS * 32;
    ctx->last_pair_kernel = pme ? 8 : 5;
    if (pme && energies) launch(k_ewpair64<true>, pg, th, st, d, D, forces, energies);
    else if (pme) launch(k_ewpair64<false>, pg, th, st, d, D, forces, energies);
    else if (energies && ctx->periodic) launch(k_pair_f64<true, true>, pg, th, st, d, D, forces, energies);
    else if (energies) launch(k_pair_f64<true, false>, pg, th, st, d, D, forces, energies);
    else if (ctx->periodic) launch(k_pair_f64<false, true>, pg, th, st, d, D, forces, energies);
    else launch(k_pair_f64<false, false>, pg, th, st, d, D, forces, energies);
    TMD_LAUNCHED(ctx, "k_pair_f64");
    if (sample) {
      TMD_CUDA(cudaEventRecord(pv.ev[pv.ev_used + 1], st));
      pv.ev_used += 2;
    }
    if (pme)
      if (int rc = enqueue_pme_gather<double>(ctx, pos, forces, energies, st)) return rc;
  } else {
    TMD_CUDA(cudaMemsetAsync(forces, 0, (size_t)R * N * 3 * sizeof(double), st));
  }
  if (ctx->bonded_nentries > 0) {
    const BondedTables64 T = bonded_tables<BondedTables64>(ctx, ctx->bonds64, ctx->angles64, ctx->torsions64, ctx->pairs1464);
    const TermLayout lay = term_layout(T);
    launch(k_bonded_terms_f64, dim3((std::max(lay.nterms, 1) + BONDED_THREADS - 1) / BONDED_THREADS, R), BONDED_THREADS, st, d, D, T, lay,
           pos, energies, priv(ctx).term_forces);
    TMD_LAUNCHED(ctx, "k_bonded_terms_f64");
    launch(k_bonded_sum_f64, atoms_grid(ctx, BONDED_THREADS), BONDED_THREADS, st, d, T, lay, (const double*)priv(ctx).term_forces, forces);
    TMD_LAUNCHED(ctx, "k_bonded_sum_f64");
  }
  return TMD_OK;
}

static int enqueue_forces(tmd_ctx* ctx, const float* pos, float* forces, double* energies, cudaStream_t st) {
  DeviceState& d = ctx->d;
  const int N = ctx->natoms, R = ctx->nrep;
  ctx->force_calls++;
  if (energies) TMD_CUDA(cudaMemsetAsync(energies, 0, (size_t)R * TMD_NUM_ENERGIES * sizeof(double), st));
  // particle-mesh Ewald: the reciprocal chain needs only the positions, so it runs on its own stream beside the list
  // check and the pair kernel; k_pme_gather joins it after the pair kernel
  const bool pme = pme_on(ctx);
  if (pme) {
    CtxPriv& pv = priv(ctx);
    TMD_CUDA(cudaEventRecord(pv.pme_fork, st));
    TMD_CUDA(cudaStreamWaitEvent(pv.pme_side, pv.pme_fork, 0));
    if (int prc = enqueue_pme_chain<float>(ctx, pos, energies, pv.pme_side)) return prc;
    TMD_CUDA(cudaEventRecord(pv.pme_join, pv.pme_side));
  }

  BondedTables T;
  const bool have_bonded = ctx->bonded_nentries > 0;
  if (have_bonded) T = bonded_tables<BondedTables>(ctx, ctx->bonds, ctx->angles, ctx->torsions, ctx->pairs14);
  // bonded forces of the owned atoms: terms in parallel, then the fixed-order sum per atom (bonded.cuh)
  auto launch_bonded = [&](cudaStream_t bs, double* scratch) -> int {
    CtxPriv& pv = priv(ctx);
    if (!pv.bonded_terms) {
      launch(k_bonded, owned_grid(ctx, BONDED_THREADS), BONDED_THREADS, bs, d, T, ctx->q, pos, forces, energies, scratch);
      TMD_LAUNCHED(ctx, "k_bonded");
      return TMD_OK;
    }
    const TermLayout lay = term_layout(T);
    launch(k_bonded_terms, dim3((std::max(lay.nterms, 1) + BONDED_THREADS - 1) / BONDED_THREADS, R), BONDED_THREADS, bs, d, T, lay, ctx->q, pos,
           energies, pv.term_forces);
    TMD_LAUNCHED(ctx, "k_bonded_terms");
    launch(k_bonded_sum, owned_grid(ctx, BONDED_THREADS), BONDED_THREADS, bs, d, T, lay, pv.term_forces, forces, scratch);
    TMD_LAUNCHED(ctx, "k_bonded_sum");
    return TMD_OK;
  };
  // fork: the bonded terms need only the positions, so they run on a second stream while the
  // list check and the pair kernel run here; joined by k_add_bonded below
  const bool overlap = have_bonded && ctx->pair_mask && priv(ctx).side != nullptr;
  if (overlap) {
    CtxPriv& pv = priv(ctx);
    TMD_CUDA(cudaEventRecord(pv.ev_fork, st));
    TMD_CUDA(cudaStreamWaitEvent(pv.side, pv.ev_fork, 0));
    if (int brc = launch_bonded(pv.side, pv.bonded_scratch)) return brc;
    TMD_CUDA(cudaEventRecord(pv.ev_join, pv.side));
  }

  if (ctx->pair_mask) {
    // Being captured into a CUDA graph?  Then the rebuild becomes the body of a conditional node.
    cudaGraph_t cap_graph = nullptr;
    bool in_body = false;
    if (priv(ctx).use_cond) {
      cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
      if (cudaStreamGetCaptureInfo(st, &cs, nullptr, &cap_graph, nullptr, nullptr) != cudaSuccess ||
          cs != cudaStreamCaptureStatusActive)
        cap_graph = nullptr;
    }
    cudaGraphConditionalHandle handle = 0;
    if (priv(ctx).prepared) {  // k_vv_first_prepare did k_prepare's work (tmd_md_steps)
      handle = priv(ctx).prepared_cond;
      priv(ctx).prepared = false;
    } else {
      DeviceState dp = d;  // k_prepare's copy carries the handle it switches on
      if (cap_graph) {
        TMD_CUDA(cudaGraphConditionalHandleCreate(&handle, cap_graph, 0, cudaGraphCondAssignDefault));
        dp.cond = (unsigned long long)handle;
      }
      launch(k_prepare, atoms_grid(ctx, 256), 256, st, dp, pos);
      TMD_LAUNCHED(ctx, "k_prepare");
    }
    const int need_bounds = (!ctx->periodic && ctx->cutoff >= 0) ? 1 : 0;
    cudaStream_t rs = st;  // stream the rebuild kernels are enqueued on
    cudaGraphNode_t cond_node = nullptr;
    if (cap_graph) {
      cudaStreamCaptureStatus cs;
      const cudaGraphNode_t* deps = nullptr;
      size_t ndeps = 0;
      TMD_CUDA(cudaStreamGetCaptureInfo(st, &cs, nullptr, &cap_graph, &deps, &ndeps));
      cudaGraphNodeParams np = {};  // (anonymous union member: no default constructor)
      np.type = cudaGraphNodeTypeConditional;
      np.conditional.handle = handle;
      np.conditional.type = cudaGraphCondTypeIf;
      np.conditional.size = 1;
      TMD_CUDA(cudaGraphAddNode(&cond_node, cap_graph, deps, ndeps, &np));
      TMD_CUDA(cudaStreamBeginCaptureToGraph(priv(ctx).helper, np.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                             cudaStreamCaptureModeRelaxed));
      rs = priv(ctx).helper;
      in_body = true;
    }
    const int64_t body_l0 = ctx->launches;
    priv(ctx).last_body_launches = 0;
    if (d.cl.on) {
      // cluster path: cell binning as before, then the row-padded sort and the cluster lists (cluster.cuh)
      if (need_bounds) {
        launch(k_bounds, atoms_grid(ctx, 256), 256, rs, d, pos);
        TMD_LAUNCHED(ctx, "k_bounds");
        launch(k_grid, (R + 63) / 64, 64, rs, d);
        TMD_LAUNCHED(ctx, "k_grid");
      }
      launch(k_cbin, dim3(std::min((N + 255) / 256, ctx->nsm * 8), R), 256, rs, d, pos);
      TMD_LAUNCHED(ctx, "k_cbin");
      launch(k_cscan, R, 1024, rs, d);
      TMD_LAUNCHED(ctx, "k_cscan");
      launch(k_ccells, dim3(std::max(1, std::min((d.cl.max_rows + 7) / 8, ctx->nsm * 4)), R), 256, rs, d);
      TMD_LAUNCHED(ctx, "k_ccells");
      launch(k_csort, dim3(std::min((N + 255) / 256, ctx->nsm * 8), R), 256, rs, d);
      TMD_LAUNCHED(ctx, "k_csort");
      launch(k_cbuild, dim3(std::max(1, std::min((d.cl.nclusters_cap + CLB_WARPS - 1) / CLB_WARPS, ctx->nsm * 16)), R), CLB_WARPS * 32, rs, d);
      TMD_LAUNCHED(ctx, "k_cbuild");
    } else if (ctx->coop_blocks > 0 && !in_body) {
      // the whole (gated) rebuild in one cooperative launch
      const float* pos_arg = pos;
      int nb_arg = need_bounds;
      void* args[] = {(void*)&d, (void*)&pos_arg, (void*)&nb_arg};
      TMD_CUDA(cudaLaunchCooperativeKernel((const void*)k_rebuild, dim3(ctx->coop_blocks, R), dim3(BT_WARPS * 32),
                                           args, 0, st));
      TMD_LAUNCHED(ctx, "k_rebuild");
    } else {
      if (int brc = enqueue_rebuild_rows(ctx, pos, need_bounds, rs)) return brc;
    }
    if (in_body) {
      priv(ctx).last_body_launches = ctx->launches - body_l0;
      cudaGraph_t body = nullptr;
      TMD_CUDA(cudaStreamEndCapture(priv(ctx).helper, &body));
      TMD_CUDA(cudaStreamUpdateCaptureDependencies(st, &cond_node, 1, cudaStreamSetCaptureDependencies));
    }

    const dim3 pg((std::max(d.own_n, 1) + PAIR_WARPS - 1) / PAIR_WARPS, R);
    CtxPriv& pv = priv(ctx);
    const bool sample = pv.profiling && (size_t)(pv.ev_used + 2) <= pv.ev.size();
    if (sample) TMD_CUDA(cudaEventRecord(pv.ev[pv.ev_used], st));
    if (d.cl.on && pme) {
      ctx->last_pair_kernel = 10;
      const SwitchConsts sc = make_switch_consts_ewald(d.pp);
      const dim3 cg(pv.cl_blocks, R);
      if (energies) launch_smem(k_cpair_ew<true>, cg, CL_WARPS * 32, pv.cl_smem, st, d, sc, energies);
      else launch_smem(k_cpair_ew<false>, cg, CL_WARPS * 32, pv.cl_smem, st, d, sc, energies);
    } else if (d.cl.on) {
      ctx->last_pair_kernel = 4;
      const SwitchConsts sc = make_switch_consts(d.pp);
      const dim3 cg(pv.cl_blocks, R);
      const bool e = energies != nullptr;
      if (e && ctx->periodic) launch_smem(k_cpair<true, true>, cg, CL_WARPS * 32, pv.cl_smem, st, d, sc, energies);
      else if (e) launch_smem(k_cpair<true, false>, cg, CL_WARPS * 32, pv.cl_smem, st, d, sc, energies);
      else if (ctx->periodic) launch_smem(k_cpair<false, true>, cg, CL_WARPS * 32, pv.cl_smem, st, d, sc, energies);
      else launch_smem(k_cpair<false, false>, cg, CL_WARPS * 32, pv.cl_smem, st, d, sc, energies);
    } else {
      launch_pair(ctx, pg, st, forces, energies);
    }
    TMD_LAUNCHED(ctx, "k_pair");
    if (sample) {
      TMD_CUDA(cudaEventRecord(pv.ev[pv.ev_used + 1], st));
      pv.ev_used += 2;
    }
    if (pme) {
      TMD_CUDA(cudaStreamWaitEvent(st, pv.pme_join, 0));
      if (int prc = enqueue_pme_gather<float>(ctx, pos, forces, energies, st)) return prc;
    }
  } else {
    TMD_CUDA(cudaMemsetAsync(forces, 0, (size_t)R * N * 3 * sizeof(float), st));
  }

  if (overlap) {
    CtxPriv& pv = priv(ctx);
    TMD_CUDA(cudaStreamWaitEvent(st, pv.ev_join, 0));
    if (pv.fold_next) {  // the integrator kernel that follows adds them (enqueue_vv_second)
      pv.fold_pending = true;
    } else if (d.cl.on) {
      launch(k_cadd_bonded, owned_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, d, forces, pv.bonded_scratch);
      TMD_LAUNCHED(ctx, "k_cadd_bonded");
    } else {
      launch(k_add_bonded, owned_grid(ctx, BONDED_THREADS), BONDED_THREADS, st, N, d.own_lo, d.own_n, forces, pv.bonded_scratch);
      TMD_LAUNCHED(ctx, "k_add_bonded");
    }
  } else if (d.cl.on && ctx->pair_mask && priv(ctx).defer_bonded && d.own_all) {
    // tmd_md_steps: bonded terms, the trip home from slot order and the second half-kick are one kernel
    priv(ctx).bonded_deferred = true;
    if (!have_bonded) memset(&T, 0, sizeof(T));
    priv(ctx).deferred_tables = T;
    priv(ctx).deferred_energies = energies;
    priv(ctx).deferred_pos = pos;
  } else if (have_bonded) {
    // (cluster path: this kernel also brings the pair forces home from slot order)
    if (int brc = launch_bonded(st, nullptr)) return brc;
  } else if (d.cl.on && ctx->pair_mask) {
    launch(k_cunsort, atoms_grid(ctx, 256), 256, st, d, forces);
    TMD_LAUNCHED(ctx, "k_cunsort");
  }
  return TMD_OK;
}

// the step boundary of tmd_md_steps (fused.cuh, k_cstep_boundary): what enqueue_vv_second + enqueue_vv_first would do
struct BoundaryArgs {
  double gamma;
  const float* vcoeff;
  uint64_t seed, step;
};

// ---- constraints (constrain.cuh) ------------------------------------------------------------
static inline bool has_constraints(tmd_ctx* ctx) { return priv(ctx).con_ngroups > 0; }
static inline ConstraintTables con_tables(tmd_ctx* ctx) {
  const CtxPriv& p = priv(ctx);
  return ConstraintTables{p.con_ngroups, p.con_groups, p.con_nfree, p.con_free, p.con_L};
}
// the positions before the drift: the bond directions SHAKE moves the atoms along
template <typename T>
static int con_save_ref(tmd_ctx* ctx, const T* pos, cudaStream_t st) {
  TMD_CUDA(cudaMemcpyAsync(priv(ctx).con_ref, pos, (size_t)ctx->nrep * ctx->natoms * 3 * sizeof(T), cudaMemcpyDeviceToDevice, st));
  return TMD_OK;
}
// ref == nullptr: the positions themselves give the directions (projection of a state)
template <typename T>
static int enqueue_constrain_pos(tmd_ctx* ctx, T* pos, const T* ref, T* vel, const T* masses, double dt, cudaStream_t st) {
  const dim3 g((priv(ctx).con_ngroups + CON_THREADS - 1) / CON_THREADS, ctx->nrep);
  launch(k_constrain_pos<T, false>, g, CON_THREADS, st, ctx->natoms, con_tables(ctx), pos, ref ? ref : pos, vel, masses,
         dt > 0.0 ? 1.0 / dt : 0.0, priv(ctx).con_fail, ctx->d);
  TMD_LAUNCHED(ctx, "k_constrain_pos");
  return TMD_OK;
}
// tmd_md_steps (fp32, whole system, TMD_B200_FUSEPREP): the position constraint also prepares the force call that
// follows on this stream (list check, slot records), as k_vv_first_prepare does without constraints
static bool con_can_prepare(tmd_ctx* ctx) { return priv(ctx).fuse_prepare && ctx->d.own_all && ctx->pair_mask; }
static int enqueue_constrain_pos_prepare(tmd_ctx* ctx, float* pos, const float* ref, float* vel, const float* masses, double dt,
                                         cudaStream_t st) {
  CtxPriv& pv = priv(ctx);
  DeviceState dp = ctx->d;
  pv.prepared_cond = 0;
  if (pv.use_cond) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaGraph_t cap_graph = nullptr;
    if (cudaStreamGetCaptureInfo(st, &cs, nullptr, &cap_graph, nullptr, nullptr) == cudaSuccess &&
        cs == cudaStreamCaptureStatusActive && cap_graph) {
      TMD_CUDA(cudaGraphConditionalHandleCreate(&pv.prepared_cond, cap_graph, 0, cudaGraphCondAssignDefault));
      dp.cond = (unsigned long long)pv.prepared_cond;
    }
  }
  const dim3 g((pv.con_ngroups + pv.con_nfree + CON_THREADS - 1) / CON_THREADS, ctx->nrep);
  launch(k_constrain_pos<float, true>, g, CON_THREADS, st, ctx->natoms, con_tables(ctx), pos, ref, vel, masses, 1.0 / dt,
         pv.con_fail, dp);
  TMD_LAUNCHED(ctx, "k_constrain_pos");
  pv.prepared = true;
  return TMD_OK;
}
// velocity projection; with ke, the kinetic energy after it
template <typename T>
static int enqueue_constrain_vel(tmd_ctx* ctx, const T* pos, T* vel, const T* masses, double* ke, cudaStream_t st) {
  const CtxPriv& p = priv(ctx);
  const int items = p.con_ngroups + (ke ? p.con_nfree : 0);
  const dim3 g((items + CON_THREADS - 1) / CON_THREADS, ctx->nrep);
  if (ke) {
    TMD_CUDA(cudaMemsetAsync(ke, 0, (size_t)ctx->nrep * sizeof(double), st));
    launch(k_constrain_vel<T, true>, g, CON_THREADS, st, ctx->natoms, con_tables(ctx), pos, vel, masses, ke);
  } else {
    launch(k_constrain_vel<T, false>, g, CON_THREADS, st, ctx->natoms, con_tables(ctx), pos, vel, masses, ke);
  }
  TMD_LAUNCHED(ctx, "k_constrain_vel");
  return TMD_OK;
}

static int enqueue_vv_first(tmd_ctx* ctx, float* pos, float* vel, const float* forces, const float* masses,
                            double dt, cudaStream_t st, bool forces_follow = false, const BoundaryArgs* boundary = nullptr) {
  CtxPriv& pv = priv(ctx);
  if (forces_follow && pv.fuse_prepare && ctx->d.own_all && ctx->pair_mask) {
    // the force call that follows on this stream finds its preparation done
    DeviceState dp = ctx->d;
    pv.prepared_cond = 0;
    if (pv.use_cond) {
      cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
      cudaGraph_t cap_graph = nullptr;
      if (cudaStreamGetCaptureInfo(st, &cs, nullptr, &cap_graph, nullptr, nullptr) == cudaSuccess &&
          cs == cudaStreamCaptureStatusActive && cap_graph) {
        TMD_CUDA(cudaGraphConditionalHandleCreate(&pv.prepared_cond, cap_graph, 0, cudaGraphCondAssignDefault));
        dp.cond = (unsigned long long)pv.prepared_cond;
      }
    }
    if (boundary) {  // the force call before left its fold to us (fold_pending)
      pv.fold_pending = false;
      const bool thermo = (boundary->gamma >= 0.0) && boundary->vcoeff != nullptr;
      const float fdt = (float)dt, hdt = (float)(0.5 * dt), ng = (float)(-boundary->gamma);
      if (thermo) launch(k_cstep_boundary<true>, atoms_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, dp, pos, vel, masses, fdt, hdt, ng, boundary->vcoeff, boundary->seed, boundary->step, pv.bonded_scratch);
      else launch(k_cstep_boundary<false>, atoms_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, dp, pos, vel, masses, fdt, hdt, ng, boundary->vcoeff, boundary->seed, boundary->step, pv.bonded_scratch);
      TMD_LAUNCHED(ctx, "k_cstep_boundary");
      pv.prepared = true;
      return TMD_OK;
    }
    launch(k_vv_first_prepare, atoms_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, dp, pos, vel, forces, masses, (float)dt,
           (float)(0.5 * dt));
    TMD_LAUNCHED(ctx, "k_vv_first_prepare");
    pv.prepared = true;
    return TMD_OK;
  }
  launch(k_vv_first, owned_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, 
      ctx->natoms, ctx->d.own_lo, ctx->d.own_n, ctx->d.counters, pos, vel, forces, masses, (float)dt, (float)(0.5 * dt));
  TMD_LAUNCHED(ctx, "k_vv_first");
  return TMD_OK;
}

static int enqueue_vv_second(tmd_ctx* ctx, float* vel, const float* forces, const float* masses, double dt,
                             double gamma, const float* vcoeff, const float* noise, uint64_t seed,
                             uint64_t step, double* ke, cudaStream_t st) {
  const bool thermo = (gamma >= 0.0) && vcoeff != nullptr;
  const dim3 g = owned_grid(ctx, INTEG_THREADS);
  const int lo = ctx->d.own_lo, cnt = ctx->d.own_n;
  const unsigned long long* ctr = ctx->d.counters;
  const float fdt = (float)dt, hdt = (float)(0.5 * dt), ng = (float)(-gamma);
  if (ke) TMD_CUDA(cudaMemsetAsync(ke, 0, (size_t)ctx->nrep * sizeof(double), st));
  if (priv(ctx).bonded_deferred) {
    CtxPriv& pv = priv(ctx);
    pv.bonded_deferred = false;
    float* fw = const_cast<float*>(forces);  // (tmd_md_steps owns this buffer: the force call's output)
    const dim3 gb = atoms_grid(ctx, BONDED_THREADS);
    const BondedTables& T = pv.deferred_tables;
    if (thermo) {
      if (ke) launch(k_bonded_vv_second<true, true>, gb, BONDED_THREADS, st, ctx->d, T, ctx->q, pv.deferred_pos, fw, pv.deferred_energies, vel, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
      else launch(k_bonded_vv_second<true, false>, gb, BONDED_THREADS, st, ctx->d, T, ctx->q, pv.deferred_pos, fw, pv.deferred_energies, vel, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
    } else {
      if (ke) launch(k_bonded_vv_second<false, true>, gb, BONDED_THREADS, st, ctx->d, T, ctx->q, pv.deferred_pos, fw, pv.deferred_energies, vel, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
      else launch(k_bonded_vv_second<false, false>, gb, BONDED_THREADS, st, ctx->d, T, ctx->q, pv.deferred_pos, fw, pv.deferred_energies, vel, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
    }
    TMD_LAUNCHED(ctx, "k_bonded_vv_second");
    return TMD_OK;
  }
  if (priv(ctx).fold_pending) {
    priv(ctx).fold_pending = false;
    float* fw = const_cast<float*>(forces);  // (tmd_md_steps owns this buffer: it handed it to enqueue_forces as the output)
    const double* sc = priv(ctx).bonded_scratch;
    if (ctx->d.cl.on) {  // cluster path: the pair forces come home from slot order on the way
      if (thermo) {
        if (ke) launch(k_cvv_second_fold<true, true>, g, INTEG_THREADS, st, ctx->d, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
        else launch(k_cvv_second_fold<true, false>, g, INTEG_THREADS, st, ctx->d, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
      } else {
        if (ke) launch(k_cvv_second_fold<false, true>, g, INTEG_THREADS, st, ctx->d, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
        else launch(k_cvv_second_fold<false, false>, g, INTEG_THREADS, st, ctx->d, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
      }
      TMD_LAUNCHED(ctx, "k_cvv_second_fold");
      return TMD_OK;
    }
    if (thermo) {
      if (ke) launch(k_vv_second_fold<true, true>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
      else launch(k_vv_second_fold<true, false>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
    } else {
      if (ke) launch(k_vv_second_fold<false, true>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
      else launch(k_vv_second_fold<false, false>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, fw, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke, sc);
    }
    TMD_LAUNCHED(ctx, "k_vv_second_fold");
    return TMD_OK;
  }
  if (thermo) {
    if (ke) launch(k_vv_second<true, true>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, forces, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
    else launch(k_vv_second<true, false>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, forces, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
  } else {
    if (ke) launch(k_vv_second<false, true>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, forces, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
    else launch(k_vv_second<false, false>, g, INTEG_THREADS, st, ctx->natoms, lo, cnt, ctr, vel, forces, masses, fdt, hdt, ng, vcoeff, noise, seed, step, ke);
  }
  TMD_LAUNCHED(ctx, "k_vv_second");
  return TMD_OK;
}

extern "C" {

int tmd_forces(tmd_ctx* ctx, const float* pos, float* forces, double* energies, tmd_stream stream) {
  if (!ctx || !pos || !forces) return fail(TMD_ERR_ARG, "tmd_forces: null pointer");
  TMD_PRECISION(ctx, 32, "tmd_forces")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (priv(ctx).dirty && (rc = finalize(ctx, st))) return rc;
  priv(ctx).prepared = false;  // (only tmd_md_steps prepares ahead of the force call)
  return enqueue_forces(ctx, pos, forces, energies, st);
}

int tmd_vv_first(tmd_ctx* ctx, float* pos, float* vel, const float* forces, const float* masses, double dt,
                 tmd_stream stream) {
  if (!ctx || !pos || !vel || !forces || !masses) return fail(TMD_ERR_ARG, "tmd_vv_first: null pointer");
  TMD_PRECISION(ctx, 32, "tmd_vv_first")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!has_constraints(ctx)) return enqueue_vv_first(ctx, pos, vel, forces, masses, dt, st);
  int rc;
  if ((rc = con_save_ref(ctx, pos, st)) || (rc = enqueue_vv_first(ctx, pos, vel, forces, masses, dt, st))) return rc;
  priv(ctx).con_pos = pos;
  return enqueue_constrain_pos(ctx, pos, static_cast<const float*>(priv(ctx).con_ref), vel, masses, dt, st);
}

int tmd_vv_second(tmd_ctx* ctx, float* vel, const float* forces, const float* masses, double dt, double gamma,
                  const float* vcoeff, const float* noise, uint64_t seed, uint64_t step_index, double* ke,
                  tmd_stream stream) {
  if (!ctx || !vel || !forces || !masses) return fail(TMD_ERR_ARG, "tmd_vv_second: null pointer");
  TMD_PRECISION(ctx, 32, "tmd_vv_second")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (!has_constraints(ctx)) return enqueue_vv_second(ctx, vel, forces, masses, dt, gamma, vcoeff, noise, seed, step_index, ke, st);
  if (!priv(ctx).con_pos) return fail(TMD_ERR_STATE, "tmd_vv_second: constraints are set but tmd_vv_first has not run");
  int rc;
  if ((rc = enqueue_vv_second(ctx, vel, forces, masses, dt, gamma, vcoeff, noise, seed, step_index, nullptr, st))) return rc;
  return enqueue_constrain_vel(ctx, static_cast<const float*>(priv(ctx).con_pos), vel, masses, ke, st);
}

int tmd_kinetic_energy(tmd_ctx* ctx, const float* vel, const float* masses, double* ke, tmd_stream stream) {
  if (!ctx || !vel || !masses || !ke) return fail(TMD_ERR_ARG, "tmd_kinetic_energy: null pointer");
  TMD_PRECISION(ctx, 32, "tmd_kinetic_energy")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  TMD_CUDA(cudaMemsetAsync(ke, 0, (size_t)ctx->nrep * sizeof(double), st));
  launch(k_kinetic, owned_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, ctx->natoms, ctx->d.own_lo, ctx->d.own_n, vel, masses, ke);
  TMD_LAUNCHED(ctx, "k_kinetic");
  return TMD_OK;
}

int tmd_md_steps(tmd_ctx* ctx, int niter, float* pos, float* vel, float* forces, const float* masses,
                 double dt, double gamma, const float* vcoeff, const float* noise, uint64_t seed,
                 uint64_t first_step, double* energies, double* ke, tmd_stream stream) {
  if (!ctx || !pos || !vel || !forces || !masses || niter < 0) return fail(TMD_ERR_ARG, "tmd_md_steps: bad arguments");
  TMD_PRECISION(ctx, 32, "tmd_md_steps")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (priv(ctx).dirty && (rc = finalize(ctx, st))) return rc;
  const size_t per_step = (size_t)ctx->nrep * ctx->natoms * 3;
  CtxPriv& pv = priv(ctx);
  pv.prepared = false;
  pv.fold_pending = false;
  pv.bonded_deferred = false;
  struct DeferScope {  // only inside tmd_md_steps does a vv_second follow every force call
    CtxPriv& p;
    explicit DeferScope(CtxPriv& q) : p(q) { p.defer_bonded = true; }
    ~DeferScope() { p.defer_bonded = false; }
  } defer_scope(pv);
  struct FoldScope {  // only inside tmd_md_steps does a vv_second follow every force call
    CtxPriv& p;
    explicit FoldScope(CtxPriv& q, bool on) : p(q) { p.fold_next = on; }
    ~FoldScope() { p.fold_next = false; }
  } fold_scope(pv, pv.fuse_prepare);
  // TMD_B200_FUSESTEP: inside one call the second half of a step and the first half of the next are one kernel
  // (cluster path with the bonded kernel on the side stream: the force call leaves its fold to the integrator)
  // With constraints the step is RATTLE: the position constraint sits between the drift and the force call and the
  // velocity constraint after the second half-kick, so neither the boundary kernel nor the fused prepare applies.
  const bool con = has_constraints(ctx);
  const bool fuse = pv.fuse_step && pv.fuse_prepare && ctx->d.cl.on && ctx->d.own_all && ctx->pair_mask && !noise &&
                    ctx->bonded_nentries > 0 && pv.side != nullptr && niter >= 2 && !con;
  const float* cref = static_cast<const float*>(pv.con_ref);
  if (con) pv.con_pos = pos;
  const BoundaryArgs bargs{gamma, vcoeff, seed, first_step};
  if (pv.use_graph && !noise && !pv.profiling && niter > 0) {
    // One MD step captured once (with and without the energy outputs) and replayed: one graph
    // launch per step, the rebuild kernels inside a conditional node.  Everything that changes
    // between steps lives on the device, so the captured step is valid until an argument or a
    // context buffer changes.
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cs);
    if (cs == cudaStreamCaptureStatusNone) {
      const CtxPriv::StepKey key{pos, vel, forces, masses, vcoeff, dt, gamma, seed, first_step, energies, ke};
      if (!pv.steps_valid || memcmp(&key, &pv.step_key, sizeof(key)) != 0 || memcmp(&ctx->d, &pv.step_state, sizeof(DeviceState)) != 0) {
        for (int k = 0; k < CtxPriv::NGRAPH; ++k) {
          if (pv.exec[k]) cudaGraphExecDestroy(pv.exec[k]);
          if (pv.graph[k]) cudaGraphDestroy(pv.graph[k]);
          pv.exec[k] = nullptr;
          pv.graph[k] = nullptr;
        }
        pv.steps_valid = false;
      }
      // variants: 0 whole step, 1 whole step + energies, 2 first step without its second half-kick,
      // 3 boundary + force call, 4 boundary + force call with energies + second half-kick with the kinetic energy
      auto capture = [&](int k) -> int {
        if (pv.exec[k]) return TMD_OK;
        const bool with_e = (k == 1 || k == 4), opens_with_boundary = (k >= 3), closes = (k != 2 && k != 3);
        const int64_t l0 = ctx->launches, f0 = ctx->force_calls;
        TMD_CUDA(cudaStreamBeginCapture(pv.gstream, cudaStreamCaptureModeRelaxed));
        int rc2 = con ? con_save_ref(ctx, pos, pv.gstream) : TMD_OK;
        if (!rc2) rc2 = enqueue_vv_first(ctx, pos, vel, forces, masses, dt, pv.gstream, !con, opens_with_boundary ? &bargs : nullptr);
        if (!rc2 && con)
          rc2 = con_can_prepare(ctx) ? enqueue_constrain_pos_prepare(ctx, pos, cref, vel, masses, dt, pv.gstream)
                                     : enqueue_constrain_pos(ctx, pos, cref, vel, masses, dt, pv.gstream);
        if (!rc2) rc2 = enqueue_forces(ctx, pos, forces, with_e ? energies : nullptr, pv.gstream);
        if (!rc2 && closes) rc2 = enqueue_vv_second(ctx, vel, forces, masses, dt, gamma, vcoeff, nullptr, seed, first_step,
                                                    with_e && !con ? ke : nullptr, pv.gstream);
        if (!rc2 && closes && con) rc2 = enqueue_constrain_vel(ctx, pos, vel, masses, with_e ? ke : nullptr, pv.gstream);
        pv.fold_pending = false;  // (variants 2 and 3 leave the fold to the graph that follows)
        cudaError_t ce = cudaStreamEndCapture(pv.gstream, &pv.graph[k]);
        if (rc2) return rc2;
        if (ce != cudaSuccess) return fail(TMD_ERR_CUDA, std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce));
        TMD_CUDA(cudaGraphInstantiate(&pv.exec[k], pv.graph[k], 0));
        ++pv.step_captures;
        pv.step_launches[k] = ctx->launches - l0 - pv.last_body_launches;  // (the body runs on rebuild steps only: not counted)
        ctx->launches = l0;  // the capture launched nothing; replays are counted below
        ctx->force_calls = f0;
        return TMD_OK;
      };
      if (fuse) {
        for (int k : {2, 3, 4})
          if ((rc = capture(k))) return rc;
      } else {
        if (niter > 1 && (rc = capture(0))) return rc;
        if ((rc = capture(1))) return rc;
      }
      if (!pv.steps_valid) {
        memset(&pv.step_key, 0, sizeof(pv.step_key));
        pv.step_key = key;
        pv.step_state = ctx->d;
        pv.steps_valid = true;
      }
      TMD_CUDA(cudaEventRecord(pv.ev_in, st));
      TMD_CUDA(cudaStreamWaitEvent(pv.gstream, pv.ev_in, 0));
      for (int it = 0; it < niter; ++it) {
        const int k = fuse ? (it == 0 ? 2 : (it == niter - 1 ? 4 : 3)) : (it == niter - 1 ? 1 : 0);
        TMD_CUDA(cudaGraphLaunch(pv.exec[k], pv.gstream));
        ctx->launches += pv.step_launches[k];
      }
      TMD_CUDA(cudaEventRecord(pv.ev_out, pv.gstream));
      TMD_CUDA(cudaStreamWaitEvent(st, pv.ev_out, 0));
      ctx->force_calls += niter;
      return TMD_OK;
    }
  }
  for (int it = 0; it < niter; ++it) {
    const bool last = (it == niter - 1);
    if (con && (rc = con_save_ref(ctx, pos, st))) return rc;
    if ((rc = enqueue_vv_first(ctx, pos, vel, forces, masses, dt, st, !con, fuse && it > 0 ? &bargs : nullptr))) return rc;
    if (con && (rc = con_can_prepare(ctx) ? enqueue_constrain_pos_prepare(ctx, pos, cref, vel, masses, dt, st)
                                          : enqueue_constrain_pos(ctx, pos, cref, vel, masses, dt, st)))
      return rc;
    if ((rc = enqueue_forces(ctx, pos, forces, last ? energies : nullptr, st))) return rc;
    if (fuse && !last) continue;  // the next iteration's boundary kernel finishes this step
    if ((rc = enqueue_vv_second(ctx, vel, forces, masses, dt, gamma, vcoeff, noise ? noise + it * per_step : nullptr,
                                seed, first_step, last && !con ? ke : nullptr, st)))
      return rc;
    if (con && (rc = enqueue_constrain_vel(ctx, pos, vel, masses, last ? ke : nullptr, st))) return rc;
  }
  return TMD_OK;
}

int tmd_md_steps_host(tmd_ctx* ctx, int niter, float* pos_host, float* vel_host, float* forces_dev,
                      const float* masses_dev, float* pos_dev, float* vel_dev, double dt, double gamma,
                      const float* vcoeff_dev, uint64_t seed, uint64_t first_step, double* energies_host,
                      double* ke_host, tmd_stream stream) {
  if (!ctx || !pos_host || !vel_host || !pos_dev || !vel_dev) return fail(TMD_ERR_ARG, "tmd_md_steps_host: null pointer");
  TMD_PRECISION(ctx, 32, "tmd_md_steps_host")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t bytes = (size_t)ctx->nrep * ctx->natoms * 3 * sizeof(float);
  TMD_CUDA(cudaMemcpyAsync(pos_dev, pos_host, bytes, cudaMemcpyHostToDevice, st));
  TMD_CUDA(cudaMemcpyAsync(vel_dev, vel_host, bytes, cudaMemcpyHostToDevice, st));
  int rc = tmd_md_steps(ctx, niter, pos_dev, vel_dev, forces_dev, masses_dev, dt, gamma, vcoeff_dev, nullptr, seed,
                        first_step, energies_host ? ctx->e_scratch : nullptr, ke_host ? ctx->ke_scratch : nullptr, stream);
  if (rc) return rc;
  TMD_CUDA(cudaMemcpyAsync(pos_host, pos_dev, bytes, cudaMemcpyDeviceToHost, st));
  TMD_CUDA(cudaMemcpyAsync(vel_host, vel_dev, bytes, cudaMemcpyDeviceToHost, st));
  if (energies_host)
    TMD_CUDA(cudaMemcpyAsync(energies_host, ctx->e_scratch, (size_t)ctx->nrep * TMD_NUM_ENERGIES * sizeof(double),
                             cudaMemcpyDeviceToHost, st));
  if (ke_host)
    TMD_CUDA(cudaMemcpyAsync(ke_host, ctx->ke_scratch, (size_t)ctx->nrep * sizeof(double), cudaMemcpyDeviceToHost, st));
  TMD_CUDA(cudaStreamSynchronize(st));
  return TMD_OK;
}

// ---- "precision: double" per-step entry points ---------------------------------------------
int tmd_forces_f64(tmd_ctx* ctx, const double* pos, double* forces, double* energies, tmd_stream stream) {
  if (!ctx || !pos || !forces) return fail(TMD_ERR_ARG, "tmd_forces_f64: null pointer");
  TMD_PRECISION(ctx, 64, "tmd_forces_f64")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (priv(ctx).dirty && (rc = finalize(ctx, st))) return rc;
  return enqueue_forces_f64(ctx, pos, forces, energies, st);
}

static void enqueue_vv_first_f64(tmd_ctx* ctx, double* pos, double* vel, const double* forces, const double* masses, double dt,
                                 cudaStream_t st) {
  launch(k_vv_first_f64, atoms_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, ctx->natoms, ctx->d.counters, pos, vel, forces, masses,
         dt, 0.5 * dt);
}
static void enqueue_vv_second_f64(tmd_ctx* ctx, double* vel, const double* forces, const double* masses, double dt, double gamma,
                                  const double* vcoeff, const double* noise, uint64_t seed, uint64_t step, double* ke,
                                  cudaStream_t st) {
  const bool thermo = (gamma >= 0.0) && vcoeff != nullptr;
  const dim3 g = atoms_grid(ctx, INTEG_THREADS);
  const int n = ctx->natoms;
  const unsigned long long* ctr = ctx->d.counters;
  if (thermo) {
    if (ke) launch(k_vv_second_f64<true, true>, g, INTEG_THREADS, st, n, ctr, vel, forces, masses, dt, 0.5 * dt, -gamma, vcoeff, noise, seed, step, ke);
    else launch(k_vv_second_f64<true, false>, g, INTEG_THREADS, st, n, ctr, vel, forces, masses, dt, 0.5 * dt, -gamma, vcoeff, noise, seed, step, ke);
  } else {
    if (ke) launch(k_vv_second_f64<false, true>, g, INTEG_THREADS, st, n, ctr, vel, forces, masses, dt, 0.5 * dt, -gamma, vcoeff, noise, seed, step, ke);
    else launch(k_vv_second_f64<false, false>, g, INTEG_THREADS, st, n, ctr, vel, forces, masses, dt, 0.5 * dt, -gamma, vcoeff, noise, seed, step, ke);
  }
}

int tmd_vv_first_f64(tmd_ctx* ctx, double* pos, double* vel, const double* forces, const double* masses, double dt,
                     tmd_stream stream) {
  if (!ctx || !pos || !vel || !forces || !masses) return fail(TMD_ERR_ARG, "tmd_vv_first_f64: null pointer");
  TMD_PRECISION(ctx, 64, "tmd_vv_first_f64")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const bool con = has_constraints(ctx);
  int rc;
  if (con && (rc = con_save_ref(ctx, pos, st))) return rc;
  enqueue_vv_first_f64(ctx, pos, vel, forces, masses, dt, st);
  TMD_LAUNCHED(ctx, "k_vv_first_f64");
  if (!con) return TMD_OK;
  priv(ctx).con_pos = pos;
  return enqueue_constrain_pos(ctx, pos, static_cast<const double*>(priv(ctx).con_ref), vel, masses, dt, st);
}

int tmd_vv_second_f64(tmd_ctx* ctx, double* vel, const double* forces, const double* masses, double dt, double gamma,
                      const double* vcoeff, const double* noise, uint64_t seed, uint64_t step_index, double* ke,
                      tmd_stream stream) {
  if (!ctx || !vel || !forces || !masses) return fail(TMD_ERR_ARG, "tmd_vv_second_f64: null pointer");
  TMD_PRECISION(ctx, 64, "tmd_vv_second_f64")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  const bool con = has_constraints(ctx);
  if (con && !priv(ctx).con_pos) return fail(TMD_ERR_STATE, "tmd_vv_second_f64: constraints are set but tmd_vv_first_f64 has not run");
  if (ke && !con) TMD_CUDA(cudaMemsetAsync(ke, 0, (size_t)ctx->nrep * sizeof(double), st));
  enqueue_vv_second_f64(ctx, vel, forces, masses, dt, gamma, vcoeff, noise, seed, step_index, con ? nullptr : ke, st);
  TMD_LAUNCHED(ctx, "k_vv_second_f64");
  if (con) return enqueue_constrain_vel(ctx, static_cast<const double*>(priv(ctx).con_pos), vel, masses, ke, st);
  return TMD_OK;
}

int tmd_kinetic_energy_f64(tmd_ctx* ctx, const double* vel, const double* masses, double* ke, tmd_stream stream) {
  if (!ctx || !vel || !masses || !ke) return fail(TMD_ERR_ARG, "tmd_kinetic_energy_f64: null pointer");
  TMD_PRECISION(ctx, 64, "tmd_kinetic_energy_f64")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  TMD_CUDA(cudaMemsetAsync(ke, 0, (size_t)ctx->nrep * sizeof(double), st));
  launch(k_kinetic_f64, atoms_grid(ctx, INTEG_THREADS), INTEG_THREADS, st, ctx->natoms, vel, masses, ke);
  TMD_LAUNCHED(ctx, "k_kinetic_f64");
  return TMD_OK;
}

int tmd_md_steps_f64(tmd_ctx* ctx, int niter, double* pos, double* vel, double* forces, const double* masses, double dt,
                     double gamma, const double* vcoeff, const double* noise, uint64_t seed, uint64_t first_step,
                     double* energies, double* ke, tmd_stream stream) {
  if (!ctx || !pos || !vel || !forces || !masses || niter < 0) return fail(TMD_ERR_ARG, "tmd_md_steps_f64: bad arguments");
  TMD_PRECISION(ctx, 64, "tmd_md_steps_f64")
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (priv(ctx).dirty && (rc = finalize(ctx, st))) return rc;
  const size_t per_step = (size_t)ctx->nrep * ctx->natoms * 3;
  const bool con = has_constraints(ctx);  // RATTLE: see tmd_md_steps
  const double* cref = static_cast<const double*>(priv(ctx).con_ref);
  if (con) priv(ctx).con_pos = pos;
  for (int it = 0; it < niter; ++it) {
    const bool last = (it == niter - 1);
    if (con && (rc = con_save_ref(ctx, pos, st))) return rc;
    enqueue_vv_first_f64(ctx, pos, vel, forces, masses, dt, st);
    TMD_LAUNCHED(ctx, "k_vv_first_f64");
    if (con && (rc = enqueue_constrain_pos(ctx, pos, cref, vel, masses, dt, st))) return rc;
    if ((rc = enqueue_forces_f64(ctx, pos, forces, last ? energies : nullptr, st))) return rc;
    double* ke2 = last && !con ? ke : nullptr;
    if (ke2) TMD_CUDA(cudaMemsetAsync(ke2, 0, (size_t)ctx->nrep * sizeof(double), st));
    enqueue_vv_second_f64(ctx, vel, forces, masses, dt, gamma, vcoeff, noise ? noise + it * per_step : nullptr, seed, first_step,
                          ke2, st);
    TMD_LAUNCHED(ctx, "k_vv_second_f64");
    if (con && (rc = enqueue_constrain_vel(ctx, pos, vel, masses, last ? ke : nullptr, st))) return rc;
  }
  return TMD_OK;
}

int tmd_export_pairs_f64(tmd_ctx* ctx, const double* pos, int replica, int32_t* pairs, int64_t capacity, int64_t* count,
                         tmd_stream stream) {
  if (!ctx || !pairs || !count || replica < 0 || replica >= ctx->nrep)
    return fail(TMD_ERR_ARG, "tmd_export_pairs_f64: bad arguments");
  TMD_PRECISION(ctx, 64, "tmd_export_pairs_f64")
  if (!ctx->pair_mask) return fail(TMD_ERR_STATE, "tmd_export_pairs_f64: no pair term enabled");
  if (priv(ctx).dirty || ctx->force_calls == 0)
    return fail(TMD_ERR_STATE, "tmd_export_pairs_f64: call tmd_forces_f64 on these positions first");
  (void)pos;
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  TMD_CUDA(cudaMemsetAsync(count, 0, sizeof(int64_t), st));
  launch(k_export_pairs_f64, (ctx->natoms + 3) / 4, 128, st, ctx->d, ctx->d64, replica, pairs, (long long)capacity,
         reinterpret_cast<unsigned long long*>(count));
  TMD_LAUNCHED(ctx, "k_export_pairs_f64");
  return TMD_OK;
}

int tmd_export_pairs(tmd_ctx* ctx, const float* pos, int replica, int32_t* pairs, int64_t capacity,
                     int64_t* count, tmd_stream stream) {
  if (!ctx || !pairs || !count || replica < 0 || replica >= ctx->nrep)
    return fail(TMD_ERR_ARG, "tmd_export_pairs: bad arguments");
  TMD_PRECISION(ctx, 32, "tmd_export_pairs")
  if (!ctx->pair_mask) return fail(TMD_ERR_STATE, "tmd_export_pairs: no pair term enabled");
  if (priv(ctx).dirty || ctx->force_calls == 0)
    return fail(TMD_ERR_STATE, "tmd_export_pairs: call tmd_forces on these positions first");
  (void)pos;
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  TMD_CUDA(cudaMemsetAsync(count, 0, sizeof(int64_t), st));
  if (ctx->d.cl.on)
    launch(k_cexport_pairs, (ctx->d.cl.nclusters_cap + 3) / 4, 128, st, ctx->d, replica, pairs, (long long)capacity,
           reinterpret_cast<unsigned long long*>(count));
  else
    launch(k_export_pairs, (ctx->natoms + 3) / 4, 128, st, ctx->d, replica, pairs, (long long)capacity,
           reinterpret_cast<unsigned long long*>(count));
  TMD_LAUNCHED(ctx, "k_export_pairs");
  return TMD_OK;
}

int tmd_pair_kernel(tmd_ctx* ctx) { return ctx ? ctx->last_pair_kernel : -1; }

int tmd_set_force_convention(tmd_ctx* ctx, int exact_gradient) {
  if (!ctx) return fail(TMD_ERR_ARG, "tmd_set_force_convention: null context");
  ctx->exact_gradient = exact_gradient ? 1 : 0;
  ctx->d.pp.true_gradient = ctx->exact_gradient;  // uniform kernel parameter: takes effect at the next launch
  ctx->d64.pp.true_gradient = ctx->exact_gradient;
  ctx->pair_mode = pair_mode_of(ctx);
  return TMD_OK;
}

int tmd_set_owned_atoms(tmd_ctx* ctx, int first_atom, int count) {
  if (!ctx || first_atom < 0 || count < 0 || first_atom + count > ctx->natoms)
    return fail(TMD_ERR_ARG, "tmd_set_owned_atoms: range outside the system");
  if (ctx->precision == 64) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_owned_atoms: fp64 contexts run the whole system on one GPU");
  if (has_constraints(ctx)) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_owned_atoms: a context with constraints runs the whole system on one GPU");
  if (pme_on(ctx)) return fail(TMD_ERR_UNSUPPORTED, "tmd_set_owned_atoms: a particle-mesh Ewald context runs the whole system on one GPU");
  ctx->d.own_lo = first_atom;
  ctx->d.own_n = count;
  ctx->d.own_all = (first_atom == 0 && count == ctx->natoms) ? 1 : 0;
  if (ctx->d.cl.on) priv(ctx).dirty = true;  // the cluster lists are built for the owned atoms: start over
  return TMD_OK;
}

// ---- constraints ---------------------------------------------------------------------------
int tmd_set_constraints(tmd_ctx* ctx, int nwater, const int32_t* water_idx, const double* water_d, int ncluster,
                        const int32_t* cluster_ptr, const int32_t* cluster_idx, const double* cluster_d) {
  if (!ctx || nwater < 0 || ncluster < 0 || (nwater && (!water_idx || !water_d)) ||
      (ncluster && (!cluster_ptr || !cluster_idx || !cluster_d)))
    return fail(TMD_ERR_ARG, "tmd_set_constraints: bad arguments");
  if (ctx->dd_base || !ctx->d.own_all)
    return fail(TMD_ERR_UNSUPPORTED, "tmd_set_constraints: decomposed runs cannot hold constraints");
  const int N = ctx->natoms;
  std::vector<CGroup> groups;
  groups.reserve((size_t)nwater + ncluster);
  std::vector<char> used(N, 0);
  auto take = [&](int a) { return a >= 0 && a < N && !used[a] ? (used[a] = 1, true) : false; };
  for (int w = 0; w < nwater; ++w) {
    CGroup g{};
    g.na = 3;
    g.nc = 3;
    for (int j = 0; j < 3; ++j) g.atom[j] = water_idx[3 * w + j];
    const int ca[3] = {0, 0, 1}, cb[3] = {1, 2, 2};
    const double d[3] = {water_d[2 * w], water_d[2 * w], water_d[2 * w + 1]};  // O-H, O-H, H-H
    for (int c = 0; c < 3; ++c) {
      g.ca[c] = ca[c];
      g.cb[c] = cb[c];
      g.d[c] = d[c];
      if (!(d[c] > 0.0)) return fail(TMD_ERR_ARG, "tmd_set_constraints: a water distance is not positive");
    }
    for (int j = 0; j < 3; ++j)
      if (!take(g.atom[j])) return fail(TMD_ERR_ARG, "tmd_set_constraints: atom out of range or in two constraint groups");
    groups.push_back(g);
  }
  for (int c = 0; c < ncluster; ++c) {
    const int lo = cluster_ptr[c], hi = cluster_ptr[c + 1];  // cluster_idx[lo]: heavy atom, then its hydrogens
    if (lo < 0 || hi - lo < 2 || hi - lo > CON_MAX_ATOMS)
      return fail(TMD_ERR_ARG, "tmd_set_constraints: a cluster has one heavy atom and 1-4 hydrogens");
    CGroup g{};
    g.na = hi - lo;
    g.nc = g.na - 1;
    for (int j = 0; j < g.na; ++j) {
      g.atom[j] = cluster_idx[lo + j];
      if (!take(g.atom[j])) return fail(TMD_ERR_ARG, "tmd_set_constraints: atom out of range or in two constraint groups");
    }
    for (int k = 0; k < g.nc; ++k) {
      g.ca[k] = 0;
      g.cb[k] = k + 1;
      g.d[k] = cluster_d[lo + k - c];  // one distance per hydrogen: cluster_d is indexed like cluster_idx without the heavy atoms
      if (!(g.d[k] > 0.0)) return fail(TMD_ERR_ARG, "tmd_set_constraints: a cluster distance is not positive");
    }
    groups.push_back(g);
  }
  std::vector<int> free_atoms;
  for (int i = 0; i < N; ++i)
    if (!used[i]) free_atoms.push_back(i);
  DeviceGuard guard(ctx->device);
  CtxPriv& p = priv(ctx);
  p.steps_valid = false;  // the captured steps do not hold the constraint kernels (or hold stale ones)
  p.con_pos = nullptr;
  p.con_ngroups = 0;
  p.con_nfree = 0;
  if (groups.empty()) return TMD_OK;
  int rc;
  if ((rc = upload(&p.con_groups, groups.data(), groups.size()))) return rc;
  if ((rc = upload(&p.con_free, free_atoms.data(), free_atoms.size()))) return rc;
  std::vector<double> L = ctx->have_box ? ctx->box64_host : std::vector<double>((size_t)ctx->nrep * 3, 0.0);
  if ((rc = upload(&p.con_L, L.data(), L.size()))) return rc;
  if (!p.con_ref && (rc = device_alloc(reinterpret_cast<double**>(&p.con_ref), (size_t)ctx->nrep * N * 3))) return rc;
  if (!p.con_fail && (rc = device_alloc(&p.con_fail, 1))) return rc;
  TMD_CUDA(cudaMemset(p.con_fail, 0, sizeof(int)));
  p.con_ngroups = (int)groups.size();
  p.con_nfree = (int)free_atoms.size();
  return TMD_OK;
}

extern "C++" {  // (templates inside the C-linkage block)
template <typename T>
static int constrain_state(tmd_ctx* ctx, T* pos, T* vel, const T* masses, tmd_stream stream, const char* name) {
  if (!ctx || !pos || !masses) return fail(TMD_ERR_ARG, std::string(name) + ": null pointer");
  DeviceGuard guard(ctx->device);
  if (!has_constraints(ctx)) return TMD_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if ((rc = enqueue_constrain_pos(ctx, pos, (const T*)nullptr, (T*)nullptr, masses, 0.0, st))) return rc;
  if (vel && (rc = enqueue_constrain_vel(ctx, (const T*)pos, vel, masses, nullptr, st))) return rc;
  return TMD_OK;
}
}  // extern "C++"
int tmd_constrain(tmd_ctx* ctx, float* pos, float* vel, const float* masses, tmd_stream stream) {
  if (ctx) TMD_PRECISION(ctx, 32, "tmd_constrain")
  return constrain_state(ctx, pos, vel, masses, stream, "tmd_constrain");
}
int tmd_constrain_f64(tmd_ctx* ctx, double* pos, double* vel, const double* masses, tmd_stream stream) {
  if (ctx) TMD_PRECISION(ctx, 64, "tmd_constrain_f64")
  return constrain_state(ctx, pos, vel, masses, stream, "tmd_constrain_f64");
}

// ---- box changes without re-finalising, and the molecule move of the barostat -------------------
extern "C++" {  // (templates inside the C-linkage block)
template <typename T>
static int rescale_box(tmd_ctx* ctx, const T* box_diag, tmd_stream stream, const char* name) {
  if (!ctx || !box_diag) return fail(TMD_ERR_ARG, std::string(name) + ": bad arguments");
  CtxPriv& pv = priv(ctx);
  const int R = ctx->nrep;
  const std::string who = std::string(name) + ": ";
  for (int e = 0; e < R * 3; ++e)
    if (!(box_diag[e] > T(0)) || !((double)box_diag[e] < INFINITY)) return fail(TMD_ERR_ARG, who + "box lengths must be positive and finite");
  if (ctx->dd_base || !ctx->d.own_all) return fail(TMD_ERR_UNSUPPORTED, who + "decomposed and peer-to-peer runs change the box with tmd_set_box");
  if (pv.dirty || !ctx->have_box) return fail(TMD_ERR_UNSUPPORTED, who + "the context is not finalised (a setter ran, or no force call yet)");
  if (!ctx->periodic) return fail(TMD_ERR_UNSUPPORTED, who + "the box is not periodic");
  const bool f64 = ctx->precision == 64;
  std::vector<float> b32(box_diag, box_diag + R * 3);
  std::vector<double> b64(box_diag, box_diag + R * 3);
  float lmin = INFINITY;
  for (int e = 0; e < R * 3; ++e) lmin = std::min(lmin, b32[e]);
  if (f64)
    for (int e = 0; e < R * 3; ++e)
      if (b32[e] > 4096.f) return fail(TMD_ERR_UNSUPPORTED, who + "fp64 contexts take box lengths up to 4096 A");
  const double margin = list_margin(ctx), rl = ctx->cutoff + ctx->skin + margin;
  if (ctx->safe_image && !((ctx->cutoff + 2.0 * ctx->skin + 2.0 * margin) < 0.45 * (double)lmin))
    return fail(TMD_ERR_UNSUPPORTED, who + "the box is too small for the guard-free minimum image the context was set up with");
  double cl_bound = pv.cl_bound;
  if (ctx->d.cl.on) {
    // cl.max_extent is held by value in the captured steps: at the first rescale it becomes the bound of a box 10 %
    // shorter than the one finalised (at least the 8 A the path needs), and every later box must keep it
    const double limit = 0.5 * (double)lmin - rl - ctx->skin - 0.05;
    if (!pv.rescaled) {
      float lmin0 = INFINITY;
      for (const Grid& g : pv.grids)
        for (int k = 0; k < 3; ++k) lmin0 = std::min(lmin0, g.L[k]);
      cl_bound = std::max(8.0, std::min((double)ctx->d.cl.max_extent, 0.5 * 0.9 * (double)lmin0 - rl - ctx->skin - 0.05));
    }
    if (limit < cl_bound) return fail(TMD_ERR_UNSUPPORTED, who + "the box is too small for the cluster lists' extent bound");
  }
  if (pme_on(ctx))
    for (int e = 0; e < R * 3; ++e)
      if (ctx->cutoff > 0.5 * b64[e]) return fail(TMD_ERR_UNSUPPORTED, who + "particle-mesh Ewald needs cutoff <= half of every box length");
  std::vector<Grid> grids(R);
  for (int r = 0; r < R; ++r)
    if (!box_grid(ctx, grids[r], &b32[r * 3], rl, margin, pv.grids[r].n))
      return fail(TMD_ERR_UNSUPPORTED, who + "the cell grid would fall below 2 nsub + 1 cells along an axis");
  // accepted: nothing above changed the context
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  if (ctx->d.cl.on && !pv.rescaled) ctx->d.cl.max_extent = (float)cl_bound;  // (the one recapture)
  pv.cl_bound = cl_bound;
  pv.rescaled = true;
  pv.pme_pinned = pme_on(ctx);
  ctx->box_host = b32;
  ctx->box64_host = b64;
  pv.grids = grids;
  // staging: grids | box lengths (fp64) | PME self + background energies
  const size_t gb = (size_t)R * sizeof(Grid), lb = (size_t)R * 3 * sizeof(double), eb = (size_t)R * sizeof(double);
  if (pv.rs_stage_bytes < gb + lb + eb) {
    if (pv.rs_done) TMD_CUDA(cudaEventSynchronize(pv.rs_done));
    stage_free(pv.rs_stage);
    pv.rs_stage = stage_alloc(gb + lb + eb);
    if (!pv.rs_stage) return fail(TMD_ERR_CUDA, who + "page-locked staging allocation failed");
    pv.rs_stage_bytes = gb + lb + eb;
  }
  if (!pv.rs_done) TMD_CUDA(cudaEventCreateWithFlags(&pv.rs_done, cudaEventDisableTiming));
  TMD_CUDA(cudaEventSynchronize(pv.rs_done));  // the previous rescale's copies have read the staging (done long ago in a run)
  char* sp = static_cast<char*>(pv.rs_stage);
  memcpy(sp, grids.data(), gb);
  memcpy(sp + gb, b64.data(), lb);
  double* ec = reinterpret_cast<double*>(sp + gb + lb);
  for (int r = 0; r < R; ++r) ec[r] = pme_on(ctx) ? pme_econst(pv.pme_alpha, pv.pme_q2, pv.pme_qsum, &b64[3 * r]) : 0.0;
  TMD_CUDA(cudaMemcpyAsync(ctx->d.grid, sp, gb, cudaMemcpyHostToDevice, st));
  for (double* dst : {pv.box_dev, pv.con_L, ctx->L64, pv.pme_L})
    if (dst) TMD_CUDA(cudaMemcpyAsync(dst, sp + gb, lb, cudaMemcpyHostToDevice, st));
  if (pme_on(ctx)) {
    TMD_CUDA(cudaMemcpyAsync(pv.pme_econst, ec, eb, cudaMemcpyHostToDevice, st));
    if (f64) launch_pme_influence<double>(ctx, st);
    else launch_pme_influence<float>(ctx, st);
    TMD_LAUNCHED(ctx, "k_pme_influence");
  }
  TMD_CUDA(cudaEventRecord(pv.rs_done, st));
  // NaN reference positions: the next force call rebuilds the lists (both pair paths, fp64 included)
  TMD_CUDA(cudaMemsetAsync(ctx->d.pos_ref, 0xFF, (size_t)R * ctx->natoms * sizeof(float4), st));
  return TMD_OK;
}

template <typename T>
static int scale_molecules(tmd_ctx* ctx, T* pos, const double* scale, tmd_stream stream, const char* name) {
  if (!ctx || !pos || !scale) return fail(TMD_ERR_ARG, std::string(name) + ": null pointer");
  CtxPriv& pv = priv(ctx);
  if (pv.mol_n == 0) return fail(TMD_ERR_STATE, std::string(name) + ": call tmd_set_molecules first");
  if (!pv.box_dev || !ctx->periodic) return fail(TMD_ERR_STATE, std::string(name) + ": needs a finalised context with a periodic box");
  DeviceGuard guard(ctx->device);
  const MolTables m{pv.mol_n, ctx->natoms, pv.mol_ptr, pv.mol_atoms, pv.mol_parent, pv.mol_u};
  launch(k_scale_molecules<T>, dim3((pv.mol_n + MOL_THREADS - 1) / MOL_THREADS, ctx->nrep), MOL_THREADS, (cudaStream_t)stream, m, pos,
         scale, (const double*)pv.box_dev);
  TMD_LAUNCHED(ctx, "k_scale_molecules");
  return TMD_OK;
}
}  // extern "C++"

int tmd_rescale_box(tmd_ctx* ctx, const float* box_diag, tmd_stream stream) {
  if (ctx) TMD_PRECISION(ctx, 32, "tmd_rescale_box")
  return rescale_box(ctx, box_diag, stream, "tmd_rescale_box");
}
int tmd_rescale_box_f64(tmd_ctx* ctx, const double* box_diag, tmd_stream stream) {
  if (ctx) TMD_PRECISION(ctx, 64, "tmd_rescale_box_f64")
  return rescale_box(ctx, box_diag, stream, "tmd_rescale_box_f64");
}
int64_t tmd_step_captures(tmd_ctx* ctx) { return ctx ? priv(ctx).step_captures : -1; }

int tmd_set_molecules(tmd_ctx* ctx, int nmol, const int32_t* ptr, const int32_t* atoms, const int32_t* parent) {
  if (!ctx || nmol < 0 || (nmol > 0 && (!ptr || !atoms || !parent))) return fail(TMD_ERR_ARG, "tmd_set_molecules: bad arguments");
  const int N = ctx->natoms;
  if (nmol > 0) {
    if (ptr[0] != 0 || ptr[nmol] != N) return fail(TMD_ERR_ARG, "tmd_set_molecules: the molecules must hold every atom once");
    std::vector<int> pos_of(N, -1);
    for (int m = 0; m < nmol; ++m) {
      if (ptr[m + 1] <= ptr[m]) return fail(TMD_ERR_ARG, "tmd_set_molecules: empty molecule");
      for (int k = ptr[m]; k < ptr[m + 1]; ++k) {
        const int a = atoms[k], p = parent[k];
        if (a < 0 || a >= N || pos_of[a] >= 0) return fail(TMD_ERR_ARG, "tmd_set_molecules: the molecules must hold every atom once");
        pos_of[a] = k;
        const bool root = k == ptr[m];
        // the parent comes earlier in the same molecule (breadth-first order); the first atom is its own
        if (root ? p != a : (p < 0 || p >= N || pos_of[p] < ptr[m] || pos_of[p] >= k))
          return fail(TMD_ERR_ARG, "tmd_set_molecules: parent of atom " + std::to_string(a) + " is not an earlier atom of its molecule");
      }
    }
  }
  DeviceGuard guard(ctx->device);
  CtxPriv& pv = priv(ctx);
  pv.mol_n = 0;
  if (nmol == 0) return TMD_OK;
  int rc;
  if ((rc = upload(&pv.mol_ptr, ptr, (size_t)nmol + 1))) return rc;
  if ((rc = upload(&pv.mol_atoms, atoms, (size_t)N))) return rc;
  if ((rc = upload(&pv.mol_parent, parent, (size_t)N))) return rc;
  if (!pv.mol_u && (rc = device_alloc(&pv.mol_u, (size_t)ctx->nrep * N * 3))) return rc;
  pv.mol_n = nmol;
  return TMD_OK;
}
int tmd_scale_molecules(tmd_ctx* ctx, float* pos, const double* scale, tmd_stream stream) {
  if (ctx) TMD_PRECISION(ctx, 32, "tmd_scale_molecules")
  return scale_molecules(ctx, pos, scale, stream, "tmd_scale_molecules");
}
int tmd_scale_molecules_f64(tmd_ctx* ctx, double* pos, const double* scale, tmd_stream stream) {
  if (ctx) TMD_PRECISION(ctx, 64, "tmd_scale_molecules_f64")
  return scale_molecules(ctx, pos, scale, stream, "tmd_scale_molecules_f64");
}

// ---- peer-to-peer position exchange (helpers above, next to priv()) ------------------------
int tmd_dd_create(tmd_ctx* ctx, int rank, int world, unsigned char* handle_out) {
  if (!ctx || !handle_out || world < 1 || world > TMD_MAX_PEERS || rank < 0 || rank >= world)
    return fail(TMD_ERR_ARG, "tmd_dd_create: bad arguments (at most 16 ranks)");
  if (ctx->precision == 64) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_create: fp64 contexts run the whole system on one GPU");
  if (has_constraints(ctx)) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_create: a context with constraints runs the whole system on one GPU");
  if (pme_on(ctx)) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_create: a particle-mesh Ewald context runs the whole system on one GPU");
  if (ctx->nrep != 1) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_create: decomposed runs take one replica");
  static_assert(sizeof(cudaIpcMemHandle_t) == TMD_IPC_HANDLE_BYTES, "IPC handle size");
  DeviceGuard guard(ctx->device);
  dd_release(ctx);
  ctx->dd_pos_bytes = (((size_t)ctx->natoms * 3 * sizeof(float)) + 255) / 256 * 256;
  const size_t bytes = 2 * ctx->dd_pos_bytes + 256 /* flags */ + 256 /* sync */;
  TMD_CUDA(cudaMalloc(&ctx->dd_base, bytes));
  TMD_CUDA(cudaMemset(ctx->dd_base, 0, bytes));
  TMD_CUDA(cudaDeviceSynchronize());
  ctx->dd_rank = rank;
  ctx->dd_world = world;
  ctx->dd_peer_base[rank] = ctx->dd_base;
  ctx->dd_sync = reinterpret_cast<unsigned*>(static_cast<char*>(ctx->dd_base) + 2 * ctx->dd_pos_bytes + 256);
  cudaIpcMemHandle_t h;
  memset(&h, 0, sizeof(h));
  if (world > 1) TMD_CUDA(cudaIpcGetMemHandle(&h, ctx->dd_base));
  memcpy(handle_out, &h, sizeof(h));
  return TMD_OK;
}

int tmd_dd_connect(tmd_ctx* ctx, const unsigned char* handles) {
  if (!ctx || !handles) return fail(TMD_ERR_ARG, "tmd_dd_connect: null pointer");
  if (ctx->precision == 64) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_connect: fp64 contexts run the whole system on one GPU");
  if (has_constraints(ctx)) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_connect: a context with constraints runs the whole system on one GPU");
  if (pme_on(ctx)) return fail(TMD_ERR_UNSUPPORTED, "tmd_dd_connect: a particle-mesh Ewald context runs the whole system on one GPU");
  if (!ctx->dd_base) return fail(TMD_ERR_STATE, "tmd_dd_connect: tmd_dd_create has not been called");
  DeviceGuard guard(ctx->device);
  for (int p = 0; p < ctx->dd_world; ++p) {
    if (p == ctx->dd_rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)p * TMD_IPC_HANDLE_BYTES, sizeof(h));
    void* ptr = nullptr;
    TMD_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    ctx->dd_peer_base[p] = ptr;
  }
  ctx->dd_connected = true;
  return TMD_OK;
}

#define TMD_DD_READY(name)                                                                     \
  if (!ctx) return fail(TMD_ERR_ARG, name ": null context");                                   \
  if (ctx->precision == 64) return fail(TMD_ERR_UNSUPPORTED, name ": fp64 contexts run the whole system on one GPU"); \
  if (has_constraints(ctx)) return fail(TMD_ERR_UNSUPPORTED, name ": a context with constraints runs the whole system on one GPU"); \
  if (pme_on(ctx)) return fail(TMD_ERR_UNSUPPORTED, name ": a particle-mesh Ewald context runs the whole system on one GPU"); \
  if (!ctx->dd_connected) return fail(TMD_ERR_STATE, name ": tmd_dd_create / tmd_dd_connect first"); \
  DeviceGuard guard(ctx->device);

int tmd_dd_load(tmd_ctx* ctx, int which, const float* pos, tmd_stream stream) {
  TMD_DD_READY("tmd_dd_load")
  if (!pos || (which != 0 && which != 1)) return fail(TMD_ERR_ARG, "tmd_dd_load: bad arguments");
  TMD_CUDA(cudaMemcpyAsync(dd_pos_of(ctx, ctx->dd_rank, which), pos, (size_t)ctx->natoms * 3 * sizeof(float),
                           cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return TMD_OK;
}

int tmd_dd_store(tmd_ctx* ctx, int which, float* pos, tmd_stream stream) {
  TMD_DD_READY("tmd_dd_store")
  if (!pos || (which != 0 && which != 1)) return fail(TMD_ERR_ARG, "tmd_dd_store: bad arguments");
  TMD_CUDA(cudaMemcpyAsync(pos, dd_pos_of(ctx, ctx->dd_rank, which), (size_t)ctx->natoms * 3 * sizeof(float),
                           cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return TMD_OK;
}

int tmd_dd_vv_first_push(tmd_ctx* ctx, int which_in, float* vel, const float* forces, const float* masses, double dt,
                         tmd_stream stream) {
  TMD_DD_READY("tmd_dd_vv_first_push")
  if (!vel || !forces || !masses || (which_in != 0 && which_in != 1))
    return fail(TMD_ERR_ARG, "tmd_dd_vv_first_push: bad arguments");
  PeerTable pt;
  memset(&pt, 0, sizeof(pt));
  pt.world = ctx->dd_world;
  pt.rank = ctx->dd_rank;
  for (int p = 0; p < ctx->dd_world; ++p) {
    pt.pos[p] = dd_pos_of(ctx, p, 1 - which_in);
    pt.flags[p] = dd_flags_of(ctx, p);
  }
  const unsigned blocks = (unsigned)((std::max(ctx->d.own_n, 1) + INTEG_THREADS - 1) / INTEG_THREADS);
  launch(k_vv_first_push, blocks, INTEG_THREADS, (cudaStream_t)stream, 
      ctx->natoms, ctx->d.own_lo, ctx->d.own_n, ctx->d.counters, dd_pos_of(ctx, ctx->dd_rank, which_in), vel, forces,
      masses, (float)dt, (float)(0.5 * dt), pt, ctx->dd_sync);
  TMD_LAUNCHED(ctx, "k_vv_first_push");
  return TMD_OK;
}

int tmd_dd_wait(tmd_ctx* ctx, tmd_stream stream) {
  TMD_DD_READY("tmd_dd_wait")
  launch(k_wait_peers, 1, 32, (cudaStream_t)stream, dd_flags_of(ctx, ctx->dd_rank), ctx->dd_sync, ctx->dd_world,
                                                    ctx->d.flags + F_PEERWAIT);
  TMD_LAUNCHED(ctx, "k_wait_peers");
  return TMD_OK;
}

int tmd_dd_forces(tmd_ctx* ctx, int which, float* forces, double* energies, tmd_stream stream) {
  TMD_DD_READY("tmd_dd_forces")
  if (which != 0 && which != 1) return fail(TMD_ERR_ARG, "tmd_dd_forces: bad arguments");
  return tmd_forces(ctx, dd_pos_of(ctx, ctx->dd_rank, which), forces, energies, stream);
}

// ---- Wrapper.wrap ---------------------------------------------------------------------------
int tmd_wrapper_create(tmd_wrapper** out, int device, int natoms, int ngroups, const int32_t* group_ptr,
                       const int32_t* group_atoms) {
  if (!out || natoms <= 0 || ngroups < 0 || !group_ptr || (ngroups > 0 && !group_atoms))
    return fail(TMD_ERR_ARG, "tmd_wrapper_create: bad arguments");
  if (group_ptr[0] != 0) return fail(TMD_ERR_ARG, "tmd_wrapper_create: group_ptr[0] must be 0");
  for (int g = 0; g < ngroups; ++g)
    if (group_ptr[g + 1] < group_ptr[g]) return fail(TMD_ERR_ARG, "tmd_wrapper_create: group_ptr must not decrease");
  const int total = group_ptr[ngroups];
  if (total > natoms) return fail(TMD_ERR_ARG, "tmd_wrapper_create: more group members than atoms");
  std::vector<char> seen((size_t)natoms, 0);
  for (int e = 0; e < total; ++e) {
    const int a = group_atoms[e];
    if (a < 0 || a >= natoms || seen[a]) return fail(TMD_ERR_ARG, "tmd_wrapper_create: atom index out of range or in two groups");
    seen[a] = 1;
  }
  int ndev = 0;
  TMD_CUDA(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(TMD_ERR_ARG, "tmd_wrapper_create: no such CUDA device");
  DeviceGuard guard(device);
  tmd_wrapper* w = new tmd_wrapper();
  w->device = device;
  w->natoms = natoms;
  w->ngroups = ngroups;
  int rc;
  if ((rc = upload(&w->group_ptr, group_ptr, (size_t)ngroups + 1)) || (rc = upload(&w->group_atoms, group_atoms, (size_t)total)) ||
      (rc = device_alloc(&w->flag, (size_t)1))) {
    tmd_wrapper_destroy(w);
    return rc;
  }
  *out = w;
  return TMD_OK;
}

extern "C++" {  // (templates inside the C-linkage block)
template <typename T>
static int wrapper_wrap(tmd_wrapper* w, T* pos, const T* box, int nrep, tmd_stream stream) {
  if (!w || !pos || !box || nrep <= 0 || nrep > 65535) return fail(TMD_ERR_ARG, "tmd_wrapper_wrap: bad arguments");
  if (w->ngroups == 0) return TMD_OK;
  DeviceGuard guard(w->device);
  cudaStream_t st = (cudaStream_t)stream;
  launch(k_wrap_boxflag<T>, 1, 256, st, box, nrep, w->flag);
  launch(k_wrap<T>, dim3((unsigned)((w->ngroups + WRAP_WARPS - 1) / WRAP_WARPS), (unsigned)nrep), WRAP_WARPS * 32, st, 
      w->natoms, w->ngroups, w->group_ptr, w->group_atoms, pos, box, w->flag);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(TMD_ERR_CUDA, std::string("launch k_wrap: ") + cudaGetErrorString(e));
  return TMD_OK;
}
}  // extern "C++"
int tmd_wrapper_wrap(tmd_wrapper* w, float* pos, const float* box, int nrep, tmd_stream stream) {
  return wrapper_wrap(w, pos, box, nrep, stream);
}
int tmd_wrapper_wrap_f64(tmd_wrapper* w, double* pos, const double* box, int nrep, tmd_stream stream) {
  return wrapper_wrap(w, pos, box, nrep, stream);
}

int tmd_wrapper_destroy(tmd_wrapper* w) {
  if (!w) return TMD_OK;
  DeviceGuard guard(w->device);
  if (w->group_ptr) cudaFree(w->group_ptr);
  if (w->group_atoms) cudaFree(w->group_atoms);
  if (w->flag) cudaFree(w->flag);
  delete w;
  return TMD_OK;
}

int tmd_profile_begin(tmd_ctx* ctx, int max_samples) {
  if (!ctx || max_samples <= 0) return fail(TMD_ERR_ARG, "tmd_profile_begin: bad arguments");
  DeviceGuard guard(ctx->device);
  CtxPriv& pv = priv(ctx);
  while ((int)pv.ev.size() < 2 * max_samples) {
    cudaEvent_t e;
    TMD_CUDA(cudaEventCreate(&e));
    pv.ev.push_back(e);
  }
  pv.ev_used = 0;
  pv.profiling = true;
  return TMD_OK;
}

int tmd_profile_end(tmd_ctx* ctx, double* total_ms, int* nsamples, tmd_stream stream) {
  if (!ctx || !total_ms || !nsamples) return fail(TMD_ERR_ARG, "tmd_profile_end: bad arguments");
  DeviceGuard guard(ctx->device);
  CtxPriv& pv = priv(ctx);
  pv.profiling = false;
  TMD_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  double tot = 0.0;
  for (int k = 0; k + 1 < pv.ev_used; k += 2) {
    float ms = 0.f;
    TMD_CUDA(cudaEventElapsedTime(&ms, pv.ev[k], pv.ev[k + 1]));
    tot += ms;
  }
  *total_ms = tot;
  *nsamples = pv.ev_used / 2;
  pv.ev_used = 0;
  return TMD_OK;
}

int tmd_get_stats(tmd_ctx* ctx, tmd_stats* out, tmd_stream stream) {
  if (!ctx || !out) return fail(TMD_ERR_ARG, "tmd_get_stats: null pointer");
  DeviceGuard guard(ctx->device);
  cudaStream_t st = (cudaStream_t)stream;
  TMD_CUDA(cudaStreamSynchronize(st));
  memset(out, 0, sizeof(*out));
  out->force_calls = ctx->force_calls;
  out->kernel_launches = ctx->launches;
  out->row_capacity = ctx->d.row_cap;
  out->rebuilds = ctx->rebuilds_before;
  // a constraint group without a solution since the last check: reported after the list checks below, whose
  // overflow makes the caller run the steps again (a truncated force can be what broke the constraint)
  int con_failed = 0;
  if (priv(ctx).con_fail) {
    TMD_CUDA(cudaMemcpy(&con_failed, priv(ctx).con_fail, sizeof(int), cudaMemcpyDeviceToHost));
    if (con_failed) TMD_CUDA(cudaMemset(priv(ctx).con_fail, 0, sizeof(int)));
  }
  auto con_error = [&]() {
    return con_failed ? fail(TMD_ERR_STATE, "a constraint group has no solution (SETTLE) or SHAKE did not converge: the "
                                            "time step is too long or the system blew up")
                      : TMD_OK;
  };
  if (priv(ctx).dirty || !ctx->d.flags) return con_error();
  std::vector<int> fl((size_t)ctx->nrep * F_COUNT);
  TMD_CUDA(cudaMemcpy(fl.data(), ctx->d.flags, fl.size() * sizeof(int), cudaMemcpyDeviceToHost));
  Grid g0;
  TMD_CUDA(cudaMemcpy(&g0, ctx->d.grid, sizeof(Grid), cudaMemcpyDeviceToHost));
  for (int k = 0; k < 3; ++k) out->ncells[k] = g0.n[k];
  bool overflow = false;
  for (int r = 0; r < ctx->nrep; ++r) {
    out->rebuilds += fl[r * F_COUNT + F_NREBUILD];
    out->max_neighbours = std::max(out->max_neighbours, fl[r * F_COUNT + F_MAXNBR]);
    overflow |= fl[r * F_COUNT + F_OVERFLOW] != 0;
  }
  out->overflow = overflow;
  if (fl[F_PEERWAIT])
    return fail(TMD_ERR_STATE, "the wait for the other ranks' position stores timed out (a rank stopped or the "
                               "ranks ran different numbers of steps): the decomposed run is invalid");
  for (int r = 0; r < ctx->nrep; ++r)
    if (fl[r * F_COUNT + F_FARPOS])
      return fail(TMD_ERR_UNSUPPORTED,
                  ctx->precision == 64
                      ? "a position is 8192 A or more from the origin (fp64 contexts), or not finite: wrap the coordinates "
                        "(torchmd Wrapper) -- results since the last check are not reliable"
                      : "a position is more than 2000 box lengths from the origin: wrap the coordinates "
                        "(torchmd Wrapper) -- results since the last check are not reliable");
  if (ctx->cluster_failed && ctx->force_calls >= ctx->cluster_retry_at && !priv(ctx).dirty) {
    ctx->cluster_failed = false;  // try the cluster lists again from the next force call on
    priv(ctx).dirty = true;
  }
  if (ctx->d.cl.on) {
    int maxa = 0, maxb = 0;
    bool clfail = false;
    for (int r = 0; r < ctx->nrep; ++r) {
      maxa = std::max(maxa, fl[r * F_COUNT + F_CLMAXA]);
      maxb = std::max(maxb, fl[r * F_COUNT + F_CLMAXB]);
      clfail |= fl[r * F_COUNT + F_CLFAIL] != 0;
    }
    if (getenv("TMD_B200_DEBUG")) {
      fprintf(stderr, "[tmd] cluster flags:");
      for (int k = 0; k < F_COUNT; ++k) fprintf(stderr, " %d", fl[k]);
      fprintf(stderr, "  (slots %d, ecap %d, mcap %d)\n", ctx->d.cl.slots, ctx->d.cl.ecap, ctx->d.cl.mcap);
    }
    if (clfail) {
      // a cluster too long for the box (a lattice start, a void), or an exclusion set / segment table / cell bucket
      // overflow: this context continues on the full Verlet rows -- and tries the cluster lists again later (a lattice
      // start has melted by then), with the waiting time doubling at every failure
      ctx->cluster_failed = true;
      ctx->cluster_retry_after = std::min<int64_t>(std::max<int64_t>(2 * ctx->cluster_retry_after, 1000), 1 << 20);
      ctx->cluster_retry_at = ctx->force_calls + ctx->cluster_retry_after;
      priv(ctx).dirty = true;
      return fail(TMD_ERR_OVERFLOW, "cluster lists do not fit this system; switched to full neighbour rows, recompute required");
    }
    if (overflow) {
      if (maxb > ctx->d.cl.ecap) ctx->d.cl.ecap = (int)(((long long)(maxb * 1.25) + 32 + 31) / 32 * 32);
      if (maxa > ctx->d.cl.mcap) ctx->d.cl.mcap = (int)(((long long)(maxa * 1.25) + 32 + 31) / 32 * 32);
      priv(ctx).dirty = true;
      return fail(TMD_ERR_OVERFLOW, "cluster list capacity exceeded; capacity grown, recompute required");
    }
    return con_error();
  }
  if (overflow) {
    // grow the rows, invalidate the list; the caller recomputes (standalone force call)
    // or reports the run as invalid (fused multi-step call)
    ctx->d.row_cap = (int)((((long long)(out->max_neighbours * 1.25) + 32 + 63) / 64) * 64);
    priv(ctx).dirty = true;
    return fail(TMD_ERR_OVERFLOW, "neighbour row capacity exceeded; capacity grown, recompute required");
  }
  return con_error();
}

}  // extern "C"
