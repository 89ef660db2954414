/*
 * tmd_b200.h -- C ABI of the H100-native MD inner loop that sits behind
 * torchmd's Forces.compute() / Integrator.step().
 *
 * The reference (torchmd/torchmd) has no FFI: its hot path is stock torch ops
 * issued from Python.  Each entry point below therefore names the reference
 * Python it replaces (paths relative to the reference checkout), and
 * INTEGRATION.md shows the ctypes binding a maintainer would add there.
 *
 * Conventions
 *   - every function returns 0 on success, a negative TMD_ERR_* otherwise;
 *     tmd_last_error() gives the message (thread-local).  Nothing aborts.
 *   - "dev" pointers are CUDA device pointers owned by the caller (PyTorch
 *     tensors: fp32, contiguous).  "host" pointers are ordinary host memory,
 *     read during the call only (topology is copied into the context).
 *   - per-step calls only ENQUEUE work on the given CUDA stream: no
 *     allocation, no synchronisation, CUDA-graph capturable.  Calls marked
 *     [sync] synchronise the stream and may (re)allocate context scratch.
 *   - a context belongs to one device and is not thread-safe.
 *   - arithmetic is fp32 ("precision: single" in torchmd) by default, energies
 *     are accumulated and returned in fp64.  A context set to 64 bits
 *     (tmd_set_precision) runs "precision: double": fp64 state, parameters and
 *     arithmetic through the *_f64 entry points, full neighbour rows, one GPU.
 */
#ifndef TMD_B200_H
#define TMD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tmd_ctx tmd_ctx;
typedef void* tmd_stream; /* cudaStream_t */

enum {
  TMD_OK = 0,
  TMD_ERR_ARG = -1,      /* bad argument */
  TMD_ERR_CUDA = -2,     /* CUDA runtime error (message has the string) */
  TMD_ERR_STATE = -3,    /* call order / missing setup */
  TMD_ERR_OVERFLOW = -4, /* neighbour rows overflowed their capacity */
  TMD_ERR_UNSUPPORTED = -5
};

/* Energy slots, in the order of torchmd Forces.terms (forces.py:23-25). */
enum {
  TMD_E_BONDS = 0,
  TMD_E_ANGLES = 1,
  TMD_E_DIHEDRALS = 2,
  TMD_E_IMPROPERS = 3,
  TMD_E_14 = 4, /* stays 0: 1-4 energies are booked under lj/electrostatics, forces.py:185-236 */
  TMD_E_ELECTROSTATICS = 5,
  TMD_E_LJ = 6,
  TMD_E_REPULSION = 7,
  TMD_E_REPULSIONCG = 8,
  TMD_NUM_ENERGIES = 9
};

/* Term bit mask (1 << energy slot). */
#define TMD_TERM(slot) (1u << (slot))

const char* tmd_last_error(void);
int tmd_version(void);

/* ---- lifetime ------------------------------------------------------------ */

/* One context per (device, system).  Replaces nothing in the reference; it is
 * the state Forces.__init__ (forces.py:27-74) keeps in Python attributes. */
int tmd_create(tmd_ctx** out, int device, int natoms, int nreplicas);
int tmd_destroy(tmd_ctx* ctx);

/* ---- topology / parameters: host pointers, copied; once per run ----------- */

/* Per-atom charge and atom-type id, and the LJ A/B type tables
 * (Parameters.charges, .mapped_atom_types, .A, .B; parameters.py:449-457).
 * A and B may be NULL when no LJ/repulsion term is used. */
int tmd_set_atoms(tmd_ctx* ctx, const float* charges_host, const int32_t* types_host,
                  int ntypes, const float* A_host, const float* B_host);

/* Symmetric exclusion adjacency in CSR form (row_ptr has natoms+1 entries).
 * Replaces the N x N bool matrix of Forces._make_indeces (forces.py:348-357). */
int tmd_set_exclusions(tmd_ctx* ctx, const int64_t* row_ptr_host, const int32_t* cols_host);

/* Non-bonded set-up: which pair terms, cutoff (< 0: none), switch distance
 * (< 0: none), reaction field, solvent dielectric, Coulomb constant
 * (forces.py:375-378) and Verlet skin.  Arguments of Forces.__init__. */
int tmd_set_nonbonded(tmd_ctx* ctx, uint32_t term_mask, double cutoff, double switch_dist,
                      int rfa, double solvent_dielectric, double coulomb_constant, double skin);

/* Bonded terms, one parameter row per term instance (the reference's
 * params[map[:,1]] gather, forces.py:122-258, done once here).
 *   bonds    idx (n,2)  prm (n,2) = k, r0
 *   angles   idx (n,3)  prm (n,2) = k, theta0 [rad]
 *   torsions idx (n,4)  term_ptr (n+1) into terms (nterms,3) = k, phi0 [rad], periodicity
 *            which = 0 proper dihedrals, 1 impropers; amber_form = all(per>0) (forces.py:566)
 *   pairs14  idx (n,2)  prm (n,4) = A, B, scnb, scee */
int tmd_set_bonds(tmd_ctx* ctx, int n, const int32_t* idx_host, const float* prm_host);
int tmd_set_angles(tmd_ctx* ctx, int n, const int32_t* idx_host, const float* prm_host);
int tmd_set_torsions(tmd_ctx* ctx, int which, int n, const int32_t* idx_host,
                     const int32_t* term_ptr_host, const float* terms_host, int amber_form);
int tmd_set_pairs14(tmd_ctx* ctx, int n, const int32_t* idx_host, const float* prm_host);

/* Box diagonal per replica, host (nreplicas,3).  All zeros = no periodic
 * wrapping (forces.py:361).  Sizes the cell grid; call again if the box changes. [sync] */
int tmd_set_box(tmd_ctx* ctx, const float* box_diag_host);

/* ---- per-step work: device pointers, enqueue only -------------------------- */

/* Forces.compute(pos, box, forces) explicit-force path (forces.py:83-346):
 * overwrites forces_dev (R,N,3) and, if energies_dev != NULL, writes
 * (R, TMD_NUM_ENERGIES) doubles.  Internally: displacement check, (gated)
 * cell-list + neighbour-list rebuild, non-bonded pair kernel, bonded kernels. */
int tmd_forces(tmd_ctx* ctx, const float* pos_dev, float* forces_dev, double* energies_dev,
               tmd_stream stream);

/* _first_VV (integrator.py:61-64): pos += v dt + 0.5 (F/m) dt^2 ; v += 0.5 dt F/m */
int tmd_vv_first(tmd_ctx* ctx, float* pos_dev, float* vel_dev, const float* forces_dev,
                 const float* masses_dev, double dt, tmd_stream stream);

/* langevin (integrator.py:72-74) followed by _second_VV (integrator.py:67-69).
 * gamma < 0 or vcoeff_dev == NULL: no thermostat.  noise_dev (R,N,3) N(0,1)
 * draws, or NULL to draw in-kernel from Philox4x32-10(seed, step_index + number of
 * tmd_vv_first calls on this context so far -- the count lives on the device so a
 * captured CUDA graph of one step can be replayed).
 * ke_dev != NULL: also write the kinetic energy per replica (R doubles)
 * (kinetic_energy, integrator.py:8-30). */
int tmd_vv_second(tmd_ctx* ctx, float* vel_dev, const float* forces_dev, const float* masses_dev,
                  double dt, double gamma, const float* vcoeff_dev, const float* noise_dev,
                  uint64_t seed, uint64_t step_index, double* ke_dev, tmd_stream stream);

/* kinetic_energy (integrator.py:8-30) on its own. */
int tmd_kinetic_energy(tmd_ctx* ctx, const float* vel_dev, const float* masses_dev, double* ke_dev,
                       tmd_stream stream);

/* niter iterations of Integrator.step's loop body (integrator.py:115-120) with
 * no host round trip; energies/ke are those of the LAST iteration, which is all
 * Integrator.step returns (integrator.py:122-125).  noise_dev: (niter,R,N,3) or NULL. */
int tmd_md_steps(tmd_ctx* ctx, int niter, float* pos_dev, float* vel_dev, float* forces_dev,
                 const float* masses_dev, double dt, double gamma, const float* vcoeff_dev,
                 const float* noise_dev, uint64_t seed, uint64_t first_step_index,
                 double* energies_dev, double* ke_dev, tmd_stream stream);

/* Same as tmd_md_steps but with HOST state: copies pos/vel (R,N,3) in, runs,
 * copies pos/vel/energies/ke out and synchronises.  The end-to-end entry a
 * host-resident caller (e.g. minimizers.py:19-32 style) would use. [sync] */
int tmd_md_steps_host(tmd_ctx* ctx, int niter, float* pos_host, float* vel_host,
                      float* forces_dev, const float* masses_dev, float* pos_dev, float* vel_dev,
                      double dt, double gamma, const float* vcoeff_dev, uint64_t seed,
                      uint64_t first_step_index, double* energies_host, double* ke_host,
                      tmd_stream stream);

/* Which force the switched LJ term returns.  0 (default): the reference's explicit formula
 * s*dE/dr + E*s'/r with its extra 1/r (forces.py:410-412), what Forces.compute returns with
 * explicit_forces=True.  1: the exact derivative d(E*s)/dr = s*dE/dr + E*s', what the
 * reference obtains by autograd with explicit_forces=False (forces.py:328-336).  Every other
 * term's explicit force already is its exact gradient.  Takes effect at the next call. */
int tmd_set_force_convention(tmd_ctx* ctx, int exact_gradient);

/* ---- decomposed runs (one context per rank, every rank holds all positions) --------- */

/* Restrict the FORCE and INTEGRATION work of this context to the atoms
 * [first_atom, first_atom+count) (original indices): tmd_forces fills forces only for
 * them (their complete force: every partner is visible locally), tmd_vv_first /
 * tmd_vv_second / tmd_kinetic_energy update only them, energies are this rank's share
 * (sum over ranks = total).  The caller exchanges positions between tmd_vv_first and
 * tmd_forces (one all-gather per step).  Default: all atoms.  No reference counterpart
 * (the reference is single-device). */
int tmd_set_owned_atoms(tmd_ctx* ctx, int first_atom, int count);

/* ---- decomposed runs: integrate + position exchange over NVLink peer memory ------------
 *
 * Instead of a collective between tmd_vv_first and tmd_forces, the integration kernel of
 * every rank stores the new positions of its owned atoms straight into the position
 * buffers of ALL ranks (peer-to-peer stores through NVLink / NVSwitch), then raises a flag
 * in every rank's flag array; a one-warp kernel on each rank waits until all flags of the
 * step have arrived.  One launch + one tiny wait per step, no library collective on the
 * path.  Positions live in two buffers per rank (read buffer / write buffer alternate each
 * step) allocated by the context and shared between the processes of one node through CUDA
 * IPC.  Single replica.  No reference counterpart (SURVEY.md section 8e).
 *
 * Set-up, once: every rank calls tmd_dd_create (after tmd_set_owned_atoms), all-gathers the
 * 64-byte handles with whatever transport it has (torch.distributed), then tmd_dd_connect.
 * Per step, parity p = 0,1,0,...:  tmd_dd_vv_first_push(p)  tmd_dd_wait  tmd_dd_forces(1-p)
 * tmd_vv_second.  All four only enqueue; every per-step counter is device resident, so a
 * captured CUDA graph of a step of given parity can be replayed. */
#define TMD_MAX_PEERS 16
#define TMD_IPC_HANDLE_BYTES 64

/* Allocates the two position buffers and the flag array of this rank; handle_out receives
 * TMD_IPC_HANDLE_BYTES bytes to be sent to the other ranks. [sync] */
int tmd_dd_create(tmd_ctx* ctx, int rank, int world, unsigned char* handle_out_host);
/* handles_host: world * TMD_IPC_HANDLE_BYTES bytes, rank order (own entry ignored).  Opens the
 * peers' buffers in this process. [sync] */
int tmd_dd_connect(tmd_ctx* ctx, const unsigned char* handles_host);
/* Copy caller positions (1,N,3) into / out of position buffer `which` (0 or 1). */
int tmd_dd_load(tmd_ctx* ctx, int which, const float* pos_dev, tmd_stream stream);
int tmd_dd_store(tmd_ctx* ctx, int which, float* pos_dev, tmd_stream stream);
/* _first_VV (integrator.py:61-64) on the owned atoms: reads positions from buffer which_in,
 * writes the new ones into buffer 1-which_in of EVERY rank, then signals all ranks. */
int tmd_dd_vv_first_push(tmd_ctx* ctx, int which_in, float* vel_dev, const float* forces_dev,
                         const float* masses_dev, double dt, tmd_stream stream);
/* Wait (on the device) until every rank's stores of this step have landed here. */
int tmd_dd_wait(tmd_ctx* ctx, tmd_stream stream);
/* tmd_forces on position buffer `which`. */
int tmd_dd_forces(tmd_ctx* ctx, int which, float* forces_dev, double* energies_dev, tmd_stream stream);

/* ---- Wrapper.wrap (wrapper.py:8-30): molecules back into the box -----------------------
 *
 * Groups are the connected components of the bond graph (calculate_molecule_groups,
 * wrapper.py:33-55) as a CSR over atom indices: group g holds
 * group_atoms[group_ptr[g] .. group_ptr[g+1]); an atom without bonds is a group of one atom
 * (the reference's "nongrouped" branch is the same arithmetic).  tmd_wrapper_wrap moves every
 * group by  -floor(com / box) * box  per dimension, com being the plain mean of the group's
 * coordinates, in place on pos_dev (R,N,3), for every replica; box_dev is the (R,3,3) box
 * tensor (diagonal used).  If every box length is zero nothing happens (wrapper.py:14-15).
 * The optional re-centring on a wrap-index group (wrapper.py:17-21) rebinds a local name in
 * the reference and never reaches the caller's tensor; it is not part of this entry point.
 * Independent of tmd_ctx; only enqueues. */
typedef struct tmd_wrapper tmd_wrapper;
int tmd_wrapper_create(tmd_wrapper** out, int device, int natoms, int ngroups,
                       const int32_t* group_ptr_host, const int32_t* group_atoms_host);
int tmd_wrapper_wrap(tmd_wrapper* w, float* pos_dev, const float* box_dev, int nreplicas,
                     tmd_stream stream);
int tmd_wrapper_destroy(tmd_wrapper* w);

/* ---- "precision: double" ---------------------------------------------------------
 *
 * tmd_set_precision(ctx, 64) right after tmd_create, before any setter (TMD_ERR_STATE
 * otherwise); the default is 32.  An fp64 context takes its parameters through the _f64
 * setters below (tmd_set_exclusions, tmd_set_nonbonded and tmd_set_force_convention are
 * shared) and its per-step work through the _f64 entry points, which mirror the fp32 ones
 * with double state; an fp32 entry point on an fp64 context, or the reverse, returns
 * TMD_ERR_STATE.  Neighbour decisions are the reference's fp64 chain bit for bit
 * (d = p_i - p_j, w = d - L rint(d / L), sqrt_rn(fma(z,z,fma(y,y,x*x))) <= cutoff).  Full
 * neighbour rows only; tmd_set_owned_atoms and tmd_dd_* return TMD_ERR_UNSUPPORTED.  With a
 * cutoff, a coordinate of 8192 A or more from the origin is reported by tmd_get_stats
 * (TMD_ERR_UNSUPPORTED: wrap the system) and a box length above 4096 A is refused
 * (TMD_ERR_UNSUPPORTED at the first force call). */
int tmd_set_precision(tmd_ctx* ctx, int bits);
int tmd_set_atoms_f64(tmd_ctx* ctx, const double* charges_host, const int32_t* types_host,
                      int ntypes, const double* A_host, const double* B_host);
int tmd_set_bonds_f64(tmd_ctx* ctx, int n, const int32_t* idx_host, const double* prm_host);
int tmd_set_angles_f64(tmd_ctx* ctx, int n, const int32_t* idx_host, const double* prm_host);
int tmd_set_torsions_f64(tmd_ctx* ctx, int which, int n, const int32_t* idx_host,
                         const int32_t* term_ptr_host, const double* terms_host, int amber_form);
int tmd_set_pairs14_f64(tmd_ctx* ctx, int n, const int32_t* idx_host, const double* prm_host);
int tmd_set_box_f64(tmd_ctx* ctx, const double* box_diag_host);
int tmd_forces_f64(tmd_ctx* ctx, const double* pos_dev, double* forces_dev, double* energies_dev,
                   tmd_stream stream);
int tmd_vv_first_f64(tmd_ctx* ctx, double* pos_dev, double* vel_dev, const double* forces_dev,
                     const double* masses_dev, double dt, tmd_stream stream);
/* noise_dev NULL: fp64 normals from the Philox4x32-10 stream of tmd_vv_second (seed, step, atom) */
int tmd_vv_second_f64(tmd_ctx* ctx, double* vel_dev, const double* forces_dev, const double* masses_dev,
                      double dt, double gamma, const double* vcoeff_dev, const double* noise_dev,
                      uint64_t seed, uint64_t step_index, double* ke_dev, tmd_stream stream);
int tmd_kinetic_energy_f64(tmd_ctx* ctx, const double* vel_dev, const double* masses_dev, double* ke_dev,
                           tmd_stream stream);
/* niter steps enqueued with no host synchronisation (eager launches, no graph). */
int tmd_md_steps_f64(tmd_ctx* ctx, int niter, double* pos_dev, double* vel_dev, double* forces_dev,
                     const double* masses_dev, double dt, double gamma, const double* vcoeff_dev,
                     const double* noise_dev, uint64_t seed, uint64_t first_step_index,
                     double* energies_dev, double* ke_dev, tmd_stream stream);
int tmd_export_pairs_f64(tmd_ctx* ctx, const double* pos_dev, int replica, int32_t* pairs_dev,
                         int64_t capacity, int64_t* count_dev, tmd_stream stream);
int tmd_wrapper_wrap_f64(tmd_wrapper* w, double* pos_dev, const double* box_dev, int nreplicas,
                         tmd_stream stream);

/* ---- constraints: rigid water and bonds to hydrogen (library version >= 102) ----
 *
 * tmd_set_constraints holds the constraint tables in the context (host arrays, copied):
 *   water_idx[3*nwater]   heavy atom, hydrogen, hydrogen of each water
 *   water_d[2*nwater]     O-H and H-H distance (A)
 *   cluster_ptr[ncluster+1], cluster_idx: CSR of the X-H clusters, heavy atom first, then its 1-4 hydrogens
 *   cluster_d             one distance per hydrogen, in cluster_idx order with the heavy atoms left out
 * No atom may be in two groups.  nwater = ncluster = 0 clears the tables.  The call invalidates the
 * captured steps of tmd_md_steps.  While tables are set, tmd_md_steps[_f64], tmd_vv_first[_f64] and
 * tmd_vv_second[_f64] run RATTLE: analytic SETTLE for the waters and SHAKE for the clusters, against
 * the pre-drift positions after the drift (velocities
 * corrected by the displacement over dt), the velocity projection after the second half-kick, and
 * the kinetic energy after it.  tmd_vv_second[_f64] constrains against the positions of the last
 * tmd_vv_first[_f64] call.  Constraint arithmetic is fp64 in both precisions.  tmd_set_owned_atoms
 * and tmd_dd_* return TMD_ERR_UNSUPPORTED on a context with constraints.  A water without a SETTLE
 * solution or a cluster whose SHAKE iteration did not converge is reported by tmd_get_stats
 * (TMD_ERR_STATE, after its list-overflow report). */
int tmd_set_constraints(tmd_ctx* ctx, int nwater, const int32_t* water_idx_host, const double* water_d_host,
                        int ncluster, const int32_t* cluster_ptr_host, const int32_t* cluster_idx_host,
                        const double* cluster_d_host);
/* Projects a state onto the constraints: SETTLE / SHAKE with the state's own bond directions, then
 * (vel_dev not NULL) the velocity projection.  No-op without tables.  Unlike tmd_set_constraints it
 * takes the masses: a context holds none (the per-step calls pass them, and so does this one). */
int tmd_constrain(tmd_ctx* ctx, float* pos_dev, float* vel_dev, const float* masses_dev, tmd_stream stream);
int tmd_constrain_f64(tmd_ctx* ctx, double* pos_dev, double* vel_dev, const double* masses_dev, tmd_stream stream);

/* ---- particle-mesh Ewald electrostatics (library version >= 103) ----
 *
 * tmd_set_pme(ctx, tolerance > 0) turns PME on; tolerance <= 0 turns it off.  Call it after
 * tmd_set_nonbonded: it needs the electrostatics term, a cutoff and no reaction field
 * (TMD_ERR_UNSUPPORTED otherwise).  The electrostatic energy slot then holds
 *   real space    sum k qi qj erfc(alpha r) / r over the cutoff's pair set (no shift, no switch)
 *   reciprocal    smooth PME, order-5 B-splines, fp64 accumulation
 *   exclusions    - sum k qi qj erf(alpha r) / r over the excluded pairs (minimum image)
 *   self          - k alpha / sqrt(pi) sum qi^2
 *   background    - k pi Q^2 / (2 V alpha^2), Q the net charge
 * and the forces are its exact gradient.  alpha = sqrt(-ln 2 tol) / cutoff and the grid
 * n_d = smallest 2^a 3^b 5^c >= max(2 alpha L_d / (3 tol^(1/5)), 10), the largest over the
 * replicas, are chosen here and again by every tmd_set_box[_f64]; each replica keeps its own box
 * and influence function.  tmd_set_box[_f64] returns TMD_ERR_UNSUPPORTED for a box that is not
 * periodic, a cutoff above half a box length on any axis, or a grid above 512 points on an axis.
 * The reciprocal forces are bitwise reproducible (fixed-point charge grid, per-atom gather).
 * The exclusion correction reads the rows of tmd_set_exclusions as the set of excluded pairs: each pair
 * must appear in both atoms' rows, once, and no atom in its own row; otherwise the first force call
 * returns TMD_ERR_ARG.  The real-space term is cut at the cutoff without a shift, so energy
 * conservation improves with a smaller tolerance (DESIGN.md §5b).
 * tmd_set_owned_atoms and tmd_dd_* return TMD_ERR_UNSUPPORTED on a PME context.
 * tmd_get_pme reports the chosen alpha (1/A) and grid (TMD_ERR_STATE while PME is off or no box
 * has been set). */
int tmd_set_pme(tmd_ctx* ctx, double tolerance);
int tmd_get_pme(tmd_ctx* ctx, double* alpha, int32_t grid[3]);

/* ---- box changes in stream order, and the molecule move of a barostat (library version >= 104) ----
 *
 * tmd_rescale_box[_f64](ctx, box_diag_host, stream) gives every replica the box lengths
 * box_diag_host (R,3), in stream order: no re-finalisation, no allocation, no synchronisation, and
 * the captured tmd_md_steps step graphs stay valid.  The cell grids keep their cell counts while the
 * cells stay at least a list radius / nsub wide and otherwise drop to what the box holds; the next
 * force call rebuilds the lists.  With PME, alpha and the grid stay as they were (the influence
 * function and the self + background energy follow the box); a later tmd_set_box[_f64] chooses both
 * again.  The first rescale of a cluster-path context sets the cluster extent bound of a box 10 %
 * shorter than the one finalised, which makes the captured steps recapture once.  The call changes
 * nothing and returns TMD_ERR_UNSUPPORTED when the box cannot take this path: a context not yet
 * finalised (after a setter, or before its first force call), a box that is not periodic, a
 * decomposed or peer-to-peer context, a box that breaks the guard-free minimum-image condition the
 * context was set up with, the cluster lists' extent bound, 2 nsub + 1 cells along an axis, PME's
 * cutoff <= L/2, or the fp64 limit of 4096 A.  The caller then uses tmd_set_box[_f64].
 *
 * tmd_set_molecules(ctx, nmol, ptr, atoms, parent) holds a CSR of molecules: the atoms of molecule
 * m are atoms[ptr[m] .. ptr[m+1]), every atom exactly once, in breadth-first order of a spanning
 * tree of its bonds; parent[k] is the atom atoms[k] was reached from (an earlier atom of the same
 * molecule; the first atom is its own parent).  nmol = 0 clears them.
 * tmd_scale_molecules[_f64](ctx, pos_dev, scale_dev, stream) moves every molecule of every replica
 * rigidly with its centroid by the per-axis factors scale_dev (R,3) fp64 device memory, relative to
 * the box the context holds: unwrapped along its tree, centroid c, each atom to
 * r + (s - 1) c + n (s L - L), n its image in the molecule's unwrapped frame (csrc/barostat.cuh).
 * Call it before the tmd_rescale_box[_f64] / tmd_set_box[_f64] to the scaled box.
 *
 * tmd_step_captures returns how many step graphs tmd_md_steps has captured so far (-1 for NULL). */
int tmd_rescale_box(tmd_ctx* ctx, const float* box_diag_host, tmd_stream stream);
int tmd_rescale_box_f64(tmd_ctx* ctx, const double* box_diag_host, tmd_stream stream);
int tmd_set_molecules(tmd_ctx* ctx, int nmol, const int32_t* ptr, const int32_t* atoms, const int32_t* parent);
int tmd_scale_molecules(tmd_ctx* ctx, float* pos_dev, const double* scale_dev, tmd_stream stream);
int tmd_scale_molecules_f64(tmd_ctx* ctx, double* pos_dev, const double* scale_dev, tmd_stream stream);
int64_t tmd_step_captures(tmd_ctx* ctx);

/* ---- inspection ------------------------------------------------------------ */

/* The reference's neighbour list for one replica: every non-excluded pair
 * (i<j, original atom indices) with dist <= cutoff under the reference's own
 * fp32 predicate (forces.py:76-81,264-269), unordered.  pairs_dev holds
 * capacity*2 int32; *count_dev receives the number found (may exceed capacity). */
int tmd_export_pairs(tmd_ctx* ctx, const float* pos_dev, int replica, int32_t* pairs_dev,
                     int64_t capacity, int64_t* count_dev, tmd_stream stream);

/* Which pair kernel the last tmd_forces / tmd_md_steps launched: 0 k_pair (float separations, the
 * default), 1 k_pair_fx (fixed-point separations), 2 k_pair_fx2 (fixed point + fp32x2
 * arithmetic), 3 k_pair2_open (no box, fp32x2 arithmetic), 4 k_cpair (cluster lists),
 * 5 k_pair_f64 (fp64 context); with particle-mesh Ewald, the real-space Ewald instantiations
 * 6 k_pair<MODE 2>, 7 k_pair_fx<MODE 2>, 8 k_ewpair64 (fp64).  For tests and bench labels. */
int tmd_pair_kernel(tmd_ctx* ctx);

typedef struct {
  int64_t rebuilds;        /* neighbour-list rebuilds so far (all replicas) */
  int64_t force_calls;     /* tmd_forces invocations */
  int32_t max_neighbours;  /* longest neighbour row seen */
  int32_t row_capacity;    /* entries reserved per atom */
  int32_t overflow;        /* 1 if a row ever overflowed (results invalid) */
  int32_t ncells[3];       /* cell grid of replica 0 */
  int64_t kernel_launches; /* kernels launched by this context so far */
} tmd_stats;

/* Reads counters back. [sync]  If a row overflowed, grows the capacity,
 * forces a rebuild on the next call and returns TMD_ERR_OVERFLOW once. */
int tmd_get_stats(tmd_ctx* ctx, tmd_stats* out, tmd_stream stream);

/* Device-side timing of the non-bonded pair kernel: between begin and end every
 * tmd_forces brackets its pair-kernel launch with CUDA events on the launching
 * stream (at most max_samples of them).  tmd_profile_end synchronises and returns
 * the summed and the number of sampled launches. [sync] */
int tmd_profile_begin(tmd_ctx* ctx, int max_samples);
int tmd_profile_end(tmd_ctx* ctx, double* total_ms, int* nsamples, tmd_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* TMD_B200_H */
