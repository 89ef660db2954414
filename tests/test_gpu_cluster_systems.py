"""The cluster pair path (k_cpair, and k_cpair_ew with PME) on the systems it is the default for: a solvated protein
whose 1-2, 1-3 and 1-4 exclusions cross clusters, up to 128 atom types, and cutoffs long enough that the lists no longer
fit the kernel's shared-memory staging (the context must then take the full rows, not raise).  Every case first asserts
which pair kernel ran, so a silent fall-back fails.  tests/test_cluster_systems_on_interpreter.py runs these functions
on the host interpreter build of the kernels.

Test systems (built here, no new fixtures):
* ``tiled_system(name, t)``: a golden fixture repeated t x t x t times with its own box lengths.  ala2_xsc_rf at t = 2
  is 5,504 atoms in a 39.7 x 39.2 x 39.3 A box, just above the cluster condition L >= 2 (8 A + rl + skin + 0.05 A) =
  38.1 A at its own cutoff of 9 A, so the all-pairs oracle still holds it.  It runs with a skin of 0.5 A: the default
  1 A leaves clusters 8.6 A of room along an axis (L/2 - rl - skin), which a few of this box's clusters exceed, and the
  context would rightly continue on the full rows (F_CLFAIL); 0.5 A leaves 9.6 A.
* ``retyped(sysd, T)``: the tiled water box with T atom types (oxygens from [0, T/2), hydrogens from [T/2, T)), sigma
  and epsilon perturbed per type around TIP3P's.

Bounds (those of test_gpu_cluster.py and test_gpu_pme.py): the fp32 pair set bit-exact against the oracle's fp32
pairs; fp32 forces within 1e-4 kcal/mol/A of the fp64 oracle evaluated on the fp32 decisions (5e-4 with PME); energies
per term within 1e-5 |E| + 2e-3 (PME: 2e-5 relative); fp64 within 1e-9 of the largest force.  The retyped water boxes
take 1.5e-4 in fp32 (RETYPED_TOL): an oxygen sigma up to 10 % larger makes the closest O-O contacts up to 1.1^12 = 3x
more repulsive, and the fp32 rounding of each pair force (r^-14 carries 7 roundings of r^2) grows with it -- 1.1e-4 on
the interpreter's exactly rounded arithmetic, against 4e-5 for plain TIP3P.
"""
import numpy as np
import pytest
import torch

from oracle import refmd
from test_simt_cluster import tiled_water
from torchmd_b200._lib import PAIR_CLUSTER, PAIR_EWALD_CLUSTER, PAIR_F64, PAIR_ROWS_FX2

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
TABLES = {"bonds": "bond_params", "angles": "angle_params", "dihedrals": "dihedral_params", "impropers": "improper_params",
          "pairs14": "nonbonded_14_params"}
BONDED = ("bonds", "angles", "dihedrals", "impropers", "1-4")
WATER_TERMS = ["lj", "electrostatics", "bonds", "angles"]
RETYPED_TOL = 1.5e-4  # fp32 force bound of the retyped water boxes (module docstring)


def _L():
    from torchmd_b200 import _lib

    return _lib.lib()


# ---------------------------------------------------------------------------------------------------- test systems
def _spec_of(par, coords, box, terms, cfg, name):
    """Plain arrays of a TopologyParameters (fp64) plus coordinates and run settings."""
    spec = dict(name=name, types=par.mapped_atom_types.cpu().numpy(), sigma=par.nonbonded_params["params"][:, 0].numpy(),
                eps=par.nonbonded_params["params"][:, 1].numpy(), charges=par.charges.cpu().double().numpy(),
                masses=par.masses[:, 0].cpu().double().numpy(), coords=np.asarray(coords, np.float32),
                box=np.asarray(box, np.float32), terms=list(terms), cfg=dict(cfg))
    for key, attr in TABLES.items():
        tp = getattr(par, attr)
        spec[key] = None if tp is None else tuple(tp[k].cpu().numpy() for k in ("idx", "map", "params"))
    return spec


def params(spec, precision=torch.float32, device="cpu"):
    from torchmd_b200 import TopologyParameters

    return TopologyParameters(atom_types=spec["types"], type_sigma=spec["sigma"], type_epsilon=spec["eps"],
                              charges=spec["charges"], masses=spec["masses"], precision=precision, device=device,
                              **{k: spec[k] for k in TABLES})


def oracle_params(spec, decision_dtype=torch.float32):
    """fp64 parameters for an oracle.  For an fp32 run the LJ tables are the fp32 ones the kernels receive, in fp64: the
    oracle then evaluates exactly the kernels' inputs (positions, pair set and LJ tables), as it does for the positions.
    (sigma^12 amplifies the rounding of a perturbed sigma: with 17 types, the fp64 and fp32 tables alone differ by 1e-4
    kcal/mol/A in the force of a close O-O contact.)"""
    par = params(spec, torch.float64)
    if decision_dtype == torch.float32:
        A, B = params(spec, torch.float32).get_AB()
        par.get_AB = lambda: (A.double(), B.double())
    return par


def tiled_system(name, t):
    """Fixture ``name`` repeated t times along every axis with its own box lengths: tile (a, b, c) at c0 + (a, b, c) L0,
    per-atom arrays tiled, every bonded table's atom indices shifted by k N0 and its map rows by k M0 (M0 the rows of
    that table's idx: a map row may share an idx row, as multi-term dihedrals do), parameters unchanged."""
    from torchmd_b200 import testsystems

    par, c0, L0, terms, cfg = testsystems.golden_system(name, precision=torch.float64)
    base = _spec_of(par, c0, L0, terms, cfg, name)
    n0, L0 = len(c0), np.asarray(L0, np.float64)
    shifts = [np.array([a, b, c]) for a in range(t) for b in range(t) for c in range(t)]
    k = len(shifts)
    spec = dict(base, name=f"{name}x{t}", types=np.tile(base["types"], k), charges=np.tile(base["charges"], k),
                masses=np.tile(base["masses"], k), box=(L0 * t).astype(np.float32),
                coords=np.concatenate([np.asarray(c0, np.float64) + s * L0 for s in shifts]).astype(np.float32))
    for key in TABLES:
        if base[key] is None:
            continue
        idx, mp, prm = base[key]
        m0 = len(idx)
        spec[key] = (np.concatenate([idx + j * n0 for j in range(k)]),
                     np.concatenate([np.stack([mp[:, 0] + j * m0, mp[:, 1]], 1) for j in range(k)]), prm)
    assert len(params(spec).get_exclusions()) == k * len(par.get_exclusions())
    return spec


def water_spec(sysd, cfg=None):
    from torchmd_b200 import testsystems

    par = testsystems.water_parameters(sysd, precision=torch.float64)
    cfg = dict(cutoff=5.0, rfa=True, switch_dist=4.0) if cfg is None else cfg
    return _spec_of(par, sysd["coords"], sysd["box"], WATER_TERMS, cfg, sysd["name"])


def retyped(sysd, T, seed=0, cfg=None):
    """A water box with T atom types: oxygens draw theirs from [0, T/2), hydrogens from [T/2, T), and both T/2 - 1 and
    T - 1 occur; sigma and epsilon per type are TIP3P's perturbed by up to 10 % and 50 % (sign kept).  Charges and
    bonded terms unchanged."""
    from torchmd_b200 import testsystems as ts

    spec = water_spec(sysd, cfg)
    rng = np.random.default_rng(seed)
    oxy = spec["types"] == ts.WATER_TYPES.index("OT")
    h = T // 2
    types = np.where(oxy, rng.integers(0, h, len(oxy)), rng.integers(h, T, len(oxy)))
    types[np.flatnonzero(oxy)[0]] = h - 1
    types[np.flatnonzero(~oxy)[0]] = T - 1
    o, hy = ts.WATER_TYPES.index("OT"), ts.WATER_TYPES.index("HT")
    sig0 = np.where(np.arange(T) < h, ts.WATER_SIGMA[o], ts.WATER_SIGMA[hy])
    eps0 = np.where(np.arange(T) < h, ts.WATER_EPSILON[o], ts.WATER_EPSILON[hy])
    spec.update(name=f"{spec['name']}_t{T}", types=types, sigma=sig0 * rng.uniform(0.9, 1.1, T),
                eps=eps0 * rng.uniform(0.5, 1.5, T))
    assert types.max() == T - 1 and (types == h - 1).any()
    return spec


def shifted_molecules(spec, seed=0, reach=2):
    """Coordinates with every molecule (bond-graph component) moved by whole boxes, up to ``reach`` along each axis."""
    rng = np.random.default_rng(seed)
    x = np.asarray(spec["coords"], np.float64).copy()
    groups, single = refmd.molecule_groups(len(x), spec["bonds"][0] if spec["bonds"] is not None else None)
    L = np.asarray(spec["box"], np.float64)
    for g in groups + [[s] for s in single]:
        x[g] += rng.integers(-reach, reach + 1, 3) * L
    return x.astype(np.float32)


def thrown_atoms(spec, seed=5, reach=3):
    """30 % of single atoms (not molecules) moved by up to ``reach`` boxes: clusters mix image counts."""
    rng = np.random.default_rng(seed)
    c = np.asarray(spec["coords"], np.float32)
    sh = rng.integers(-reach, reach + 1, size=c.shape).astype(np.float32)
    return c + sh * (rng.random(len(c)) < 0.3)[:, None] * np.asarray(spec["box"], np.float32)


def scaled_replica(spec, s=1.02):
    """Molecule centroids scaled by s about the origin, in a box s times larger."""
    x = np.asarray(spec["coords"], np.float64).copy()
    groups, single = refmd.molecule_groups(len(x), spec["bonds"][0] if spec["bonds"] is not None else None)
    for g in groups + [[a] for a in single]:
        x[g] += (s - 1.0) * x[g].mean(0)
    return x.astype(np.float32), (np.asarray(spec["box"], np.float64) * s).astype(np.float32)


def configurations(spec, variant):
    """(coords (R,N,3), boxes (R,3)) of one test variant."""
    c, L = spec["coords"], spec["box"]
    if variant == "as_is":
        return c[None], L[None]
    if variant == "molecules_shifted":
        return shifted_molecules(spec)[None], L[None]
    if variant == "atoms_thrown":
        return thrown_atoms(spec)[None], L[None]
    if variant == "two_replicas":
        c2, L2 = scaled_replica(spec)
        return np.stack([c, c2]), np.stack([L, L2])
    raise ValueError(variant)


# ---------------------------------------------------------------------------------------------------- runs, oracles
def run(spec, coords=None, boxes=None, dtype=torch.float32, pme=False, **over):
    """Forces.compute on replicas (R,N,3) in boxes (R,3); returns (forces, pos, box, F, E, kernel id)."""
    from torchmd_b200 import Forces

    coords = spec["coords"][None] if coords is None else coords
    boxes = spec["box"][None] if boxes is None else boxes
    cfg = dict(spec["cfg"], **over)
    if pme:
        cfg.pop("rfa", None)
    pos = torch.tensor(np.asarray(coords), dtype=dtype, device=DEV)
    box = torch.diag_embed(torch.tensor(np.asarray(boxes), dtype=dtype, device=DEV))
    forces = Forces(params(spec, dtype, DEV), terms=spec["terms"], pme=pme, **cfg)
    F = torch.zeros_like(pos)
    E = forces.compute(pos, box, F, returnDetails=True)
    return forces, pos, box, F, E, _L().tmd_pair_kernel(forces._ctx)


def _ocfg(spec, **over):
    """The run settings the oracles take (everything but the list skin)."""
    return {k: v for k, v in dict(spec["cfg"], **over).items() if k != "skin"}


def oracle(spec, pos, box, decision_dtype, **over):
    """All-pairs fp64 oracle (forces (R,N,3), energies per replica) and, for fp32 decisions, the reference's pair set of
    every replica."""
    cfg = _ocfg(spec, **over)
    of = refmd.OracleForces(oracle_params(spec, decision_dtype), spec["terms"], decision_dtype=decision_dtype, **cfg)
    pos64 = pos.cpu().double()
    F = torch.zeros_like(pos64)
    E = of.compute(pos64, box.cpu().double(), F)
    pairs = None
    if decision_dtype == torch.float32:
        pairs = [of.neighbour_pairs(pos[r].cpu().float(), torch.diagonal(box[r]).cpu().float()).numpy() for r in range(len(pos))]
    return F, E, pairs


def check_fp32(spec, forces, pos, box, F, E, what, tol=1e-4, **over):
    Fo, Eo, pairs = oracle(spec, pos, box, torch.float32, **over)
    for r in range(len(pos)):
        got = forces.neighbour_pairs(pos, box, replica=r).cpu().numpy()
        assert got.shape == pairs[r].shape and np.array_equal(got, pairs[r].astype(np.int32)), (what, r)
    err = (F.cpu().double() - Fo).abs().max().item()
    print(f"{what}: max|dF| vs fp64 oracle {err:.3e} (max |F| {Fo.abs().max().item():.1f}), {len(pairs[0])} pairs")
    assert err < tol, (what, err)
    for r in range(len(pos)):
        for k in spec["terms"]:
            assert abs(E[r][k] - Eo[r][k]) <= 1e-5 * abs(Eo[r][k]) + 2e-3, (what, r, k, E[r][k], Eo[r][k])
    return err


def check_fp64(spec, pos, box, F, E, what, **over):
    Fo, Eo, _ = oracle(spec, pos, box, torch.float64, **over)
    err = (F.cpu().double() - Fo).abs().max().item()
    fmax = Fo.abs().max().item()
    print(f"{what}: max|dF| vs fp64 oracle {err:.3e} (max |F| {fmax:.1f})")
    assert err <= 1e-9 * fmax, (what, err, fmax)
    for r in range(len(pos)):
        for k in spec["terms"]:
            assert abs(E[r][k] - Eo[r][k]) <= 1e-9 * max(1.0, abs(Eo[r][k])), (what, r, k, E[r][k], Eo[r][k])
    return err


def check_pme(spec, forces, pos, boxes, F, E, what):
    from test_gpu_pme import _oracle as pme_oracle

    cfg = {k: v for k, v in _ocfg(spec).items() if k != "rfa"}
    alpha, grid = forces.pme_parameters()
    Eo, Fo = pme_oracle(oracle_params(spec), spec["terms"], cfg, pos.cpu().double().numpy(), np.asarray(boxes),
                        alpha, grid, torch.float32)
    err = np.abs(F.cpu().double().numpy() - Fo).max()
    print(f"{what}: alpha {alpha:.4f} grid {grid}: max|dF| vs fp64 oracle {err:.3e} (max |F| {np.abs(Fo).max():.1f})")
    assert err <= 5e-4, (what, err)
    for r in range(len(Eo)):
        for k in spec["terms"]:
            assert abs(E[r][k] - Eo[r][k]) <= 2e-5 * max(1.0, abs(Eo[r][k])), (what, r, k, E[r][k], Eo[r][k])
    return err


def bonded_oracle(spec, pos64, box_diag64, cutoff):
    """fp64 forces and energies of the bonded terms alone (the 1-4 pairs included, booked under lj / electrostatics as
    the reference books them), without the all-pairs table a large system cannot hold."""
    terms = [t for t in spec["terms"] if t in BONDED]
    of = refmd.OracleForces(params(spec, torch.float64), terms, cutoff=cutoff)
    of.terms = list(spec["terms"])  # the 1-4 pairs need lj / electrostatics in the terms ...
    of.needs_pairs = False          # ... but not the all-pairs non-bonded sum
    F = torch.zeros((1,) + tuple(pos64.shape), dtype=torch.float64)
    E = of.compute(pos64[None], torch.diag(box_diag64)[None], F)[0]
    return F[0], E


def check_sampled(spec, forces, pos, box, F, what, nsample=600, npartners=200, seed=7, tol=1e-4, **over):
    """Systems too large for the all-pairs oracle: the non-bonded force on ``nsample`` atoms from all their partners
    (refmd.sampled_rows) plus the bonded terms, against the kernels' forces; the partner sets of ``npartners`` of them
    against the exported pair list; the bonded energies."""
    cfg = _ocfg(spec, **over)
    n = pos.shape[1]
    atoms = sorted(np.random.default_rng(seed).choice(n, nsample, replace=False).tolist())
    pos64 = pos[0].cpu().double()
    bd = torch.diagonal(box[0]).cpu().double()
    pair_terms = [t for t in spec["terms"] if t in ("lj", "electrostatics")]
    f_nb, partners = refmd.sampled_rows(oracle_params(spec), pair_terms, pos64, bd, atoms, chunk=48, **cfg)
    f_b, e_b = bonded_oracle(spec, pos64, bd, cfg["cutoff"])
    err = (F[0].cpu().double()[atoms] - (f_nb + f_b[atoms])).abs().max().item()
    print(f"{what}: {nsample} sampled atoms, max|dF| vs fp64 oracle rows {err:.3e}")
    assert err < tol, (what, err)
    pairs = forces.neighbour_pairs(pos, box).cpu().numpy()
    by_second = pairs[np.argsort(pairs[:, 1], kind="stable")]
    for a, ref in zip(atoms[:npartners], partners[:npartners]):
        lo = np.searchsorted(pairs[:, 0], a), np.searchsorted(pairs[:, 0], a + 1)
        lo2 = np.searchsorted(by_second[:, 1], a), np.searchsorted(by_second[:, 1], a + 1)
        got = np.sort(np.concatenate([pairs[lo[0]:lo[1], 1], by_second[lo2[0]:lo2[1], 0]]))
        assert np.array_equal(got, ref.numpy().astype(np.int32)), (what, a)
    return err, e_b


# ---------------------------------------------------------------------------------------------------- solvated protein
VARIANTS = ["as_is", "molecules_shifted", "atoms_thrown", "two_replicas"]


def protein(t):
    """ala2_xsc_rf tiled t x t x t; at t = 2 with a skin of 0.5 A (module docstring)."""
    spec = tiled_system("ala2_xsc_rf", t)
    if t == 2:
        spec["cfg"]["skin"] = 0.5
    return spec


def protein_rf(variant, t=2):
    spec = protein(t)
    coords, boxes = configurations(spec, variant)
    forces, pos, box, F, E, kern = run(spec, coords, boxes)
    assert kern == PAIR_CLUSTER, (variant, kern)
    return check_fp32(spec, forces, pos, box, F, E, f"ala2 x{t}^3 RF {variant}, kernel {kern}")


def protein_pme(variant, t=2):
    spec = protein(t)
    coords, boxes = configurations(spec, variant)
    forces, pos, box, F, E, kern = run(spec, coords, boxes, pme=True)
    assert kern == PAIR_EWALD_CLUSTER, (variant, kern)
    return check_pme(spec, forces, pos, boxes, F, E, f"ala2 x{t}^3 PME {variant}, kernel {kern}")


@pytest.mark.parametrize("variant", VARIANTS)
def test_solvated_protein_on_the_cluster_kernel(variant):
    protein_rf(variant)


@pytest.mark.parametrize("variant", VARIANTS)
def test_solvated_protein_on_the_ewald_cluster_kernel(variant):
    protein_pme(variant)


def test_solvated_protein_charmm_like_cutoff():
    """ala2 tiled 3 x 3 x 3 (18,576 atoms, 59 A) at a cutoff of 12 A, switch from 10 A: the sampled oracle."""
    spec = protein(3)
    over = dict(cutoff=12.0, switch_dist=10.0)
    forces, pos, box, F, E, kern = run(spec, **over)
    assert kern == PAIR_CLUSTER, kern
    _, e_b = check_sampled(spec, forces, pos, box, F, f"ala2 x3^3 cutoff 12, kernel {kern}", **over)
    for k in ("bonds", "angles", "dihedrals", "impropers"):
        assert abs(E[0][k] - e_b[k]) <= 1e-5 * abs(e_b[k]) + 2e-3, (k, E[0][k], e_b[k])


def _md_system(spec, dtype=torch.float32, seed=3, T=300.0):
    from torchmd_b200 import System, maxwell_boltzmann

    par = params(spec, dtype, DEV)
    system = System(len(spec["coords"]), 1, dtype, DEV)
    system.set_positions(spec["coords"])
    system.set_box(spec["box"])
    torch.manual_seed(seed)
    system.set_velocities(maxwell_boltzmann(par.masses, T, 1))
    return par, system


def fresh_epot_matches(forces, system, pot, what):
    F = torch.empty_like(system.forces)
    E = forces.compute(system.pos, system.box, F)
    assert abs(float(pot[0]) - float(E[0])) <= 1e-5 * abs(float(E[0])) + 2e-3, (what, float(pot[0]), float(E[0]))


def protein_md_follows_the_full_rows(monkeypatch, nsteps=40, t=2):
    """NVE with skin 0.3 A (several rebuilds inside the run): the cluster path and the full rows give the same
    trajectory up to the summation order of the forces; the last step's E_pot is a fresh compute's."""
    from torchmd_b200 import Forces, Integrator

    spec = protein(t)
    out = []
    for cluster in ("1", "0"):
        monkeypatch.setenv("TMD_B200_CLUSTER", cluster)
        par, system = _md_system(spec)
        forces = Forces(par, terms=spec["terms"], **dict(spec["cfg"], skin=0.3))
        integ = Integrator(system, forces, 1.0, DEV, gamma=None, T=None)
        ekin, pot, _ = integ.step(niter=nsteps)
        kern = _L().tmd_pair_kernel(forces._ctx)
        assert kern == (PAIR_CLUSTER if cluster == "1" else PAIR_ROWS_FX2), (cluster, kern)
        assert forces.stats()["rebuilds"] >= 3, forces.stats()
        fresh_epot_matches(forces, system, pot, cluster)
        out.append((system.pos.clone(), system.vel.clone(), ekin, pot))
    dp = (out[0][0] - out[1][0]).abs().max().item()
    dv = (out[0][1] - out[1][1]).abs().max().item()
    print(f"ala2 x{t}^3 NVE {nsteps} steps, cluster vs full rows: max|dpos| {dp:.2e}, max|dvel| {dv:.2e}")
    assert dp < 1e-3 and dv < 1e-2, (dp, dv)
    assert abs(out[0][3][0] - out[1][3][0]) < 1e-5 * abs(out[1][3][0]) + 2e-2


def protein_hbonds_2fs(nsteps=200, chunk=20, t=2):
    """X-H bonds and rigid water at 2 fs with Langevin: stays on the cluster kernel, every constraint holds to the
    residual bounds of test_gpu_constraints.py after every chunk of steps."""
    from oracle import constraints as OC
    from torchmd_b200 import Constraints, Forces, Integrator

    spec = protein(t)
    par, system = _md_system(spec)
    forces = Forces(par, terms=spec["terms"], **spec["cfg"])
    con = Constraints(par, "hbonds")
    integ = Integrator(system, forces, 2.0, DEV, gamma=1.0, T=300.0, constraints=con)
    groups = OC.groups_of(con)
    for _ in range(nsteps // chunk):
        _, pot, _ = integ.step(chunk)
        assert _L().tmd_pair_kernel(forces._ctx) == PAIR_CLUSTER
        box = torch.diagonal(system.box, dim1=-2, dim2=-1).cpu().double().numpy()
        er, ev = OC.residuals(system.pos.cpu().double().numpy(), system.vel.cpu().double().numpy(), groups, box)
        assert er <= 2 * float(np.spacing(np.float32(system.pos.abs().max().item()))), er
        assert ev <= 1e-6, ev
    assert np.isfinite(pot).all()
    fresh_epot_matches(forces, system, pot, "hbonds")


def test_protein_md_follows_the_full_row_trajectory(monkeypatch):
    protein_md_follows_the_full_rows(monkeypatch)


def test_protein_constraints_at_2fs_on_the_cluster_kernel():
    protein_hbonds_2fs()


# ---------------------------------------------------------------------------------------------------- atom types
def types_on_every_path(monkeypatch, T, t=2):
    """T atom types on the cluster kernel, the full rows (a global LJ table above 16 types), cluster PME and fp64."""
    spec = retyped(tiled_water(t), T, seed=T)
    what = f"water x{t}^3, {T} types"
    forces, pos, box, F, E, kern = run(spec)
    assert kern == PAIR_CLUSTER, (T, kern)
    Fo, Eo, pairs = oracle(spec, pos, box, torch.float32)
    results = {kern: (forces, F, E)}
    monkeypatch.setenv("TMD_B200_CLUSTER", "0")
    forces2, _, _, F2, E2, kern2 = run(spec)
    monkeypatch.delenv("TMD_B200_CLUSTER")
    assert kern2 == PAIR_ROWS_FX2, (T, kern2)
    results[kern2] = (forces2, F2, E2)
    for k, (fo, Fk, Ek) in results.items():
        got = fo.neighbour_pairs(pos, box).cpu().numpy()
        assert np.array_equal(got, pairs[0].astype(np.int32)), (T, k)
        err = (Fk.cpu().double() - Fo).abs().max().item()
        print(f"{what}, kernel {k}: max|dF| vs fp64 oracle {err:.3e}")
        assert err < RETYPED_TOL, (T, k, err)
        for term in spec["terms"]:
            assert abs(Ek[0][term] - Eo[0][term]) <= 1e-5 * abs(Eo[0][term]) + 2e-3, (T, k, term, Ek[0][term], Eo[0][term])
    forces, pos, box, F, E, kern = run(spec, pme=True)
    assert kern == PAIR_EWALD_CLUSTER, (T, kern)
    check_pme(spec, forces, pos, spec["box"][None], F, E, f"{what} PME, kernel {kern}")
    forces, pos, box, F, E, kern = run(spec, dtype=torch.float64)
    assert kern == PAIR_F64, (T, kern)
    check_fp64(spec, pos, box, F, E, f"{what} fp64, kernel {kern}")


@pytest.mark.parametrize("T", [2, 16, 17, 64, 65, 128])
def test_atom_types_on_every_path(monkeypatch, T):
    types_on_every_path(monkeypatch, T)


def more_than_128_types_are_refused(dtype, t=2):
    """129 types: refused in both precisions with the 128-type limit named; a valid context built afterwards works."""
    from torchmd_b200 import _lib

    with pytest.raises(_lib.TmdError, match="128 atom types"):
        run(retyped(tiled_water(t), 129), dtype=dtype)
    spec = retyped(tiled_water(t), 128)
    forces, pos, box, F, E, kern = run(spec, dtype=dtype)
    assert kern == (PAIR_CLUSTER if dtype == torch.float32 else PAIR_F64), kern
    assert torch.isfinite(F).all()
    if dtype == torch.float32:
        check_fp32(spec, forces, pos, box, F, E, "128 types after a refused context", tol=RETYPED_TOL)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_more_than_128_types_are_refused(dtype):
    more_than_128_types_are_refused(dtype)


# ---------------------------------------------------------------------------------------------------- long cutoffs
def long_cutoff(spec, cutoff, switch, want, nsteps=20, tol=1e-4):
    """Computes on the kernel(s) in ``want`` (the cluster kernel, or the full rows when the lists do not fit its
    shared-memory staging), matches the sampled oracle, and runs ``nsteps`` captured steps whose last E_pot is a fresh
    compute's."""
    from torchmd_b200 import Forces, Integrator

    over = dict(cutoff=cutoff, switch_dist=switch)
    forces, pos, box, F, E, kern = run(spec, **over)
    assert kern in want, (spec["name"], cutoff, kern)
    check_sampled(spec, forces, pos, box, F, f"{spec['name']} cutoff {cutoff}, kernel {kern}", tol=tol, **over)
    par, system = _md_system(spec)
    forces = Forces(par, terms=spec["terms"], **dict(spec["cfg"], **over))
    integ = Integrator(system, forces, 1.0, DEV, gamma=1.0, T=300.0)
    _, pot, _ = integ.step(nsteps)
    assert _L().tmd_pair_kernel(forces._ctx) in want
    fresh_epot_matches(forces, system, pot, (spec["name"], cutoff))
    return kern


def test_water_at_cutoff_16():
    """tiled water, 64.6 A, cutoff 16 A: about 190 KB of staging by the initial estimate."""
    kern = long_cutoff(water_spec(tiled_water(3)), 16.0, 14.0, (PAIR_CLUSTER, PAIR_ROWS_FX2))
    print("water x3^3 at cutoff 16: kernel", kern)


def test_128_types_at_cutoff_14():
    kern = long_cutoff(retyped(tiled_water(3), 128), 14.0, 12.0, (PAIR_CLUSTER, PAIR_ROWS_FX2), tol=RETYPED_TOL)
    print("128 types at cutoff 14: kernel", kern)


def test_128_types_at_cutoff_12_stay_on_the_cluster_kernel():
    """About 167 KB of staging: within the limit, so the fall-back must not take it."""
    long_cutoff(retyped(tiled_water(3), 128), 12.0, 10.0, (PAIR_CLUSTER,), tol=RETYPED_TOL)
