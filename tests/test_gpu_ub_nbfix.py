"""Urey-Bradley terms and NBFIX pair overrides on the GPU.  tests/test_ub_nbfix_on_interpreter.py runs most of these
functions on the host interpreter build of the kernels.

Urey-Bradley: every angle (a, b, c) of a fixture gets a term on (a, c) with k_ub = 5 + 3 (t mod 7) and
s0 = r_ac + 0.05 + 0.02 (t mod 5) - 0.08 (r_ac of the first replica, fp64, minimum image), so no term sits at its
minimum.  The kernels are checked against the fp64 numpy oracle (oracle/urey_bradley.py).

NBFIX: the reference's CHARMM fixtures 3ions (SOD + 2 CLA) and waterbox (97 TIP3P, SOD, CLA), parameterised from their
own .prm files with and without ``"nbfix"``, against the fp64 CPU oracle (oracle/refmd.py) fed the same
``TopologyParameters``.  "waterbox_periodic" is waterbox in a 15.5 A box with a 7 A cutoff (switch at 6 A) and its
CLA moved along the line to the SOD until they are 6.7 A apart (no other atom within 2.2 A of it), so that the cluster lists, the full rows and particle-mesh Ewald all
see the SOD-CLA pair.
"""
import glob
import os
import warnings

import numpy as np
import pytest
import torch

from conftest import GOLDEN, golden_cfg, golden_system_tensors, load_golden
from oracle import urey_bradley as oub

DEV = "cuda"


# ---- Urey-Bradley ------------------------------------------------------------------------------------------------
def ub_terms(g, pos0, box0):
    """(angle idx (n,3), params (n,2)) by the module docstring's rule; pos0 (N,3), box0 (3,) fp64."""
    idx = np.asarray(g["par_angle_idx"], np.int64)
    d = pos0[idx[:, 2]] - pos0[idx[:, 0]]
    if box0.any():
        d = d - box0 * np.round(d / box0)
    r = np.linalg.norm(d, axis=1)
    t = np.arange(len(idx))
    return idx, np.stack([5.0 + 3.0 * (t % 7), r + 0.05 + 0.02 * (t % 5) - 0.08], axis=1)


def make_params(g, precision, ub_only=False, with_ub=True):
    """The fixture's parameters with a Urey-Bradley term on every angle; ``ub_only``: no other bonded term."""
    from torchmd_b200.parameters import TopologyParameters

    pos, box = golden_system_tensors(g, torch.float64)
    idx, prm = ub_terms(g, pos[0].numpy(), torch.diagonal(box[0]).numpy())
    se = g["par_lj_sigma_eps"]

    def term(k):
        return None if ub_only or "par_" + k + "_idx" not in g else (g["par_" + k + "_idx"], g["par_" + k + "_map"], g["par_" + k + "_params"])

    ub = (idx, np.stack([np.arange(len(idx)), np.arange(len(idx))], 1), prm) if with_ub else None
    return TopologyParameters(atom_types=g["par_types"], type_sigma=se[:, 0], type_epsilon=se[:, 1], charges=g["par_charges"],
                              masses=g["par_masses"], bonds=term("bond"), angles=term("angle"), dihedrals=term("dihedral"),
                              impropers=term("improper"), pairs14=term("nonbonded_14"), urey_bradley=ub, precision=precision,
                              device=DEV)


def oracle(par, pos, box):
    """(E (R,), F (R,N,3)) of the Urey-Bradley terms alone, fp64, from the positions as the kernels see them."""
    u = par.ub_params
    idx = u["idx"].cpu().numpy()[:, [0, 2]]
    m = u["map"].cpu().numpy()
    prm = u["params"].double().cpu().numpy()[m[np.argsort(m[:, 0], kind="stable"), 1]]
    Es, Fs = [], []
    for r in range(pos.shape[0]):
        L = torch.diagonal(box[r]).double().cpu().numpy()
        e, f = oub.energy_forces(pos[r].double().cpu().numpy(), idx, prm[:, 0], prm[:, 1], box=L if L.any() else None)
        Es.append(e)
        Fs.append(f)
    return np.array(Es), np.stack(Fs)


def assert_close(F, Fo, dtype, what=""):
    F = F.double().cpu().numpy() if torch.is_tensor(F) else F
    scale = np.abs(Fo).max()
    if dtype == torch.float64:
        err = np.abs(F - Fo).max()
        assert err <= 1e-10 * scale, f"{what}: max |dF| {err:.3e}, max |F| {scale:.3e}"
    else:  # an fp64 sum rounded once to fp32 (plus the last bit of the fp64 arithmetic at a rounding boundary)
        bad = np.abs(F - Fo) > 2.0**-23 * np.abs(Fo) + 1e-12 * scale
        assert not bad.any(), f"{what}: {bad.sum()} components beyond fp32 rounding, max |dF| {np.abs(F - Fo).max():.3e}"


def ub_only_forces(name, dtype, pos=None, box=None, explicit_forces=True):
    """Forces(terms=["angles"]) on the Urey-Bradley terms alone against the oracle; returns (E, F) of the kernels."""
    from torchmd_b200 import Forces

    g = load_golden(name)
    par = make_params(g, dtype, ub_only=True)
    if pos is None:
        pos, box = golden_system_tensors(g, dtype, DEV)
    f = Forces(par, terms=["angles"], **golden_cfg(g))
    F = torch.zeros_like(pos)
    E = f.compute(pos, box, F, returnDetails=True)
    if not explicit_forces:  # the autograd path: forces as -dE/dpos of the differentiable energy
        p = pos.detach().clone().requires_grad_(True)
        Et = f.compute(p, box, None, toNumpy=False, calculateForces=False, explicit_forces=False)
        F = -torch.autograd.grad(Et.sum(), p)[0]
    Eo, Fo = oracle(par, pos, box)
    assert_close(F.detach(), Fo, dtype, f"{name} {dtype}")
    for r in range(pos.shape[0]):
        e = float(E[r]["angles"])
        assert abs(e - Eo[r]) <= 1e-10 * max(1.0, abs(Eo[r])), (e, Eo[r])
    return E, F


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "chain_amber_vacuum", "chain_amber_periodic", "thrombin_nobox_rf"])
def test_ub_against_oracle(name, dtype):
    ub_only_forces(name, dtype)


def replicas_boundary_and_far_images(dtype):
    """Three replicas of ala2 in its box: the fixture, a perturbed copy, and a copy whose atoms are moved by whole box
    lengths (-3..3 per axis), so terms straddle the boundary and molecules sit several boxes away."""
    g = load_golden("ala2_xsc_rf")
    pos, box = golden_system_tensors(g, torch.float64, "cpu")
    pos = pos[:1].repeat(3, 1, 1).clone()
    box = box[:1].repeat(3, 1, 1).clone()
    rng = np.random.default_rng(7)
    pos[1] += torch.tensor(rng.normal(scale=0.1, size=pos[1].shape))
    L = torch.diagonal(box[2])
    pos[2] += torch.tensor(rng.integers(-3, 4, size=pos[2].shape), dtype=torch.float64) * L
    ub_only_forces("ala2_xsc_rf", dtype, pos.to(dtype).to(DEV).contiguous(), box.to(dtype).to(DEV).contiguous())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_ub_replicas_boundary_and_far_images(dtype):
    replicas_boundary_and_far_images(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_ub_autograd_path_gives_the_same_gradient(dtype):
    ub_only_forces("chain_amber_vacuum", dtype, explicit_forces=False)


def not_cutoff_filtered(dtype):
    """A term 12 A long with a 9 A cutoff still acts (a bond that long would not, as in the reference)."""
    from torchmd_b200 import Forces
    from torchmd_b200.parameters import TopologyParameters

    x = np.array([[0.0, 0.0, 0.0], [6.0, 1.0, 0.0], [12.0, 0.0, 0.0]])
    par = TopologyParameters(atom_types=np.zeros(3, np.int64), type_sigma=[1.0], type_epsilon=[0.0], charges=np.zeros(3),
                             masses=np.ones(3), urey_bradley=([[0, 1, 2]], [[0, 0]], [[2.0, 11.0]]), precision=dtype, device=DEV)
    pos = torch.tensor(x[None], dtype=dtype, device=DEV)
    F = torch.zeros_like(pos)
    E = Forces(par, terms=["angles"], cutoff=9.0).compute(pos, torch.zeros(1, 3, 3, dtype=dtype, device=DEV), F, returnDetails=True)
    assert abs(E[0]["angles"] - 2.0) < 1e-9
    assert abs(float(F[0, 0, 0]) - 4.0) < 1e-6 and abs(float(F[0, 2, 0]) + 4.0) < 1e-6 and float(F[0, 1].abs().max()) == 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_ub_is_not_cutoff_filtered(dtype):
    not_cutoff_filtered(dtype)


def angle_slot_sums(name, dtype):
    """With the fixture's own terms and Urey-Bradley terms, the angle slot is the sum of both and the forces add up."""
    from torchmd_b200 import Forces

    g = load_golden(name)
    pos, box = golden_system_tensors(g, dtype, DEV)
    terms = [str(t) for t in g["terms"]]
    out = {}
    for with_ub in (False, True):
        par = make_params(g, dtype, with_ub=with_ub)
        f = Forces(par, terms=terms, **golden_cfg(g))
        F = torch.zeros_like(pos)
        out[with_ub] = (f.compute(pos, box, F, returnDetails=True), F.double().cpu().numpy(), par)
    Eo, Fo = oracle(out[True][2], pos, box)
    for r in range(pos.shape[0]):
        e0, e1 = out[False][0][r], out[True][0][r]
        assert abs(e1["angles"] - (e0["angles"] + Eo[r])) <= 1e-9 * max(1.0, abs(e1["angles"]))
        for k in e0:
            if k != "angles":
                assert abs(e0[k] - e1[k]) <= 1e-9 * max(1.0, abs(e0[k])), k
    Fw, Fwo = out[True][1], out[False][1]
    bound = 1e-10 if dtype == torch.float64 else 2.0**-20
    assert np.abs(Fw - Fwo - Fo).max() <= bound * np.abs(Fw).max()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "chain_amber_periodic"])
def test_angle_slot_holds_angles_and_ub(name, dtype):
    angle_slot_sums(name, dtype)


def paths_agree(name, env_sets, monkeypatch, dtype=torch.float32):
    """With and without Urey-Bradley terms under each environment setting: the difference of the forces is the oracle's
    force, a captured step leaves forces that include the terms, the launches per captured step are the same, and a
    fused Integrator.step(n) ends where n single steps do."""
    from torchmd_b200 import Forces, Integrator, System

    g = load_golden(name)
    terms = [str(t) for t in g["terms"]]
    pos, box = golden_system_tensors(g, dtype, DEV)
    Fo = oracle(make_params(g, dtype), pos, box)[1]  # (the parameters as the context holds them)
    for env in env_sets:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        launches, forces, ends = {}, {}, {}
        for with_ub in (True, False):
            par = make_params(g, dtype, with_ub=with_ub)
            f = Forces(par, terms=terms, **golden_cfg(g))
            F = torch.zeros_like(pos)
            f.compute(pos, box, F)
            forces[with_ub] = F.double().cpu().numpy()
            for fused in (True, False):
                s = System(pos.shape[1], pos.shape[0], dtype, DEV)
                s.set_positions(pos[0].cpu().numpy())
                s.set_box(torch.diagonal(box[0]).cpu().numpy())
                f.compute(s.pos, s.box, s.forces)
                integ = Integrator(s, f, 0.5, DEV)
                if fused:
                    integ.step(2)
                    n0 = f.stats()["kernel_launches"]
                    integ.step(3)
                    launches[with_ub] = f.stats()["kernel_launches"] - n0
                else:
                    for _ in range(5):
                        integ.step(1)
                ends[fused] = s.pos.double().cpu().numpy()
            F2 = torch.zeros_like(s.forces)
            f.compute(s.pos, s.box, F2)
            step_err = (s.forces.double() - F2.double()).abs().max().item()
            assert step_err <= 1e-5 * max(1.0, F2.abs().max().item()), (env, with_ub, step_err)
            assert np.abs(ends[True] - ends[False]).max() <= 1e-5 * max(1.0, np.abs(ends[False]).max()), (env, with_ub)
        assert launches[True] == launches[False], (env, launches)
        Fw, Fwo = forces[True], forces[False]
        slack = 2.0**-20 * np.abs(Fw).max() if env.get("TMD_B200_CLUSTER", "0") == "1" else 1e-12 * np.abs(Fo).max()
        bad = np.abs(Fw - Fwo - Fo) > 2.0**-23 * (np.abs(Fw) + np.abs(Fwo)) + slack
        assert not bad.any(), (env, np.abs(Fw - Fwo - Fo).max())


ENV_SETS = [{"TMD_B200_CLUSTER": c, "TMD_B200_OVERLAP": o, "TMD_B200_GRAPH": gr, "TMD_B200_FUSEPREP": fp}
            for c in "01" for o in "01" for gr, fp in (("0", "0"), ("1", "1"), ("1", "0"))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "thrombin_nobox_rf"])
def test_ub_switches_agree_and_launch_counts_unchanged(name, monkeypatch):
    paths_agree(name, ENV_SETS, monkeypatch)


def barostat_and_constraints():
    """An NPT run with X-H constraints and Urey-Bradley terms (those on X-H...Y pairs stay forces, not constraints):
    its E_pot equals a fresh Forces.compute sum, and the constrained bonds keep their lengths."""
    from torchmd_b200 import Constraints, Forces, Integrator, MonteCarloBarostat, System, maxwell_boltzmann

    g = load_golden("ala2_xsc_rf")
    terms = [str(t) for t in g["terms"]]
    par = make_params(g, torch.float32)
    pos, box = golden_system_tensors(g, torch.float32, DEV)
    s = System(pos.shape[1], 1, torch.float32, DEV)
    s.set_positions(pos[0].cpu().numpy())
    s.set_box(torch.diagonal(box[0]).cpu().numpy())
    f = Forces(par, terms=terms, **golden_cfg(g))
    torch.manual_seed(0)
    s.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    f.compute(s.pos, s.box, s.forces)
    integ = Integrator(s, f, 1.0, DEV, gamma=1.0, T=300.0, constraints=Constraints(par, "hbonds"),
                       barostat=MonteCarloBarostat(1.0, 300.0, frequency=5, seed=1))
    _, ep, _ = integ.step(20)
    F = torch.zeros_like(s.pos)
    E = f.compute(s.pos, s.box, F)
    assert abs(float(ep[0]) - float(E[0])) <= 1e-4 * max(1.0, abs(float(ep[0])))
    bp = par.bond_params
    idx, r0 = bp["idx"].cpu().numpy(), bp["params"].double().cpu().numpy()[bp["map"].cpu().numpy()[:, 1], 1]
    light = (par.masses.cpu().numpy()[:, 0] < 1.5)[idx].any(1)
    x, L = s.pos[0].double().cpu().numpy(), torch.diagonal(s.box[0]).double().cpu().numpy()
    d = x[idx[:, 1]] - x[idx[:, 0]]
    r = np.linalg.norm(d - L * np.round(d / L), axis=1)
    assert light.any() and np.abs(r - r0)[light].max() < 1e-3  # X-H bonds held; the Urey-Bradley pairs are not among them


@pytest.mark.gpu
def test_barostat_and_constraints_with_ub():
    barostat_and_constraints()


# ---- NBFIX -------------------------------------------------------------------------------------------------------
def reference_inputs_dir(tmp):
    """The reference's input files (golden/reference_inputs.npz) written under ``tmp``."""
    with np.load(os.path.join(GOLDEN, "reference_inputs.npz")) as z:
        for rel in z.files:
            if rel.startswith("data/"):
                os.makedirs(os.path.join(tmp, os.path.dirname(rel)), exist_ok=True)
                with open(os.path.join(tmp, rel), "wb") as fh:
                    fh.write(z[rel].tobytes())
    return str(tmp)


PERIODIC_WATERBOX = dict(box=np.array([15.5, 15.5, 15.5]), cutoff=7.0, switch_dist=6.0, rfa=False)


def charmm_case(inputs, name, precision, nbfix, terms=None, device=None, extra=()):
    """(TopologyParameters, terms, cfg, pos (1,N,3) fp64, box (3,)) of a CHARMM fixture from its .prm."""
    from torchmd_b200 import charmm
    from torchmd_b200.ff_yaml import yaml_parameters

    base = name.replace("_periodic", "")
    g = load_golden("charmm_" + base)
    folder = os.path.join(inputs, "data", base)
    psf, pdb, prm = (glob.glob(os.path.join(folder, e))[0] for e in ("*.psf", "*.pdb", "*.prm"))
    mol = charmm.load_molecule(psf, pdb)
    terms = [str(t) for t in g["terms"]] if terms is None else list(terms)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        par = yaml_parameters(mol, charmm.CharmmPrmForceField(prm, mol), terms=terms + (["nbfix"] if nbfix else []) + list(extra),
                              precision=precision, device=DEV if device is None else device)
    cfg, box, pos = golden_cfg(g), np.asarray(g["box"], np.float64), np.asarray(g["coords"], np.float64)
    if name.endswith("_periodic"):
        cfg = {k: PERIODIC_WATERBOX[k] for k in ("cutoff", "switch_dist", "rfa")}
        box = PERIODIC_WATERBOX["box"]
        sod, cla = (int(np.nonzero(mol.atomtype == t)[0][0]) for t in ("SOD", "CLA"))
        d = pos[cla] - pos[sod]
        pos[cla] = pos[sod] + 0.85 * (d - box * np.round(d / box))
    return par, terms, cfg, pos[None], box


def nbfix_forces(inputs, name, dtype, pme=False):
    """Kernels with and without NBFIX against the fp64 oracle on the same tables; the difference moves only the atoms
    of NBFIX types and equals the oracle's difference.  With ``pme`` the electrostatics are particle-mesh Ewald (not
    in the oracle), so only the difference of the two runs is checked there."""
    from oracle import refmd
    from torchmd_b200 import Forces

    out = {}
    for nb in (False, True):
        par, terms, cfg, pos0, box0 = charmm_case(inputs, name, dtype, nb)
        pos = torch.tensor(pos0, dtype=dtype, device=DEV)
        box = torch.tensor(np.diag(box0)[None], dtype=dtype, device=DEV)
        f = Forces(par, terms=terms, pme=pme, **cfg)
        F = torch.zeros_like(pos)
        E = f.compute(pos, box, F, returnDetails=True)[0]
        par64 = charmm_case(inputs, name, torch.float64, nb, device="cpu")[0]
        ot = ["lj"] if pme else terms
        of = refmd.OracleForces(par64, ot, decision_dtype=torch.float32 if dtype == torch.float32 else None, **cfg)
        Fo = torch.zeros(pos.shape, dtype=torch.float64)
        Eo = of.compute(pos.cpu().double(), box.cpu().double(), Fo)[0]
        out[nb] = (E, F.double().cpu().numpy()[0], Eo, Fo.numpy()[0], par64)
        if not pme:
            err, scale = np.abs(out[nb][1] - out[nb][3]).max(), np.abs(out[nb][3]).max()
            bound = 1e-9 * max(1.0, scale) if dtype == torch.float64 else 1e-4 * max(1.0, scale / 100.0)
            assert err <= bound, (name, nb, err, scale)
            for k in ("lj", "electrostatics"):
                tol = 1e-9 if dtype == torch.float64 else 1e-5
                assert abs(E[k] - Eo[k]) <= tol * max(1.0, abs(Eo[k])) + (0 if dtype == torch.float64 else 2e-3), (k, E[k], Eo[k])
    # the tables differ at the NBFIX type pairs only
    (A0, B0), (A1, B1) = out[False][4].get_AB(), out[True][4].get_AB()
    moved = ((A0 != A1) | (B0 != B1)).numpy()
    fixed = np.zeros_like(moved)
    if out[True][4].nbfix_params is not None:
        ij = out[True][4].nbfix_params["idx"].numpy()
        fixed[ij[:, 0], ij[:, 1]] = fixed[ij[:, 1], ij[:, 0]] = True
    assert not (moved & ~fixed).any()
    types = out[True][4].mapped_atom_types.numpy()
    nbfix_atoms = np.isin(types, np.nonzero(fixed.any(1))[0])
    dF, dFo = out[True][1] - out[False][1], out[True][3] - out[False][3]
    scale = max(1.0, np.abs(out[True][1]).max())
    bound = 1e-9 * scale if dtype == torch.float64 else 2e-4 * max(1.0, scale / 100.0)
    assert np.abs(dF - dFo).max() <= bound, np.abs(dF - dFo).max()
    assert np.abs(dF[~nbfix_atoms]).max(initial=0.0) <= bound
    dE, dEo = out[True][0]["lj"] - out[False][0]["lj"], out[True][2]["lj"] - out[False][2]["lj"]
    assert abs(dE - dEo) <= (1e-9 if dtype == torch.float64 else 1e-5) * max(1.0, abs(out[True][2]["lj"])) + (0 if dtype == torch.float64 else 1e-3)
    if fixed.any():
        assert abs(dEo) > 1e-6 and np.abs(dFo).max() > 1e-6  # the override does something


NBFIX_CASES = [("3ions", {}), ("waterbox", {}), ("sodiumperiodic", {}),
               ("waterbox_periodic", {"TMD_B200_CLUSTER": "1"}), ("waterbox_periodic", {"TMD_B200_CLUSTER": "0"})]


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name,env", NBFIX_CASES)
def test_nbfix_on_every_pair_path(tmp_path, monkeypatch, name, env, dtype):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    nbfix_forces(reference_inputs_dir(tmp_path), name, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_nbfix_with_pme(tmp_path, dtype):
    nbfix_forces(reference_inputs_dir(tmp_path), "waterbox_periodic", dtype, pme=True)


# ---- CHARMM36 end to end ------------------------------------------------------------------------------------------
ALA2_CHARMM_TYPES = {"HH31": "HA3", "CH3": "CT3", "HH32": "HA3", "HH33": "HA3", "C": "C", "O": "O", "N": "NH1", "H": "H",
                     "CA": "CT1", "HA": "HB1", "CB": "CT3", "HB1": "HA3", "HB2": "HA3", "HB3": "HA3"}


def ala2_charmm(inputs, precision, terms, device=None):
    """ala2 (its prmtop's 22 solute atoms, coordinates of the ala2 fixture) with CHARMM36 atom types, parameterised from the
    CHARMM36 .prm; backbone cross-term C(ACE)-N-CA-C-N(NME)."""
    import types as _t

    from torchmd_b200 import amber, charmm
    from torchmd_b200.ff_yaml import yaml_parameters

    sysm = amber.AmberSystem(os.path.join(inputs, "data", "prod_alanine_dipeptide_amber", "structure.prmtop"))
    prm = read_names(os.path.join(inputs, "data", "prod_alanine_dipeptide_amber", "structure.prmtop"))
    n = 22
    names = prm[:n]
    keep = lambda a: a[np.all(a < n, axis=1)]  # noqa: E731
    mol = _t.SimpleNamespace(atomtype=np.array([ALA2_CHARMM_TYPES[x] for x in names], dtype=object),
                             charge=sysm.charge[:n], masses=sysm.masses[:n], bonds=keep(sysm.bonds), angles=keep(sysm.angles),
                             dihedrals=keep(sysm.dihedrals), impropers=np.zeros((0, 4), np.int64),
                             crossterms=np.array([[4, 6, 8, 14, 6, 8, 14, 16]], np.int64))
    ff = charmm.CharmmPrmForceField(os.path.join(inputs, "data", "waterbox", "parameters.prm"), mol)
    par = yaml_parameters(mol, ff, terms=terms, precision=precision, device=DEV if device is None else device)
    g = load_golden("ala2_xsc_rf")
    return par, mol, ff, np.asarray(g["coords"], np.float64)[:n]


def read_names(path):
    from torchmd_b200 import amber

    return amber.read_prmtop(path)["ATOM_NAME"]


# (no proper dihedrals: CHARMM36's use wildcard types, which the .prm reader, like the reference's adapter, does not match)
C36_TERMS = ["bonds", "angles", "electrostatics", "lj", "cmap", "ureybradley"]
C36_FORCES = ["bonds", "angles", "dihedrals", "electrostatics", "lj"]  # ("dihedrals": the CMAP term)


def charmm36_ala2(inputs, dtype):
    """The number of Urey-Bradley terms is the number of angles whose type has k_ub > 0; per-term energies and forces
    match the oracle."""
    from torchmd_b200 import Forces

    par, mol, ff, x = ala2_charmm(inputs, dtype, C36_TERMS)
    uq = {tuple(a) if a[0] < a[2] else tuple(a[::-1]) for a in np.asarray(mol.angles).tolist()}
    want = sum(1 for a in uq if (ff.get_urey_bradley(*mol.atomtype[list(a)]) or (0.0,))[0] > 0)
    assert want > 0 and len(par.ub_params["idx"]) == want
    pos = torch.tensor(x[None], dtype=dtype, device=DEV)
    box = torch.zeros(1, 3, 3, dtype=dtype, device=DEV)
    F = torch.zeros_like(pos)
    f = Forces(par, terms=["angles"])
    E = f.compute(pos, box, F, returnDetails=True)[0]
    ang = par.angle_params
    Eo, Fo = oracle(par, pos, box)
    from oracle import refmd

    par64 = ala2_charmm(inputs, torch.float64, C36_TERMS, device="cpu")[0]
    of = refmd.OracleForces(par64, ["angles"])
    Fa = torch.zeros(pos.shape, dtype=torch.float64)
    Ea = of.compute(pos.cpu().double(), box.cpu().double(), Fa)[0]["angles"]
    assert ang is not None
    tot = Fa.numpy()[0] + Fo[0]
    scale = np.abs(tot).max()
    err = np.abs(F.double().cpu().numpy()[0] - tot).max()
    assert err <= (1e-9 if dtype == torch.float64 else 1e-5) * max(1.0, scale), err
    assert abs(E["angles"] - (Ea + Eo[0])) <= (1e-9 if dtype == torch.float64 else 1e-5) * max(1.0, abs(Ea + Eo[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_charmm36_ala2_against_oracle(tmp_path, dtype):
    charmm36_ala2(reference_inputs_dir(tmp_path), dtype)


@pytest.mark.gpu
def test_charmm36_ala2_fp64_nve_with_ub(tmp_path):
    """fp64, vacuum, 0.5 fs, 2000 steps from 100 K: E_tot fluctuates no more with Urey-Bradley than 1.1 x without."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann

    inputs = reference_inputs_dir(tmp_path)
    spread = {}
    for with_ub in (False, True):
        terms = C36_TERMS if with_ub else [t for t in C36_TERMS if t != "ureybradley"]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            par, _, _, x = ala2_charmm(inputs, torch.float64, terms)
        s = System(len(x), 1, torch.float64, DEV)
        s.set_positions(x)
        s.set_box(np.zeros(3))
        f = Forces(par, terms=C36_FORCES)
        torch.manual_seed(0)
        s.set_velocities(maxwell_boltzmann(par.masses, 100.0, 1))
        f.compute(s.pos, s.box, s.forces)
        integ = Integrator(s, f, 0.5, DEV)
        integ.step(400)
        etot = []
        for _ in range(40):
            ek, ep, _ = integ.step(50)
            etot.append(float(ek[0] + ep[0]))
        spread[with_ub] = float(np.std(etot))
    print("E_tot std without / with Urey-Bradley:", spread)
    assert spread[True] <= 1.1 * spread[False], spread
