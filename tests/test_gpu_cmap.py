"""CMAP correction maps on the GPU against the fp64 numpy oracle (oracle/cmap.py), on every path that evaluates bonded
terms.  tests/test_cmap_on_interpreter.py runs most of these functions on the host interpreter build of the kernels.

Test systems: the fixture's own topology with CMAP terms added.  ala2 gets its backbone term
C(ACE)-N-CA-C-N(NME), atoms 4, 6, 8, 14, 16 of its prmtop (found by ATOM_NAME in test_cmap_host.py).  Other fixtures get
terms picked by a fixed rule that does not need residue names: the unique proper dihedrals (a, b, c, d) of the fixture
in their stored order, every ``stride``-th one (about one dihedral per 16 atoms), each extended by the lowest-index bonded
neighbour e of d that is not a, b or c; dihedrals whose d has no such neighbour are skipped (thrombin: 138 terms).  The rule need not find
the true backbone: the kernels evaluate any five bonded atoms the same way.  Terms alternate between two asymmetric
maps (E(phi, psi) != E(psi, phi), != E(-phi, -psi)), so a swapped axis, a shifted origin or a flipped sign shows up.
"""
import math

import numpy as np
import pytest
import torch

from conftest import golden_cfg, golden_system_tensors, load_golden, params_from_golden
from oracle import cmap as ocmap

DEV = "cuda"
ALA2_BACKBONE = [4, 6, 8, 14, 16]


def asym_map(n=24, which=0):
    a = -math.pi + 2 * math.pi * np.arange(n) / n
    phi, psi = np.meshgrid(a, a, indexing="ij")
    if which == 0:
        return np.cos(phi) + 0.5 * np.sin(2 * psi + 0.3) + 0.2 * np.cos(phi - psi)
    return 0.8 * np.sin(phi) * np.cos(psi) + 0.3 * np.sin(3 * psi - phi) - 0.4 * np.sin(psi)


def cmap_terms(g, name):
    """(idx (n,5), map_of (n,)) for fixture g, by the module docstring's rule."""
    if name.startswith("ala2"):
        idx = np.array([ALA2_BACKBONE], np.int64)
    else:
        n = len(g["par_masses"])
        nbr = [set() for _ in range(n)]
        for a, b in g["par_bond_idx"]:
            nbr[int(a)].add(int(b))
            nbr[int(b)].add(int(a))
        dih = np.asarray(g["par_dihedral_idx"], np.int64)
        stride = max(1, len(dih) * 16 // n)
        rows = []
        for a, b, c, d in dih[::stride]:
            e = sorted(nbr[int(d)] - {int(a), int(b), int(c)})
            if e:
                rows.append([a, b, c, d, e[0]])
        idx = np.array(rows, np.int64)
    return idx, np.arange(len(idx)) % 2


def make_params(g, name, precision, cmap_only=False, with_cmap=True):
    """params_from_golden with CMAP terms (two 24x24 maps); ``cmap_only``: no other bonded term."""
    from torchmd_b200.parameters import TopologyParameters

    base = params_from_golden(g, precision=precision)
    idx, map_of = cmap_terms(g, name)
    cmaps = (idx, map_of, [24, 24], [asym_map(24, 0), asym_map(24, 1)]) if with_cmap else None
    se = g["par_lj_sigma_eps"]

    def term(k):
        return None if cmap_only or "par_" + k + "_idx" not in g else (g["par_" + k + "_idx"], g["par_" + k + "_map"], g["par_" + k + "_params"])

    par = TopologyParameters(atom_types=g["par_types"], type_sigma=se[:, 0], type_epsilon=se[:, 1], charges=g["par_charges"],
                             masses=g["par_masses"], bonds=term("bond"), angles=term("angle"), dihedrals=term("dihedral"),
                             impropers=term("improper"), pairs14=term("nonbonded_14"), cmaps=cmaps, precision=precision, device=DEV)
    assert base.natoms == par.natoms
    return par


def oracle(par, pos, box):
    """(E (R,), F (R,N,3)) of the CMAP terms alone, fp64, from the positions as the kernels see them."""
    c = par.cmap_params
    args = [c[k].cpu().numpy() for k in ("idx", "map_of", "res", "grids")]
    Es, Fs = [], []
    for r in range(pos.shape[0]):
        L = torch.diagonal(box[r]).double().cpu().numpy()
        e, f = ocmap.energy_forces(pos[r].double().cpu().numpy(), *args, box=L if L.any() else None)
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


def cmap_only_forces(name, dtype, pos=None, box=None):
    """Forces(terms=["dihedrals"]) on the CMAP terms alone against the oracle; returns (E, F) of the kernels."""
    from torchmd_b200 import Forces

    g = load_golden(name)
    par = make_params(g, name, dtype, cmap_only=True)
    if pos is None:
        pos, box = golden_system_tensors(g, dtype, DEV)
    f = Forces(par, terms=["dihedrals"], **golden_cfg(g))
    F = torch.zeros_like(pos)
    E = f.compute(pos, box, F, returnDetails=True)
    Eo, Fo = oracle(par, pos, box)
    assert_close(F, Fo, dtype, f"{name} {dtype}")
    for r in range(pos.shape[0]):
        assert abs(E[r]["dihedrals"] - Eo[r]) <= 1e-10 * max(1.0, abs(Eo[r])), (E[r]["dihedrals"], Eo[r])
    return E, F


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "thrombin_nobox_rf"])
def test_cmap_against_oracle(name, dtype):
    cmap_only_forces(name, dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_replicas_and_angles_at_the_seam(dtype):
    """Three replicas with different geometries; in one, atoms moved so that phi and psi sit within 1e-6 rad of +-180."""
    g = load_golden("ala2_xsc_rf")
    pos, box = golden_system_tensors(g, torch.float64, "cpu")
    pos = pos[:1].repeat(3, 1, 1).clone()
    box = box[:1].repeat(3, 1, 1).clone()
    rng = np.random.default_rng(5)
    pos[1] += torch.tensor(rng.normal(scale=0.15, size=pos[1].shape))
    pos[2] = torch.tensor(seam_geometry(pos[2].numpy(), ALA2_BACKBONE, math.pi - 5e-7, -math.pi + 5e-7))
    cmap_only_forces("ala2_xsc_rf", dtype, pos.to(dtype).to(DEV).contiguous(), box.to(dtype).to(DEV).contiguous())


def place_chain(phi, psi):
    """Five atoms of a chain with 1.5 A bonds, 110 deg angles and IUPAC dihedrals phi (atoms 0-3) and psi (1-4)."""
    x = [np.array([0.0, 0.0, 0.0]), np.array([1.5, 0.0, 0.0])]
    t = math.radians(110.0)
    x.append(x[1] + 1.5 * np.array([-math.cos(t), math.sin(t), 0.0]))
    for tors in (phi, psi):  # NeRF: the next atom from the last three and the dihedral
        a, b, c = x[-3], x[-2], x[-1]
        bc = (c - b) / np.linalg.norm(c - b)
        n = np.cross(b - a, bc)
        n /= np.linalg.norm(n)
        m = np.cross(n, bc)
        d2 = 1.5 * np.array([-math.cos(t), math.sin(t) * math.cos(tors), math.sin(t) * math.sin(tors)])
        x.append(c + d2[0] * bc + d2[1] * m + d2[2] * n)
    return np.array(x)


def seam_geometry(pos, atoms, phi, psi):
    """pos with the five atoms replaced by a chain at (phi, psi), placed where the first one was."""
    p = pos.copy()
    p[atoms] = place_chain(phi, psi) + pos[atoms[0]]
    return p


def sign_check(dtype):
    """A chain at IUPAC phi = +60 deg, psi = -45 deg gives E(+60, -45) of an asymmetric map (kernels and oracle)."""
    from torchmd_b200 import Forces
    from torchmd_b200.parameters import TopologyParameters

    x = place_chain(math.radians(60.0), math.radians(-45.0))
    phi, _ = ocmap.dihedral(x[None, 0], x[None, 1], x[None, 2], x[None, 3])
    psi, _ = ocmap.dihedral(x[None, 1], x[None, 2], x[None, 3], x[None, 4])
    assert abs(math.degrees(phi[0]) - 60.0) < 1e-9 and abs(math.degrees(psi[0]) + 45.0) < 1e-9
    grid = asym_map(24, 0)
    par = TopologyParameters(atom_types=np.zeros(5, np.int64), type_sigma=[1.0], type_epsilon=[0.0], charges=np.zeros(5),
                             masses=np.ones(5), cmaps=([[0, 1, 2, 3, 4]], [0], [24], [grid]), precision=dtype, device=DEV)
    pos = torch.tensor(x[None], dtype=dtype, device=DEV)
    f = Forces(par, terms=["dihedrals"])
    E = f.compute(pos, torch.zeros(1, 3, 3, dtype=dtype, device=DEV), torch.zeros_like(pos), returnDetails=True)[0]["dihedrals"]
    want = ocmap.map_energy(ocmap.coefficients(grid), math.radians(60.0), math.radians(-45.0))[0]
    wrong = ocmap.map_energy(ocmap.coefficients(grid), math.radians(-60.0), math.radians(45.0))[0]
    assert abs(want - wrong) > 0.3
    tol = 1e-10 if dtype == torch.float64 else 1e-5  # (fp32: the positions' rounding moves the angles)
    assert abs(E - float(want)) < tol, (E, float(want), float(wrong))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_angle_sign_is_iupac(dtype):
    sign_check(dtype)


def dihedral_slot_sums(name, dtype):
    """With the fixture's own torsions and CMAP terms, the dihedral slot is the sum of both; the forces add up."""
    from torchmd_b200 import Forces

    g = load_golden(name)
    pos, box = golden_system_tensors(g, dtype, DEV)
    terms = [str(t) for t in g["terms"]]
    out = {}
    for with_cmap in (False, True):
        par = make_params(g, name, dtype, with_cmap=with_cmap)
        f = Forces(par, terms=terms, **golden_cfg(g))
        F = torch.zeros_like(pos)
        out[with_cmap] = (f.compute(pos, box, F, returnDetails=True), F.double().cpu().numpy(), par)
    Eo, Fo = oracle(out[True][2], pos, box)
    for r in range(pos.shape[0]):
        e0, e1 = out[False][0][r], out[True][0][r]
        assert abs(e1["dihedrals"] - (e0["dihedrals"] + Eo[r])) <= 1e-9 * max(1.0, abs(e1["dihedrals"]))
        for k in e0:  # (the cluster path's unordered reductions move the last bits of the pair terms between runs)
            if k != "dihedrals":
                assert abs(e0[k] - e1[k]) <= 1e-9 * max(1.0, abs(e0[k])), k
    Fw, Fwo = out[True][1], out[False][1]
    if dtype == torch.float64:
        assert np.abs(Fw - Fwo - Fo).max() <= 1e-10 * np.abs(Fw).max()
    else:
        assert np.abs(Fw - Fwo - Fo).max() <= 2.0**-20 * np.abs(Fw).max()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "chain_amber_periodic"])
def test_dihedral_slot_holds_torsions_and_cmap(name, dtype):
    dihedral_slot_sums(name, dtype)


def invariance_and_determinism(name):
    """fp64: net force and net torque vanish; two runs are bitwise equal."""
    E, F = cmap_only_forces(name, torch.float64)
    _, F2 = cmap_only_forces(name, torch.float64)
    assert torch.equal(F, F2)
    g = load_golden(name)
    pos, _ = golden_system_tensors(g, torch.float64, "cpu")
    Fn = F.cpu().numpy()[0]
    scale = np.abs(Fn).max()
    assert np.abs(Fn.sum(0)).max() <= 1e-9 * max(1.0, scale)
    if not g["box"].any():  # (a periodic fixture's terms may straddle the box: the torque needs unwrapped positions)
        torque = np.cross(pos[0].numpy(), Fn).sum(0)
        assert np.abs(torque).max() <= 1e-9 * max(1.0, scale * np.abs(pos[0].numpy()).max())


@pytest.mark.gpu
def test_net_force_torque_and_determinism():
    invariance_and_determinism("thrombin_nobox_rf")


def paths_agree(name, env_sets, monkeypatch, dtype=torch.float32):
    """The same system with and without CMAP under each environment setting: the difference of the forces is the
    oracle's CMAP force within the fp32 rounding of the two totals (and, on the cluster path, whose unordered reductions
    move the last bits of the pair forces between runs, within 2^-20 of the largest force), the forces a captured step
    leaves include the CMAP terms, and the launches per captured step are the same with and without CMAP."""
    from torchmd_b200 import Forces, Integrator, System

    g = load_golden(name)
    terms = [str(t) for t in g["terms"]]
    pos, box = golden_system_tensors(g, dtype, DEV)
    Fo = oracle(make_params(g, name, torch.float64), pos, box)[1]
    for env in env_sets:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        launches, forces = {}, {}
        for with_cmap in (True, False):
            par = make_params(g, name, dtype, with_cmap=with_cmap)
            f = Forces(par, terms=terms, **golden_cfg(g))
            F = torch.zeros_like(pos)
            f.compute(pos, box, F)
            forces[with_cmap] = F.double().cpu().numpy()
            s = System(pos.shape[1], pos.shape[0], dtype, DEV)
            s.set_positions(pos[0].cpu().numpy())
            s.set_box(torch.diagonal(box[0]).cpu().numpy())
            integ = Integrator(s, f, 0.5, DEV)
            integ.step(2)
            n0 = f.stats()["kernel_launches"]
            integ.step(3)
            launches[with_cmap] = f.stats()["kernel_launches"] - n0
            F2 = torch.zeros_like(s.forces)
            f.compute(s.pos, s.box, F2)
            step_err = (s.forces.double() - F2.double()).abs().max().item()
            assert step_err <= 1e-5 * max(1.0, F2.abs().max().item()), (env, with_cmap, step_err)
        assert launches[True] == launches[False], (env, launches)
        Fw, Fwo = forces[True], forces[False]
        slack = 2.0**-20 * np.abs(Fw).max() if env.get("TMD_B200_CLUSTER", "0") == "1" else 1e-12 * np.abs(Fo).max()
        bad = np.abs(Fw - Fwo - Fo) > 2.0**-23 * (np.abs(Fw) + np.abs(Fwo)) + slack
        assert not bad.any(), (env, np.abs(Fw - Fwo - Fo).max())


ENV_SETS = [{"TMD_B200_CLUSTER": c, "TMD_B200_OVERLAP": o, "TMD_B200_GRAPH": gr, "TMD_B200_FUSEPREP": fp}
            for c in "01" for o in "01" for gr, fp in (("0", "0"), ("1", "1"), ("1", "0"))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ala2_xsc_rf", "thrombin_nobox_rf"])
def test_switches_agree_and_launch_counts_unchanged(name, monkeypatch):
    paths_agree(name, ENV_SETS, monkeypatch)


@pytest.mark.gpu
def test_fp64_nve_energy_conservation_with_cmap():
    """thrombin in vacuum with the fixture's settings, fp64, 1 fs, 2000 steps: E_tot fluctuates no more with CMAP than
    1.1 x without."""
    from torchmd_b200 import Forces, Integrator, System, maxwell_boltzmann

    g = load_golden("thrombin_nobox_rf")
    terms = [str(t) for t in g["terms"]]
    spread = {}
    for with_cmap in (False, True):
        par = make_params(g, "thrombin_nobox_rf", torch.float64, with_cmap=with_cmap)
        pos, box = golden_system_tensors(g, torch.float64, DEV)
        s = System(pos.shape[1], 1, torch.float64, DEV)
        s.set_positions(pos[0].cpu().numpy())
        s.set_box(torch.diagonal(box[0]).cpu().numpy())
        f = Forces(par, terms=terms, **golden_cfg(g))
        torch.manual_seed(0)
        s.set_velocities(maxwell_boltzmann(par.masses, 100.0, 1))
        integ = Integrator(s, f, 1.0, DEV)
        f.compute(s.pos, s.box, s.forces)
        integ.step(200)  # settle the start
        etot = []
        for _ in range(40):
            ek, ep, _ = integ.step(50)
            etot.append(float(ek[0] + ep[0]))
        spread[with_cmap] = float(np.std(etot))
    print("E_tot std without / with CMAP:", spread)
    assert spread[True] <= 1.1 * spread[False], spread


@pytest.mark.gpu
def test_barostat_run_with_cmap():
    """An NPT Integrator with CMAP terms runs; its E_pot equals a fresh Forces.compute sum."""
    from torchmd_b200 import Forces, Integrator, MonteCarloBarostat, System, maxwell_boltzmann

    name = "chain_amber_periodic"
    g = load_golden(name)
    terms = [str(t) for t in g["terms"]]
    par = make_params(g, name, torch.float32)
    pos, box = golden_system_tensors(g, torch.float32, DEV)
    s = System(pos.shape[1], 1, torch.float32, DEV)
    s.set_positions(pos[0].cpu().numpy())
    s.set_box(torch.diagonal(box[0]).cpu().numpy())
    f = Forces(par, terms=terms, **golden_cfg(g))
    torch.manual_seed(0)
    s.set_velocities(maxwell_boltzmann(par.masses, 300.0, 1))
    f.compute(s.pos, s.box, s.forces)
    integ = Integrator(s, f, 1.0, DEV, gamma=1.0, T=300.0, barostat=MonteCarloBarostat(1.0, 300.0, frequency=5, seed=1))
    _, ep, _ = integ.step(20)
    F = torch.zeros_like(s.pos)
    E = f.compute(s.pos, s.box, F)
    assert abs(float(ep[0]) - float(E[0])) <= 1e-4 * max(1.0, abs(float(ep[0])))
