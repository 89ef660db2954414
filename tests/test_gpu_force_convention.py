"""The two force conventions of ``Forces.compute`` on every pair kernel, and forces as the gradient of the kernels' own
energies.  tests/test_force_convention_on_interpreter.py runs these functions on the host interpreter build of the
kernels.

The explicit convention (the default, what MD integrates) is the reference's switched-LJ force s dE/dr + E s'/r, which
is not the derivative of the energy; the exact-gradient one (``explicit_forces=False``, ``Epot.sum().backward()``,
``torch.vmap``, ``minimize_pytorch_bfgs``) is s dE/dr + E s'.  Both are switched per call on one context, so every
kernel must honour whichever convention the call asks for, whatever the context ran before, and the pair path a
context takes must not depend on the convention of its first call.

* ``convention_orders``: each pair kernel 0-10 (tmd_pair_kernel), picked with TMD_B200_CLUSTER / TMD_B200_FX, a box or
  none, fp32 or fp64, PME or not, runs explicit -> exact -> explicit and exact -> explicit -> exact on one ``Forces``;
  every call matches the fp64 oracle of its convention (refmd.OracleForces(true_gradient=...), oracle/pme.py for the
  reciprocal part) on the fp32 pair set, within the bounds of test_gpu_cluster_systems.py (fp32 1e-4 kcal/mol/A,
  5e-4 with PME, both scaled by |F|max / 100 above 100 kcal/mol/A; fp64 1e-9 of the largest force).  The fp32x2
  full-row kernels (2, 3, 9) have no exact-gradient instantiation and take 1, 0, 7 for those calls.
* ``autograd_surfaces_after_explicit``: backward, vmap and one L-BFGS evaluation on a cluster-path system after an
  explicit compute on the same ``Forces``, then MD that must follow the trajectory of a context that never took the
  autograd pass.
* ``finite_differences``: F = -dE/dx by central differences of the kernels' own fp64 energies, one displaced copy of the
  system per replica (replica 2k is x + h e_k, 2k+1 is x - h e_k, the last one x), per term and all terms together;
  no oracle involved.  A sample whose displacement moves a pair across the cutoff or a CMAP angle across a map-cell
  edge is skipped (those energies are not differentiable there).  The same on the fp32 cluster kernels in the exact
  convention with h = 1e-2 A, within FD32_TOL.
"""
import math

import numpy as np
import pytest
import torch

import test_gpu_cluster_systems as G
from conftest import load_golden
from oracle import refmd
from torchmd_b200._lib import (PAIR_CLUSTER, PAIR_EWALD, PAIR_EWALD_CLUSTER, PAIR_EWALD_F64, PAIR_EWALD_FX, PAIR_EWALD_FX2,
                               PAIR_F64, PAIR_OPEN_FX2, PAIR_ROWS, PAIR_ROWS_FX, PAIR_ROWS_FX2)

pytestmark = [pytest.mark.gpu]
DEV = "cuda:0"
F32, F64 = torch.float32, torch.float64
FD_H64, FD_REL64 = 1e-5, 1e-6  # fp64 central differences: step (A) and bound relative to max(1, |F|)
FD_H32 = 1e-2
# fp32 cluster kernels, h = 1e-2 A, tiled water (cutoff 5, switch 4, RF): the largest |FD - F| measured was 1.5e-2
# kcal/mol/A on an H100 (24 of 32 samples kept) and 4.2e-3 on the interpreter (3 of 4), mostly the fp32 rounding of
# the per-cluster energy sums over 2h; the explicit-convention forces are up to 0.27 away from the gradient there
FD32_TOL = 4e-2


def _L():
    from torchmd_b200 import _lib

    return _lib.lib()


def _kernel(forces):
    return _L().tmd_pair_kernel(forces._ctx)


# ---------------------------------------------------------------------------------------------------- systems
def golden_spec(name, **over):
    from torchmd_b200 import testsystems

    par, c0, L0, terms, cfg = testsystems.golden_system(name, precision=F64)
    return G._spec_of(par, c0, L0, terms, dict(cfg, **over), name)


def water(t=2):
    """The 999-atom water box tiled t^3 times, cutoff 5, switch 4, RF: the cluster path at t >= 2."""
    return G.water_spec(G.tiled_water(t))


def system_of(key):
    if key == "water_x2":
        return water(2)
    if key == "protein_x2":
        return G.protein(2)
    if key == "chain_plain":  # plain cut-off Coulomb, LJ switched
        return golden_spec("chain_amber_periodic", rfa=False)
    return golden_spec(key)


# (case id, system, environment, dtype, pme, kernel of an explicit call, kernel of an exact-gradient call)
NOCL = {"TMD_B200_CLUSTER": "0"}
MATRIX = [
    ("k0_open", "ala2_nobox_rf", dict(NOCL, TMD_B200_FX="0"), F32, False, PAIR_ROWS, PAIR_ROWS),
    ("k0_box_plain", "chain_plain", dict(NOCL, TMD_B200_FX="0"), F32, False, PAIR_ROWS, PAIR_ROWS),
    ("k1", "chain_amber_periodic", dict(NOCL, TMD_B200_FX="1"), F32, False, PAIR_ROWS_FX, PAIR_ROWS_FX),
    ("k2", "chain_amber_periodic", dict(NOCL, TMD_B200_FX="2"), F32, False, PAIR_ROWS_FX2, PAIR_ROWS_FX),
    ("k2_plain", "chain_plain", dict(NOCL, TMD_B200_FX="2"), F32, False, PAIR_ROWS_FX2, PAIR_ROWS_FX),
    ("k3", "ala2_nobox_rf", dict(NOCL, TMD_B200_FX="2"), F32, False, PAIR_OPEN_FX2, PAIR_ROWS),
    ("k4_open", "ala2_nobox_rf", {"TMD_B200_CLUSTER": "1"}, F32, False, PAIR_CLUSTER, PAIR_CLUSTER),
    ("k4_water", "water_x2", {"TMD_B200_CLUSTER": "1"}, F32, False, PAIR_CLUSTER, PAIR_CLUSTER),
    ("k4_protein", "protein_x2", {"TMD_B200_CLUSTER": "1"}, F32, False, PAIR_CLUSTER, PAIR_CLUSTER),
    ("k5", "chain_amber_periodic", {}, F64, False, PAIR_F64, PAIR_F64),
    ("k5_plain", "chain_plain", {}, F64, False, PAIR_F64, PAIR_F64),
    ("k6", "chain_amber_periodic", dict(NOCL, TMD_B200_FX="0"), F32, True, PAIR_EWALD, PAIR_EWALD),
    ("k7", "chain_amber_periodic", dict(NOCL, TMD_B200_FX="1"), F32, True, PAIR_EWALD_FX, PAIR_EWALD_FX),
    ("k8", "chain_amber_periodic", {}, F64, True, PAIR_EWALD_F64, PAIR_EWALD_F64),
    ("k9", "chain_amber_periodic", dict(NOCL, TMD_B200_FX="2"), F32, True, PAIR_EWALD_FX2, PAIR_EWALD_FX),
    ("k10_water", "water_x2", {"TMD_B200_CLUSTER": "1"}, F32, True, PAIR_EWALD_CLUSTER, PAIR_EWALD_CLUSTER),
    ("k10_protein", "protein_x2", {"TMD_B200_CLUSTER": "1"}, F32, True, PAIR_EWALD_CLUSTER, PAIR_EWALD_CLUSTER),
]
CASES = {c[0]: c[1:] for c in MATRIX}


# ---------------------------------------------------------------------------------------------------- oracles
def oracle(spec, pos, box, dtype, exact, pme_params=None):
    """fp64 forces (R,N,3) and energies of the convention ``exact``, deciding pairs in ``dtype``.  With PME
    (``pme_params`` = (alpha, grid)): test_gpu_pme's oracle (explicit) plus the switched-LJ difference of the two
    conventions, the only term where they differ."""
    cfg = G._ocfg(spec)
    par = G.oracle_params(spec, dtype)
    pos64, box64 = pos.detach().cpu().double(), box.detach().cpu().double()
    if pme_params is None:
        F = torch.zeros_like(pos64)
        E = refmd.OracleForces(par, spec["terms"], decision_dtype=dtype, true_gradient=exact, **cfg).compute(pos64, box64, F)
        return F.numpy(), E
    from test_gpu_pme import _oracle as pme_oracle

    cfg.pop("rfa", None)
    E, F = pme_oracle(par, spec["terms"], cfg, pos64.numpy(), torch.diagonal(box64, dim1=1, dim2=2).numpy(), *pme_params, dtype)
    if exact and "lj" in spec["terms"]:
        for tg, sign in ((True, 1.0), (False, -1.0)):
            Fl = torch.zeros_like(pos64)
            refmd.OracleForces(par, ["lj"], decision_dtype=dtype, true_gradient=tg, **cfg).compute(pos64, box64, Fl)
            F = F + sign * Fl.numpy()
    return F, E


def assert_matches(spec, F, E, Fo, Eo, dtype, pme, what):
    err = np.abs(F.detach().cpu().double().numpy() - Fo).max()
    fmax = np.abs(Fo).max()
    # (fp32: the bound of test_gpu_ub_nbfix for systems whose largest force exceeds 100 kcal/mol/A, e.g. 1,100 on the
    #  chain fixture: the rounding of a pair force grows with it)
    tol = 1e-9 * max(1.0, fmax) if dtype == F64 else (5e-4 if pme else 1e-4) * max(1.0, fmax / 100.0)
    print(f"{what}: max|dF| vs fp64 oracle {err:.3e} (max |F| {fmax:.1f})")
    assert err <= tol, (what, err, tol)
    for r in range(len(Eo)):
        for k in spec["terms"]:
            e, eo = float(E[r][k]), float(Eo[r][k])
            if dtype == F64:
                bound = 1e-9 * max(1.0, abs(eo))
            else:
                bound = 2e-5 * max(1.0, abs(eo)) if pme else 1e-5 * abs(eo) + 2e-3
            assert abs(e - eo) <= bound, (what, r, k, e, eo)


# ---------------------------------------------------------------------------------------------------- 1a: the matrix
def convention_orders(case, monkeypatch):
    """Both orders of the two conventions on one Forces per order, each call against the oracle of its convention; the
    kernel of every call is the intended one and that of the last explicit call is a fresh explicit context's."""
    from torchmd_b200 import Forces

    key, env, dtype, pme, k_explicit, k_exact = CASES[case]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    spec = system_of(key)
    cfg = dict(spec["cfg"])
    if pme:
        cfg.pop("rfa", None)
    pos = torch.tensor(spec["coords"][None], dtype=dtype, device=DEV)
    box = torch.diag_embed(torch.tensor(spec["box"][None], dtype=dtype, device=DEV))
    fresh = Forces(G.params(spec, dtype, DEV), terms=spec["terms"], pme=pme, **cfg)
    fresh.compute(pos, box, torch.zeros_like(pos))
    assert _kernel(fresh) == k_explicit, (case, _kernel(fresh))
    pme_params = fresh.pme_parameters() if pme else None
    decide = F32 if dtype == F32 else F64
    want = {ex: oracle(spec, pos, box, decide, ex, pme_params) for ex in (False, True)}
    for order in ((False, True, False), (True, False, True)):
        forces = Forces(G.params(spec, dtype, DEV), terms=spec["terms"], pme=pme, **cfg)
        for n, exact in enumerate(order):
            F = torch.full_like(pos, 7.0)
            p = pos.detach().clone().requires_grad_(exact)
            E = forces.compute(p, box, F, returnDetails=True, explicit_forces=not exact)
            kern = _kernel(forces)
            what = f"{case} order {['explicit', 'exact'][order[0]]}-first, call {n} ({'exact' if exact else 'explicit'}), kernel {kern}"
            assert kern == (k_exact if exact else k_explicit), what
            assert_matches(spec, F, E, *want[exact], dtype, pme, what)
        if not order[-1]:
            assert _kernel(forces) == _kernel(fresh)


def big_water_orders(t=3, nsample=300):
    """The tiled water box at t = 3 (8,991 waters) on the cluster kernel, both orders, against the sampled oracle rows
    (the all-pairs oracle cannot hold it)."""
    from torchmd_b200 import Forces

    spec = water(t)
    spec["terms"] = ["lj", "electrostatics"]
    pos = torch.tensor(spec["coords"][None], dtype=F32, device=DEV)
    box = torch.diag_embed(torch.tensor(spec["box"][None], dtype=F32, device=DEV))
    atoms = sorted(np.random.default_rng(11).choice(pos.shape[1], nsample, replace=False).tolist())
    cfg = G._ocfg(spec)
    want = {ex: refmd.sampled_rows(G.oracle_params(spec), spec["terms"], pos[0].cpu().double(), torch.diagonal(box[0]).cpu().double(),
                                   atoms, chunk=48, true_gradient=ex, **cfg)[0].numpy() for ex in (False, True)}
    for order in ((False, True, False), (True, False, True)):
        forces = Forces(G.params(spec, F32, DEV), terms=spec["terms"], **spec["cfg"])
        for exact in order:
            F = torch.zeros_like(pos)
            forces.compute(pos.detach().clone().requires_grad_(exact), box, F, explicit_forces=not exact)
            assert _kernel(forces) == PAIR_CLUSTER
            err = np.abs(F[0].cpu().double().numpy()[atoms] - want[exact]).max()
            print(f"water x{t}^3, {order}, exact={exact}: {nsample} sampled atoms, max|dF| {err:.3e}")
            assert err < 1e-4, (order, exact, err)


@pytest.mark.parametrize("case", list(CASES))
def test_both_convention_orders_on_every_pair_kernel(case, monkeypatch):
    convention_orders(case, monkeypatch)


def test_both_convention_orders_on_a_large_water_box():
    big_water_orders()


# ---------------------------------------------------------------------------------------------------- 1b: autograd
def autograd_surfaces_after_explicit(spec, monkeypatch, nsteps=20, batch=2):
    """On a cluster-path system, after an explicit compute on the same Forces: Epot.sum().backward(), torch.vmap over a
    batch and one minimize_pytorch_bfgs evaluation give -(exact-gradient oracle); MD afterwards follows the
    trajectory of a context that never took the autograd pass."""
    from torchmd_b200 import Integrator
    from torchmd_b200.minimizers import minimize_pytorch_bfgs

    monkeypatch.setenv("TMD_B200_CLUSTER", "1")
    pos = torch.tensor(spec["coords"][None], dtype=F32, device=DEV)
    box = torch.diag_embed(torch.tensor(spec["box"][None], dtype=F32, device=DEV))
    Fo, Eo = oracle(spec, pos, box, F32, True)
    Fo_explicit = oracle(spec, pos, box, F32, False)[0]
    tol = 1e-4

    def check(grad, what):
        err = np.abs(-grad.detach().cpu().double().numpy() - Fo).max()
        print(f"{what}: max|-dE/dx - F_oracle| {err:.3e}")
        assert err < tol, (what, err)

    def explicit_first(forces, p, b):
        F = torch.zeros_like(p)
        forces.compute(p, b, F)
        assert _kernel(forces) == PAIR_CLUSTER
        assert np.abs(F.cpu().double().numpy() - np.concatenate([Fo_explicit] * p.shape[0])).max() < tol

    # backward
    from torchmd_b200 import Forces

    par, system = G._md_system(spec)
    forces = Forces(par, terms=spec["terms"], **spec["cfg"])
    explicit_first(forces, pos, box)
    p = pos.detach().clone().requires_grad_(True)
    E = forces.compute(p, box, None, toNumpy=False, calculateForces=False, explicit_forces=False)
    E.sum().backward()
    assert _kernel(forces) == PAIR_CLUSTER
    check(p.grad, "backward after explicit")
    e_tot = sum(Eo[0][k] for k in spec["terms"])
    assert abs(float(E.detach()[0]) - e_tot) <= 1e-5 * abs(e_tot) + 2e-3

    # vmap: the batch folds into replicas, a context of that many replicas that computed explicit forces first
    posb, boxb = pos.repeat(batch, 1, 1), box.repeat(batch, 1, 1)
    explicit_first(forces, posb, boxb)
    xb = torch.stack([pos] * batch).requires_grad_(True)
    Eb = torch.vmap(forces.compute, in_dims=(0,))(xb, box=box, forces=None, returnDetails=False, explicit_forces=False,
                                                  calculateForces=False, toNumpy=False)
    Eb.sum().backward()
    assert _kernel(forces) == PAIR_CLUSTER
    for b in range(batch):
        check(xb.grad[b], f"vmap member {b}")

    # one L-BFGS evaluation: the gradient its closure back-propagates
    explicit_first(forces, system.pos, system.box)

    class Spy:
        def __init__(self):
            self.grads = []

        def compute(self, x, *a, **kw):
            x.register_hook(lambda g: self.grads.append(g.detach().clone()))
            return forces.compute(x, *a, **kw)

    spy = Spy()
    minimize_pytorch_bfgs(system, spy, steps=1, max_iter=1)
    assert len(spy.grads) == 1 and _kernel(forces) == PAIR_CLUSTER
    check(spy.grads[0], "minimize_pytorch_bfgs evaluation")

    # MD after the autograd passes against MD on a context that never took one
    out = []
    for autograd_first in (True, False):
        par, system = G._md_system(spec)
        forces = Forces(par, terms=spec["terms"], **dict(spec["cfg"], skin=0.5))
        explicit_first(forces, system.pos, system.box)
        if autograd_first:
            p = system.pos.detach().clone().requires_grad_(True)
            forces.compute(p, system.box, None, toNumpy=False, calculateForces=False, explicit_forces=False).sum().backward()
            check(p.grad, "backward before MD")
        integ = Integrator(system, forces, 1.0, DEV, gamma=None, T=None)
        _, pot, _ = integ.step(niter=nsteps)
        assert _kernel(forces) == PAIR_CLUSTER
        out.append((system.pos.clone(), system.vel.clone(), pot))
    dp = (out[0][0] - out[1][0]).abs().max().item()
    dv = (out[0][1] - out[1][1]).abs().max().item()
    print(f"NVE {nsteps} steps after the autograd pass vs without: max|dpos| {dp:.2e}, max|dvel| {dv:.2e}")
    assert dp < 1e-3 and dv < 1e-2, (dp, dv)
    assert abs(out[0][2][0] - out[1][2][0]) < 1e-5 * abs(out[1][2][0]) + 2e-2


def test_autograd_surfaces_after_explicit_forces_on_the_cluster_kernel(monkeypatch):
    autograd_surfaces_after_explicit(water(2), monkeypatch)


# ---------------------------------------------------------------------------------------------------- 1c: F = -dE/dx
def _angles(x, quads):
    """Dihedral angles (IUPAC sign, the kernels' convention) of the rows of ``quads`` (n,4) at positions x (..., N, 3)."""
    b0 = x[..., quads[:, 0], :] - x[..., quads[:, 1], :]
    b1 = x[..., quads[:, 2], :] - x[..., quads[:, 1], :]
    b2 = x[..., quads[:, 3], :] - x[..., quads[:, 2], :]
    n1, n2 = np.cross(b0, b1), np.cross(b1, b2)
    m = np.cross(n1, b1 / np.linalg.norm(b1, axis=-1, keepdims=True))
    return np.arctan2((m * n2).sum(-1), (n1 * n2).sum(-1))


def _crosses(x, a, axis, h, box, cutoff, cmap):
    """Whether moving atom a by +-h along ``axis`` carries a pair across the cutoff or a CMAP angle across a map cell."""
    xp, xm = x.copy(), x.copy()
    xp[a, axis] += h
    xm[a, axis] -= h
    if cutoff is not None:
        r = []
        for y in (xp, xm):
            d = y - y[a]
            if box.any():
                d -= box * np.round(d / box)
            r.append(np.linalg.norm(np.delete(d, a, 0), axis=1))
        if ((r[0] - cutoff) * (r[1] - cutoff) <= 0).any():
            return True
    if cmap is not None:
        idx, ngrid = cmap
        rows = idx[(idx == a).any(1)]
        if len(rows):
            for quads in (rows[:, :4], rows[:, 1:]):
                cell = [np.floor((_angles(y, quads) + math.pi) / (2 * math.pi / ngrid)) for y in (xp, xm)]
                if (cell[0] != cell[1]).any():
                    return True
    return False


def finite_differences(par, terms, cfg, x, box, dtype=F64, h=FD_H64, nsample=32, pme=False, cmap=None, seed=0,
                       tol=None, exact=True, what=""):
    """Central differences of the kernels' own energies against their forces (module docstring).  Returns the largest
    |FD - F| and the number of samples kept."""
    from torchmd_b200 import Forces

    x = np.asarray(x, np.float64)
    box = np.asarray(box, np.float64)
    N = len(x)
    rng = np.random.default_rng(seed)
    atoms, axes = rng.integers(0, N, nsample), rng.integers(0, 3, nsample)
    X = np.repeat(x[None], 2 * nsample + 1, 0)
    for k, (a, ax) in enumerate(zip(atoms, axes)):
        X[2 * k, a, ax] += h
        X[2 * k + 1, a, ax] -= h
    pos = torch.tensor(X, dtype=dtype, device=DEV)
    boxes = torch.diag_embed(torch.tensor(box, dtype=dtype, device=DEV).repeat(len(X), 1))
    forces = Forces(par, terms=terms, pme=pme, **cfg)
    F = torch.zeros_like(pos)
    E = forces.compute(pos.clone().requires_grad_(exact), boxes, F, explicit_forces=not exact)
    Xd = pos.cpu().double().numpy()  # (the displacements as the kernels received them)
    Fx = F[-1].cpu().double().numpy()
    fmax = max(1.0, np.abs(Fx).max())
    if tol is None:
        tol = FD_REL64 * fmax
    kept, worst = 0, 0.0
    for k, (a, ax) in enumerate(zip(atoms, axes)):
        if _crosses(Xd[-1], a, ax, h, box, cfg.get("cutoff"), cmap):
            continue
        kept += 1
        fd = -(E[2 * k] - E[2 * k + 1]) / (Xd[2 * k, a, ax] - Xd[2 * k + 1, a, ax])
        worst = max(worst, abs(fd - Fx[a, ax]))
    print(f"{what}: {kept}/{nsample} samples kept, max|FD - F| {worst:.3e} (max |F| {fmax:.1f}, bound {tol:.1e})")
    assert kept >= 0.75 * nsample, (what, kept)
    assert worst <= tol, (what, worst, tol)
    return worst, kept, forces, pos, boxes, E, atoms, axes, Xd


def ala2_params(g, precision):
    """ala2_xsc_rf's tables plus a Urey-Bradley term on every angle (test_gpu_ub_nbfix's rule) and a CMAP term on the
    backbone with test_gpu_cmap's asymmetric maps."""
    import test_gpu_cmap as CM
    import test_gpu_ub_nbfix as UB
    from conftest import golden_system_tensors
    from torchmd_b200.parameters import TopologyParameters

    pos, box = golden_system_tensors(g, F64)
    idx, prm = UB.ub_terms(g, pos[0].numpy(), torch.diagonal(box[0]).numpy())
    ub = (idx, np.stack([np.arange(len(idx)), np.arange(len(idx))], 1), prm)
    cidx, map_of = CM.cmap_terms(g, "ala2_xsc_rf")
    se = g["par_lj_sigma_eps"]

    def term(k):
        return (g["par_" + k + "_idx"], g["par_" + k + "_map"], g["par_" + k + "_params"])

    par = TopologyParameters(atom_types=g["par_types"], type_sigma=se[:, 0], type_epsilon=se[:, 1], charges=g["par_charges"],
                             masses=g["par_masses"], bonds=term("bond"), angles=term("angle"), dihedrals=term("dihedral"),
                             impropers=term("improper"), pairs14=term("nonbonded_14"), urey_bradley=ub,
                             cmaps=(cidx, map_of, [24, 24], [CM.asym_map(24, 0), CM.asym_map(24, 1)]), precision=precision,
                             device=DEV)
    return par, (np.asarray(cidx, np.int64), 24)


ALA2_TERMS = [["bonds"], ["angles"], ["dihedrals"], ["impropers"], ["dihedrals", "1-4"], ["lj"], ["electrostatics"],
              ["bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "electrostatics"]]


def ala2_gradient(terms, pme=False, nsample=32):
    """ala2_xsc_rf (periodic, cutoff 9, switch 7.5, RF or PME) with Urey-Bradley and CMAP terms."""
    from conftest import golden_cfg

    g = load_golden("ala2_xsc_rf")
    par, cmap = ala2_params(g, F64)
    cfg = golden_cfg(g)
    if pme:
        cfg.pop("rfa")
    return finite_differences(par, terms, cfg, g["coords"], np.asarray(g["box"]).ravel()[:3], pme=pme, cmap=cmap,
                              nsample=nsample, what=f"ala2 {'+'.join(terms)}{' PME' if pme else ''}")


def nbfix_gradient(inputs, terms, nsample=32):
    """The CHARMM water box with NBFIX (SOD-CLA), periodic, cutoff 7, switch 6, plain cut-off Coulomb."""
    import test_gpu_ub_nbfix as UB

    par, _, cfg, pos, box = UB.charmm_case(inputs, "waterbox_periodic", F64, True)
    return finite_differences(par, terms, cfg, pos[0], box, nsample=nsample, what=f"waterbox NBFIX {'+'.join(terms)}")


def repulsion_gradient(terms, nsample=32):
    from conftest import golden_cfg

    g = load_golden("argon100_lj_rep_mix")
    par = G.params(golden_spec("argon100_lj_rep_mix"), F64, DEV)
    return finite_differences(par, terms, golden_cfg(g), g["coords"], np.asarray(g["box"]).ravel()[:3], nsample=nsample,
                              what=f"argon {'+'.join(terms)}")


def charmm36_gradient(inputs, nsample=32):
    """CHARMM36 alanine dipeptide from its .prm, no box: its own Urey-Bradley terms and CMAP maps, every term."""
    import test_gpu_ub_nbfix as UB

    par, mol, _, x = UB.ala2_charmm(inputs, F64, UB.C36_TERMS)
    c = par.cmap_params
    assert c is not None and len(set(c["res"].tolist())) == 1
    cmap = (c["idx"].cpu().numpy(), int(c["res"][0]))
    return finite_differences(par, UB.C36_FORCES, {}, x, np.zeros(3), nsample=nsample, cmap=cmap, what="charmm36 ala2")


def cluster_gradient_fp32(nsample=32, t=2):
    """The fp32 cluster kernel in the exact-gradient convention: tiled water, pair terms, h = 1e-2 A."""
    spec = water(t)
    terms = ["lj", "electrostatics"]
    x = np.asarray(spec["coords"], np.float64)
    worst, kept, forces, pos, boxes, E, atoms, axes, Xd = finite_differences(
        G.params(spec, F32, DEV), terms, spec["cfg"], x, spec["box"], dtype=F32, h=FD_H32, nsample=nsample, tol=FD32_TOL,
        what=f"water x{t}^3 fp32 cluster, exact convention")
    # the explicit convention on the same samples, for contrast: a bound that it met would not test the convention
    Fe = torch.zeros_like(pos)
    forces.compute(pos, boxes, Fe)
    assert _kernel(forces) == PAIR_CLUSTER
    Fe = Fe[-1].cpu().double().numpy()
    fd = [-(E[2 * k] - E[2 * k + 1]) / (Xd[2 * k, a, ax] - Xd[2 * k + 1, a, ax]) for k, (a, ax) in enumerate(zip(atoms, axes))]
    far = max(abs(f - Fe[a, ax]) for f, a, ax in zip(fd, atoms, axes))
    print(f"explicit-convention forces: up to {far:.3e} from the same differences")
    if nsample >= 16:
        assert far > 2 * FD32_TOL, far
    return worst, kept


@pytest.mark.parametrize("terms", ALA2_TERMS, ids=["+".join(t) for t in ALA2_TERMS])
def test_forces_are_the_gradient_ala2(terms):
    ala2_gradient(terms)


def test_forces_are_the_gradient_pme():
    ala2_gradient(["electrostatics"], pme=True)
    ala2_gradient(["bonds", "angles", "dihedrals", "impropers", "1-4", "lj", "electrostatics"], pme=True)


@pytest.mark.parametrize("terms", [["lj"], ["electrostatics"], ["lj", "electrostatics", "bonds", "angles"]])
def test_forces_are_the_gradient_nbfix_plain_cutoff(tmp_path, terms):
    import test_gpu_ub_nbfix as UB

    nbfix_gradient(UB.reference_inputs_dir(tmp_path), terms)


@pytest.mark.parametrize("terms", [["repulsion"], ["repulsioncg"], ["lj", "repulsion", "repulsioncg"]])
def test_forces_are_the_gradient_repulsion(terms):
    repulsion_gradient(terms)


def test_forces_are_the_gradient_charmm36(tmp_path):
    import test_gpu_ub_nbfix as UB

    charmm36_gradient(UB.reference_inputs_dir(tmp_path))


def test_forces_are_the_gradient_fp32_cluster_kernel():
    cluster_gradient_fp32()
