"""``Forces`` with the interface of ``torchmd.forces.Forces`` (reference
``torchmd/forces.py:7-357``) computed by the sm_90a kernels behind
``libtmd_b200.so``.

Same constructor arguments, class attributes, error cases and return formats as
the reference, so ``torchmd/run.py:218-226,261`` and ``Integrator`` can use it
unchanged.  Differences that are deliberate:

* no O(N^2) pair table: exclusions go to the device as a CSR adjacency and the
  neighbour search is a cell list + Verlet list (``ava_idx`` is only
  materialised on request, for small systems);
* ``pos`` / ``forces`` must be CUDA contiguous tensors -- there is no CPU or
  stock-PyTorch fallback, a missing extension or a CPU tensor raises.  Their dtype is the
  run's precision: float32 ("precision: single") or float64 ("precision: double": fp64
  parameters, arithmetic and neighbour decisions, full neighbour rows, one GPU);
* energies are accumulated in fp64 on the device.
"""
import os

import numpy as np
import torch
from scipy import constants as _const

from . import _lib
from ._lib import ENERGY_SLOTS, NUM_ENERGIES

# forces.py:375-378 -- Coulomb constant from CODATA values, kcal*A/(mol*e^2)
ELEC_FACTOR = 1 / (4 * _const.pi * _const.epsilon_0)
ELEC_FACTOR *= _const.elementary_charge**2
ELEC_FACTOR /= _const.angstrom
ELEC_FACTOR *= _const.Avogadro / (_const.kilo * _const.calorie)

DEFAULT_SKIN = float(os.environ.get("TMD_B200_SKIN", "1.0"))


def _np(t, dtype):
    return np.ascontiguousarray(t.detach().cpu().numpy().astype(dtype))


def _exclusion_csr(natoms, pairs):
    """Symmetric CSR adjacency of the excluded pairs (replaces the N x N bool
    matrix of forces.py:348-357)."""
    if len(pairs) == 0:
        return np.zeros(natoms + 1, dtype=np.int64), np.zeros(0, dtype=np.int32)
    e = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    e = e[e[:, 0] != e[:, 1]]
    both = np.concatenate([e, e[:, ::-1]])
    both = np.unique(both, axis=0)  # sorted by row then column
    row_ptr = np.zeros(natoms + 1, dtype=np.int64)
    np.add.at(row_ptr, both[:, 0] + 1, 1)
    return np.cumsum(row_ptr), both[:, 1].astype(np.int32)


class Forces:
    """
    Parameters
    ----------
    parameters : object with the reference ``Parameters`` attribute layout
    terms : list of str, case-insensitive, from ``Forces.terms``.  ``"dihedrals"`` also turns on the CMAP
        correction maps the parameters carry (``cmap_params``, built by the parameter builders when asked for
        ``"cmap"``); their energy is part of the ``dihedrals`` energy.  ``"angles"`` likewise turns on the Urey-Bradley
        1-3 terms the parameters carry (``ub_params``, built when asked for ``"ureybradley"``); their energy is part of
        the ``angles`` energy.  With ``implicit_solvent``, ``"electrostatics"`` also holds both Generalized Born
        energies (polar and non-polar), as it holds PME's reciprocal energy.
    external : optional plugin exposing ``calculate(pos, box) -> (E (R,), F (R,N,3))``
    cutoff, rfa, solventDielectric, switch_dist, exclusions : as in the reference
    skin : Verlet-list buffer in Angstrom (not in the reference; results do not depend on it)
    pme : particle-mesh Ewald electrostatics (not in the reference): real space erfc(alpha r)/r on the cutoff's pair set,
        smooth PME (order-5 B-splines) in reciprocal space, minus erf(alpha r)/r of every excluded pair, minus the self
        and neutralising-background energies.  Needs "electrostatics", a cutoff, no reaction field, and a periodic box
        at least two cutoffs long on every axis.
    ewald_tolerance : the error tolerance delta that alpha and the grid are chosen from (OpenMM's convention);
        ``pme_parameters()`` reports them.  The real-space term is cut at the cutoff without a shift, so every pair
        crossing it changes the energy by k qi qj erfc(alpha rc) / rc: at the default 5e-4 an fp64 NVE run of rigid
        water at 2 fs keeps E_tot within 2.6 % of E_kin's fluctuation, at 1e-5 within 1.7 % (DESIGN.md 5b).  Runs
        that need tighter energy conservation should use a smaller tolerance.
    implicit_solvent : ``"obc2"`` for Generalized Born implicit solvent (OBC2, AMBER igb=5; not in the reference), or
        None.  Radii and screening factors come from ``parameters.gb_params`` (``amber_parameters(..., terms=[...,
        "gb"])`` reads them from a prmtop); the solvent dielectric is ``solventDielectric``, the solute's 1.  The polar
        energy -1/2 k (1 - 1/eps) sum_ij qi qj / f_GB over every pair (no exclusions, i = j included) and the
        non-polar term are part of the ``electrostatics`` energy, and the forces are their exact gradient through
        every Born radius.  Needs "electrostatics", no cutoff, no reaction field, no PME and an all-zero box.
    surface_tension : sigma of the ACE non-polar term sum_i 4 pi sigma (R_i + 1.4)^2 (R_i / B_i)^6, kcal/mol/A^2
        (OpenMM's default is 0.0054); 0 leaves it out, as AMBER's gbsa=0 does.
    """

    # 1-4 is listed with the bonded terms like in the reference (forces.py:22-25)
    bonded = ["bonds", "angles", "dihedrals", "impropers", "1-4"]
    nonbonded = ["electrostatics", "lj", "repulsion", "repulsioncg"]
    terms = bonded + nonbonded

    def __init__(
        self,
        parameters,
        terms=None,
        external=None,
        cutoff=None,
        rfa=False,
        solventDielectric=78.5,
        switch_dist=None,
        exclusions=("bonds", "angles", "1-4"),
        skin=None,
        pme=False,
        ewald_tolerance=5e-4,
        implicit_solvent=None,
        surface_tension=0.0,
    ):
        self.par = parameters
        if terms is None:
            raise RuntimeError(
                "Set force terms or leave empty brackets [].\nAvailable options: "
                + ", ".join(f'"{t}"' for t in Forces.terms)
                + "."
            )
        if self.par.nonbonded_params is not None and "lj" in terms:
            self.par.A, self.par.B = self.par.get_AB()  # forces.py:45-46

        self.energies = [t.lower() for t in terms]
        for t in self.energies:
            if t not in Forces.terms:
                raise ValueError(f"Force term {t} is not implemented.")
        if "1-4" in self.energies and "dihedrals" not in self.energies:
            raise RuntimeError("You cannot enable 1-4 interactions without enabling dihedrals")
        if rfa and cutoff is None:
            raise RuntimeError("The reaction field approximation needs a cutoff")
        if pme:
            if "electrostatics" not in self.energies:
                raise RuntimeError("Particle-mesh Ewald needs the electrostatics term")
            if cutoff is None:
                raise RuntimeError("Particle-mesh Ewald needs a cutoff")
            if rfa:
                raise RuntimeError("Particle-mesh Ewald and the reaction field approximation exclude each other")
            if not 0.0 < float(ewald_tolerance) < 0.5:
                raise RuntimeError("ewald_tolerance must be between 0 and 0.5")
        if implicit_solvent is not None:
            if str(implicit_solvent).lower() != "obc2":
                raise ValueError(f"implicit_solvent {implicit_solvent!r} is not implemented: 'obc2' or None")
            implicit_solvent = "obc2"
            if "electrostatics" not in self.energies:
                raise RuntimeError("Implicit solvent needs the electrostatics term")
            if cutoff is not None:
                raise RuntimeError("Implicit solvent sums every pair: it takes no cutoff")
            if rfa:
                raise RuntimeError("Implicit solvent and the reaction field approximation exclude each other")
            if pme:
                raise RuntimeError("Implicit solvent and particle-mesh Ewald exclude each other")
            if not (np.isfinite(float(surface_tension)) and float(surface_tension) >= 0.0):
                raise RuntimeError("surface_tension must be finite and not negative (kcal/mol/A^2)")
            if not (np.isfinite(float(solventDielectric)) and float(solventDielectric) > 0.0):
                raise RuntimeError("Implicit solvent needs a finite positive solventDielectric")
            gb = getattr(parameters, "gb_params", None)
            if gb is None:
                raise RuntimeError("Implicit solvent needs parameters.gb_params (amber_parameters(..., terms=[..., 'gb']))")
            n = len(parameters.masses)
            radius = np.asarray(gb["radius"].detach().cpu() if torch.is_tensor(gb["radius"]) else gb["radius"], np.float64).reshape(-1)
            screen = np.asarray(gb["screen"].detach().cpu() if torch.is_tensor(gb["screen"]) else gb["screen"], np.float64).reshape(-1)
            if len(radius) != n or len(screen) != n:
                raise RuntimeError(f"gb_params must hold one radius and one screen per atom ({n})")
            if not (np.isfinite(radius).all() and np.isfinite(screen).all()):
                raise RuntimeError("gb_params holds a value that is not finite")
            if (radius <= 0.09).any() or (screen <= 0).any():
                raise RuntimeError("gb_params: every radius must be above 0.09 A and every screen positive")

        self.natoms = len(parameters.masses)
        self.require_distances = any(t in self.nonbonded for t in self.energies)
        self.external = external
        self.cutoff = cutoff
        self.rfa = rfa
        self.solventDielectric = solventDielectric
        self.switch_dist = switch_dist
        self.skin = DEFAULT_SKIN if skin is None else float(skin)
        self.pme = bool(pme)
        self.ewald_tolerance = float(ewald_tolerance)
        self.implicit_solvent = implicit_solvent
        self.surface_tension = float(surface_tension)
        self._exclusion_types = tuple(exclusions)
        self._ava_idx = None
        self._ctx = None
        self._ctx_key = None
        self._box_key = None
        self._box_ref = None  # the tensor _box_key describes (held so that its storage is not recycled)
        self._scratch_forces = None
        self._exact_gradient = False  # force convention currently set in the context

    # ------------------------------------------------------------------ context
    def __del__(self):
        try:
            if self._ctx is not None:
                _lib.lib().tmd_destroy(self._ctx)
        except Exception:
            pass

    @property
    def ava_idx(self):
        """(P,2) table of all non-excluded pairs, i<j row-major (forces.py:348-357).
        Built lazily -- nothing in this class needs it."""
        if not self.require_distances:
            return None
        if self._ava_idx is None:
            if self.natoms > 20000:
                raise RuntimeError("ava_idx is O(N^2); refusing to materialise it for more than 20000 atoms")
            ok = np.ones((self.natoms, self.natoms), dtype=bool)
            ex = self.par.get_exclusions(self._exclusion_types)
            if len(ex):
                ex = np.asarray(ex)
                ok[ex[:, 0], ex[:, 1]] = False
                ok[ex[:, 1], ex[:, 0]] = False
            self._ava_idx = torch.tensor(np.argwhere(np.triu(ok, 1))).to(self.par.device)
        return self._ava_idx

    def _check_tensor(self, t, name, shape=None, dtype=None):
        if not torch.is_tensor(t) or not _lib.on_device(t):
            raise RuntimeError(f"{name} must be a CUDA tensor: torchmd_b200 has no CPU path")
        if t.dtype not in (torch.float32, torch.float64):
            raise NotImplementedError(f"{name} must be float32 (precision: single) or float64 (precision: double); got {t.dtype}")
        if dtype is not None and t.dtype != dtype:
            raise RuntimeError(f"{name} is {t.dtype} but the positions are {dtype}: one precision per call")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
        if shape is not None and tuple(t.shape) != tuple(shape):
            raise RuntimeError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")

    def _ensure_ctx(self, pos):
        """Create the device context on first use (needs the replica count and device)."""
        nrep = pos.shape[0]
        key = (pos.device.index if pos.device.index is not None else torch.cuda.current_device(), nrep, pos.dtype)
        if self._ctx is not None and self._ctx_key == key:
            return self._ctx
        L = _lib.lib()
        if self._ctx is not None:
            L.tmd_destroy(self._ctx)
            self._ctx = None
        if pos.shape[1] != self.natoms:
            raise RuntimeError(f"positions have {pos.shape[1]} atoms, parameters {self.natoms}")
        import ctypes as C

        handle = C.c_void_p()
        _lib.check(L.tmd_create(C.byref(handle), key[0], self.natoms, nrep))
        ctx = handle
        if pos.dtype == torch.float64:
            try:
                _lib.check(L.tmd_set_precision(ctx, 64))
            except Exception:
                L.tmd_destroy(ctx)
                raise
        self._configure(L, ctx, _lib.check, f64=pos.dtype == torch.float64)
        self._ctx, self._ctx_key, self._box_key, self._box_ref = ctx, key, None, None
        self._exact_gradient = False
        return ctx

    def _configure(self, L, ctx, check, f64=False):
        """Hand topology and parameters to a fresh context (every tmd_set_* call; host data only).
        ``L`` is the bound library, ``check`` raises on a non-zero return code.  ``f64``: an fp64 context
        (tmd_set_precision), whose parameters go over in fp64 through the ``_f64`` setters."""
        par = self.par
        real = np.float64 if f64 else np.float32
        sfx = "_f64" if f64 else ""

        def setter(name):
            return getattr(L, name + sfx)

        charges = _np(par.charges, real)
        if par.mapped_atom_types is not None:
            types = _np(par.mapped_atom_types, np.int32)
        else:
            types = np.zeros(self.natoms, dtype=np.int32)
        need_ab = any(t in self.energies for t in ("lj", "repulsion", "repulsioncg"))
        A = B = None
        ntypes = int(types.max()) + 1
        if need_ab:
            if getattr(par, "A", None) is None:
                par.A, par.B = par.get_AB()
            A, B = _np(par.A, real), _np(par.B, real)
            ntypes = A.shape[0]
        check(setter("tmd_set_atoms")(ctx, _lib.ptr(charges), _lib.ptr(types), ntypes, _lib.ptr(A), _lib.ptr(B)))

        if self.require_distances:
            row_ptr, cols = _exclusion_csr(self.natoms, par.get_exclusions(self._exclusion_types))
            check(L.tmd_set_exclusions(ctx, _lib.ptr(row_ptr), _lib.ptr(cols)))

        check(
            L.tmd_set_nonbonded(
                ctx,
                _lib.term_mask(self.energies),
                -1.0 if self.cutoff is None else float(self.cutoff),
                -1.0 if self.switch_dist is None else float(self.switch_dist),
                int(bool(self.rfa)),
                float(self.solventDielectric),
                float(ELEC_FACTOR),
                self.skin,
            )
        )
        if self.pme:
            check(L.tmd_set_pme(ctx, self.ewald_tolerance))
        if self.implicit_solvent:
            radius = _np(par.gb_params["radius"], np.float64)
            screen = _np(par.gb_params["screen"], np.float64)
            check(L.tmd_set_gb(ctx, self.natoms, _lib.ptr(radius), _lib.ptr(screen), float(self.solventDielectric),
                               self.surface_tension))

        def instance_rows(term):
            """Per-instance parameter rows: params[map[:,1]] ordered by map[:,0]."""
            idx = _np(term["idx"], np.int32)
            m = term["map"].detach().cpu().numpy()
            prm = _np(term["params"], real)[m[:, 1]]
            order = np.argsort(m[:, 0], kind="stable")
            return idx, m[order, 0], np.ascontiguousarray(prm[order])

        if "bonds" in self.energies and par.bond_params is not None:
            idx, _, prm = instance_rows(par.bond_params)
            check(setter("tmd_set_bonds")(ctx, len(idx), _lib.ptr(idx), _lib.ptr(prm)))
        if "angles" in self.energies and par.angle_params is not None:
            idx, _, prm = instance_rows(par.angle_params)
            check(setter("tmd_set_angles")(ctx, len(idx), _lib.ptr(idx), _lib.ptr(prm)))
        for which, name, term in (
            (0, "dihedrals", par.dihedral_params),
            (1, "impropers", par.improper_params),
        ):
            if name in self.energies and term is not None:
                idx, rows, prm = instance_rows(term)  # several terms may share one row of idx
                counts = np.bincount(rows, minlength=len(idx))
                term_ptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
                amber = bool(np.all(prm[:, 2] > 0))  # forces.py:566, decided over the whole set
                check(
                    setter("tmd_set_torsions")(ctx, which, len(idx), _lib.ptr(idx), _lib.ptr(term_ptr), _lib.ptr(prm), int(amber))
                )
        if "1-4" in self.energies and par.nonbonded_14_params is not None and len(par.nonbonded_14_params["idx"]):
            idx, _, prm = instance_rows(par.nonbonded_14_params)
            check(setter("tmd_set_pairs14")(ctx, len(idx), _lib.ptr(idx), _lib.ptr(prm)))
        cmap = getattr(par, "cmap_params", None)  # (a reference Parameters object has none)
        if "dihedrals" in self.energies and cmap is not None and len(cmap["idx"]):
            res, grids = _np(cmap["res"], np.int32), _np(cmap["grids"], np.float64)
            idx, map_of = _np(cmap["idx"], np.int32), _np(cmap["map_of"], np.int32)
            check(L.tmd_set_cmap(ctx, len(res), _lib.ptr(res), _lib.ptr(grids), len(idx), _lib.ptr(idx), _lib.ptr(map_of)))
        ub = getattr(par, "ub_params", None)  # (a reference Parameters object has none)
        if "angles" in self.energies and ub is not None and len(ub["idx"]):
            idx, _, prm = instance_rows(ub)
            ends = np.ascontiguousarray(idx[:, [0, 2]])
            check(setter("tmd_set_urey_bradley")(ctx, len(ends), _lib.ptr(ends), _lib.ptr(prm)))

    def _ensure_box(self, box):
        """Hand the box diagonal to the context when the tensor changed (one D2H copy).  The tensor the
        key was taken from is kept alive: its storage cannot go back to the caching allocator, so a
        fresh box tensor can never reproduce the (address, version) of the one already uploaded."""
        key = (box.data_ptr(), box._version, tuple(box.shape), tuple(box.stride()), box.dtype)
        if key == self._box_key and self._box_ref is not None:
            return
        f64 = self._ctx_key[2] == torch.float64
        diag = np.ascontiguousarray(torch.diagonal(box, dim1=1, dim2=2).detach().cpu().numpy().astype(np.float64 if f64 else np.float32))
        if self.implicit_solvent and np.any(diag != 0):
            raise RuntimeError("Implicit solvent needs a system without a box: every box length must be zero")
        L = _lib.lib()
        _lib.check((L.tmd_set_box_f64 if f64 else L.tmd_set_box)(self._ctx, _lib.ptr(diag)))
        self._box_key, self._box_ref = key, box

    # ------------------------------------------------------------------ compute
    def _evaluate(self, pos, box, forces, sync=True, exact_gradient=False):
        """One pass of the kernels: forces (R,N,3) overwritten, returns the (R, NUM_ENERGIES) fp64
        device energies.  The list-overflow flags are read after every pass (one small D2H read; a
        row or cluster-list overflow grows the capacity and recomputes, so no caller -- the autograd,
        vmap and toNumpy=False paths included -- ever sees a truncated list).  ``sync=False`` skips
        that read; only for a second pass over positions whose lists the first pass just checked.
        ``exact_gradient``: the switched-LJ force as the true derivative of the energy (what the
        reference's autograd path yields) instead of its explicit formula (forces.py:410-412)."""
        self._check_tensor(pos, "pos")
        nrep = pos.shape[0]
        self._check_tensor(forces, "forces", pos.shape, pos.dtype)
        if not torch.is_tensor(box) or tuple(box.shape) != (nrep, 3, 3):
            raise RuntimeError("box must be a (nreplicas, 3, 3) tensor")
        if box.dtype != pos.dtype:
            raise RuntimeError(f"box is {box.dtype} but the positions are {pos.dtype}: one precision per call")
        ctx = self._ensure_ctx(pos)
        self._ensure_box(box)
        L = _lib.lib()
        if bool(exact_gradient) != self._exact_gradient:
            _lib.check(L.tmd_set_force_convention(ctx, int(bool(exact_gradient))))
            self._exact_gradient = bool(exact_gradient)
        stream = torch.cuda.current_stream(pos.device).cuda_stream
        ene = torch.empty((nrep, NUM_ENERGIES), dtype=torch.float64, device=pos.device)
        for _attempt in range(4):
            fn = L.tmd_forces_f64 if pos.dtype == torch.float64 else L.tmd_forces
            _lib.check(fn(ctx, pos.data_ptr(), forces.data_ptr(), ene.data_ptr(), stream))
            if not sync:
                break
            try:
                self.stats()  # synchronises; grows the neighbour rows if one overflowed
                break
            except _lib.TmdError as err:
                if err.code != _lib.ERR_OVERFLOW:
                    raise
        else:
            raise RuntimeError("neighbour rows kept overflowing")
        return ene

    def compute(
        self,
        pos,
        box,
        forces,
        returnDetails=False,
        explicit_forces=True,
        toNumpy=True,
        calculateForces=True,
    ):
        """forces.py:83-346.  ``explicit_forces=False`` (forces as -dE/dpos by autograd in the
        reference) runs the same kernels with the switched-LJ term in its exact-gradient form:
        every other term's explicit force already is the derivative of its energy, the
        reference's explicit switched LJ is not (forces.py:410-412), and autograd returns the
        true one.  The convention is chosen per call: one ``Forces`` may alternate between the two,
        every pair kernel (the cluster lists included) evaluates the one the call asks for, and
        the pair path it takes does not depend on the first call's convention.
        With ``toNumpy=False`` and positions that require grad the returned energies
        carry a grad_fn whose backward is -F of that exact-gradient pass, so
        ``Epot.sum().backward()`` and ``torch.vmap`` over a batch of systems work as with the
        reference (the batch is folded into the replica dimension).  Gradients w.r.t.
        force-field parameters are not provided."""
        if calculateForces:
            if not explicit_forces and not pos.requires_grad:
                raise RuntimeError(
                    "The positions passed don't require gradients. Please use pos.detach().requires_grad_(True) before passing."
                )
            if forces is None:
                raise RuntimeError("forces tensor required when calculateForces=True")
        else:
            explicit_forces = False

        if (not toNumpy) and torch.is_tensor(pos) and ((pos.requires_grad and torch.is_grad_enabled()) or _is_batched(pos)):
            sel, F = _EnergyFunction.apply(pos, box, self)
            if forces is not None:
                if explicit_forces:  # the buffer gets the explicit-formula forces, the graph the true gradient
                    self._evaluate(pos.detach(), box, forces, exact_gradient=False)
                else:
                    forces.copy_(F)
            ext = None
            if self.external:
                ext, ext_force = self.external.calculate(pos, box)
                if forces is not None:
                    if explicit_forces:
                        forces += ext_force
                    elif calculateForces and torch.is_tensor(ext) and ext.requires_grad:
                        forces -= torch.autograd.grad(ext.sum(), pos, retain_graph=True)[0]
            return self._format_tensors(sel, ext, returnDetails)

        pos_in = pos.detach() if torch.is_tensor(pos) and pos.requires_grad else pos
        if forces is None:
            sf = self._scratch_forces
            if sf is None or sf.shape != pos_in.shape or sf.dtype != pos_in.dtype or sf.device != pos_in.device:
                self._scratch_forces = torch.empty_like(pos_in)
            forces = self._scratch_forces
        ene = self._evaluate(pos_in, box, forces, exact_gradient=calculateForces and not explicit_forces)

        ext = None
        if self.external:
            ext, ext_force = self.external.calculate(pos, box)
            if explicit_forces:
                forces += ext_force
            elif calculateForces and torch.is_tensor(ext) and ext.requires_grad:  # forces.py:328-336
                forces -= torch.autograd.grad(ext.sum(), pos, retain_graph=True)[0]
            if torch.is_tensor(ext):
                ext = ext.detach()
        if toNumpy:
            return self._format(ene, ext, pos_in.dtype, returnDetails, True)
        return self._format_tensors(ene[:, self._energy_columns()].to(pos_in.dtype), ext, returnDetails)

    def _energy_columns(self):
        return [ENERGY_SLOTS.index(t) for t in self.energies]

    def _format(self, ene, ext, dtype, returnDetails, toNumpy):
        """Marshal (R, NUM_ENERGIES) fp64 device sums into the reference's return formats
        (forces.py:338-346)."""
        nrep = ene.shape[0]
        cols = self._energy_columns()
        if toNumpy:
            host = ene.cpu().numpy()
            exth = [float(ext[r]) for r in range(nrep)] if ext is not None else [0.0] * nrep
            if returnDetails:
                out = []
                for r in range(nrep):
                    d = {t: float(host[r, c]) for t, c in zip(self.energies, cols)}
                    d["external"] = exth[r]
                    out.append(d)
                return out
            return [float(host[r, cols].sum()) + exth[r] for r in range(nrep)]
        return self._format_tensors(ene[:, cols].to(dtype), ext, returnDetails)

    def _format_tensors(self, sel, ext, returnDetails):
        """``toNumpy=False`` formats from the (R, nterms) per-term energies (forces.py:338-346)."""
        nrep = sel.shape[0]
        extt = ext.to(sel.dtype).reshape(nrep) if ext is not None else torch.zeros(nrep, dtype=sel.dtype, device=sel.device)
        if returnDetails:
            out = []
            for r in range(nrep):
                d = {t: sel[r, k].reshape(1) for k, t in enumerate(self.energies)}
                d["external"] = extt[r].reshape(1)
                out.append(d)
            return out
        return sel.sum(dim=1) + extt

    # ------------------------------------------------------------------ inspection
    def stats(self):
        """Counters of the device context (synchronises)."""
        if self._ctx is None:
            return None
        st = _lib.Stats()
        import ctypes as C

        stream = torch.cuda.current_stream(torch.device("cuda", self._ctx_key[0])).cuda_stream  # of the context's device, not the current one
        _lib.check(_lib.lib().tmd_get_stats(self._ctx, C.byref(st), stream))
        return {
            "rebuilds": st.rebuilds,
            "force_calls": st.force_calls,
            "max_neighbours": st.max_neighbours,
            "row_capacity": st.row_capacity,
            "overflow": st.overflow,
            "ncells": tuple(st.ncells),
            "kernel_launches": st.kernel_launches,
        }

    def pme_parameters(self):
        """(alpha in 1/A, (n_x, n_y, n_z)) that the library chose for the boxes set last (``pme=True``, after a
        compute)."""
        if not self.pme or self._ctx is None:
            return None
        import ctypes as C

        alpha, grid = C.c_double(), (C.c_int32 * 3)()
        _lib.check(_lib.lib().tmd_get_pme(self._ctx, C.byref(alpha), C.byref(grid)))
        return alpha.value, tuple(grid)

    def neighbour_pairs(self, pos, box, replica=0):
        """The reference's neighbour list ``ava_idx[dist <= cutoff]`` (forces.py:264-269) for
        one replica as a lexicographically sorted (P,2) int32 CUDA tensor."""
        if not self.require_distances:
            raise RuntimeError("no non-bonded term enabled")
        scratch = torch.empty_like(pos)
        self.compute(pos, box, scratch)  # make the list current for these positions
        L = _lib.lib()
        stream = torch.cuda.current_stream(pos.device).cuda_stream
        count = torch.zeros(1, dtype=torch.int64, device=pos.device)
        cap = max(1024, int(self.stats()["max_neighbours"]) * self.natoms // 2 + 1024)
        out = torch.empty((cap, 2), dtype=torch.int32, device=pos.device)
        fn = L.tmd_export_pairs_f64 if pos.dtype == torch.float64 else L.tmd_export_pairs
        _lib.check(fn(self._ctx, pos.data_ptr(), int(replica), out.data_ptr(), cap, count.data_ptr(), stream))
        n = int(count.item())
        if n > cap:
            raise RuntimeError("pair export buffer too small")
        p = out[:n].to(torch.int64)
        order = torch.argsort(p[:, 0] * self.natoms + p[:, 1])
        return out[:n][order]



def _is_batched(t):
    """Inside torch.vmap the positions are a BatchedTensor (which does not report requires_grad)."""
    fn = getattr(getattr(torch._C, "_functorch", None), "is_batchedtensor", None)
    return bool(fn(t)) if fn is not None else False


class _EnergyFunction(torch.autograd.Function):
    """Per-term energies (R, nterms) of ``Forces`` as a differentiable function of the
    positions: the backward pass is -F from the same kernel pass that produced the energies
    (forces.py:328-336 obtains F the other way round, as -dE/dpos by autograd).  The kernels
    give the gradient of the SUM of the terms, so the incoming gradient must be the same for
    every term of a replica (``Epot.sum()``, the reference's own use); anything else raises."""

    @staticmethod
    def forward(pos, box, owner):
        F = torch.empty_like(pos, memory_format=torch.contiguous_format)
        p = pos.detach().contiguous()
        ene = owner._evaluate(p, box.detach().contiguous(), F, exact_gradient=True)
        return ene[:, owner._energy_columns()].to(pos.dtype), F

    @staticmethod
    def setup_context(ctx, inputs, output):
        ctx.mark_non_differentiable(output[1])
        ctx.save_for_backward(output[1])

    @staticmethod
    def backward(ctx, grad_e, grad_f):
        (F,) = ctx.saved_tensors
        g = grad_e[:, 0]
        if grad_e.shape[1] > 1 and not bool((grad_e == g[:, None]).all()):
            raise NotImplementedError(
                "gradients that differ between energy terms need one force pass per term; "
                "differentiate the summed energy (returnDetails=False or sum the terms with equal weights)"
            )
        return -F * g.to(F.dtype)[:, None, None], None, None

    @staticmethod
    def vmap(info, in_dims, pos, box, owner):
        """``torch.vmap`` over a batch of systems: the batch is folded into the replica dimension
        (the kernels run one grid slice per replica)."""
        pd, bd, _ = in_dims
        nb = info.batch_size
        pb = pos.movedim(pd, 0) if pd is not None else pos.unsqueeze(0).expand(nb, *pos.shape)
        bb = box.movedim(bd, 0) if bd is not None else box.unsqueeze(0).expand(nb, *box.shape)
        nrep, natoms = pb.shape[1], pb.shape[2]
        e, F = _EnergyFunction.apply(pb.reshape(nb * nrep, natoms, 3), bb.reshape(nb * nrep, 3, 3), owner)
        return (e.reshape(nb, nrep, -1), F.reshape(nb, nrep, natoms, 3)), (0, 0)
