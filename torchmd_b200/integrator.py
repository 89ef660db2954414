"""``Integrator`` with the interface of ``torchmd.integrator.Integrator``
(reference ``torchmd/integrator.py:80-125``): velocity Verlet with the
reference's Langevin kick placement, running on the sm_90a kernels.

``step(niter)`` returns ``(Ekin ndarray, pot, T ndarray)`` like the reference.
When ``forces`` is a ``torchmd_b200.Forces`` without an external plugin the
whole ``niter`` loop is enqueued through one C-ABI call with no host round trip
(the reference synchronises several times per step, SURVEY.md section 3.3);
any other object exposing ``compute(pos, box, forces)`` is driven step by step
exactly like the reference does (``tests/test_integrator.py`` mock forces).

``constraints`` (a ``torchmd_b200.constraints.Constraints``) makes the step RATTLE: rigid waters and,
with ``kind="hbonds"``, fixed bonds to hydrogen, which allow 2 fs time steps.  The returned ``T`` then
counts the constrained degrees of freedom out (``Constraints.ndof``); ``Ekin`` stays sum(m v^2 / 2).

``barostat`` (a ``torchmd_b200.barostat.MonteCarloBarostat``) runs at constant pressure: the steps go in chunks that end
where the step index reaches a multiple of its ``frequency``, and each such chunk is followed by one Monte Carlo volume
move per replica, which writes the accepted box into ``systems.box``.  The returned energies describe the state after
the move.

``T`` is one temperature or a sequence of one per replica.  With a sequence, ``vcoeff`` is an (R, N, 1) table, one row
per temperature (row k is the ``vcoeff`` of a run at ``T[k]``), and replica r takes its noise from row ``ladder[r]`` of
an (R,) int32 device ladder, the identity unless ``replica_exchange`` (a ``torchmd_b200.ReplicaExchange``) swaps
temperatures between replicas.  Exchange attempts follow every ``frequency``-th step, like the barostat's moves; when
one ends a call, the returned ``Ekin`` and ``T`` describe the scaled velocities.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .forces import Forces

TIMEFACTOR = 48.88821  # integrator.py:4
BOLTZMAN = 0.001987191  # integrator.py:5
PICOSEC2TIMEU = 1000.0 / TIMEFACTOR  # integrator.py:77


def kinetic_energy(masses, vel, batch=None):
    """0.5 m v^2 per replica (R,1), or per replica and batch group (R,nbatch)
    (integrator.py:8-43).  Host-side helper on plain tensors."""
    if vel.dim() != 3:
        raise ValueError(f"vel must be 3D (nreplicas, natoms, 3), got {vel.dim()}D")
    per_atom = 0.5 * masses * (vel * vel).sum(dim=2, keepdim=True)
    if batch is None:
        return per_atom.sum(dim=1)
    nb = int(batch.max().item() + 1)
    out = torch.zeros(vel.shape[0], nb, device=vel.device, dtype=vel.dtype)
    out.index_add_(1, batch, per_atom[:, :, 0])
    return out


def _is_sequence(T):
    return isinstance(T, (list, tuple, np.ndarray, torch.Tensor)) and np.ndim(T) > 0


def maxwell_boltzmann(masses, T, replicas=1):
    """Velocities ~ sqrt(kB T / m) N(0,1) per replica (integrator.py:46-54).  ``T``: one temperature, or a sequence of
    ``replicas`` temperatures, replica r drawn at ``T[r]``."""
    if _is_sequence(T):
        temps = [float(t) for t in T]
        if len(temps) != replicas:
            raise ValueError(f"maxwell_boltzmann: {len(temps)} temperatures for {replicas} replicas")
        draws = [torch.sqrt(t * BOLTZMAN / masses) * torch.randn((len(masses), 3)).type_as(masses) for t in temps]
        return torch.stack(draws, dim=0)
    scale = torch.sqrt(T * BOLTZMAN / masses)
    draws = [scale * torch.randn((len(masses), 3)).type_as(masses) for _ in range(replicas)]
    return torch.stack(draws, dim=0)


def kinetic_to_temp(Ekin, natoms):
    """T = 2 Ekin / (3 N kB) with N atoms, not degrees of freedom (integrator.py:57-58)."""
    return 2.0 / (3.0 * natoms * BOLTZMAN) * Ekin


class Integrator:
    def __init__(self, systems, forces, timestep, device, gamma=None, T=None, batch=None, constraints=None, barostat=None,
                 replica_exchange=None):
        nrep = systems.pos.shape[0]
        self.temperatures = None  # the ladder's temperatures (a sequence T), or None
        if _is_sequence(T):
            self.temperatures = [float(t) for t in T]
            if len(self.temperatures) != nrep:
                raise ValueError(f"T has {len(self.temperatures)} temperatures for {nrep} replicas")
            if not all(t > 0.0 and np.isfinite(t) for t in self.temperatures):
                raise ValueError("the temperatures must be positive and finite")
            T = self.temperatures
        if replica_exchange is not None:
            if gamma is None or T is None:
                raise RuntimeError("replica exchange needs a thermostat: give the Integrator gamma and a list of temperatures")
            if self.temperatures is None:
                raise ValueError("replica exchange needs one temperature per replica: give T as a sequence")
            if barostat is not None:
                raise RuntimeError("replica exchange cannot run with a barostat: the barostat's kT is one temperature")
        if barostat is not None and self.temperatures is not None:
            raise RuntimeError("MonteCarloBarostat runs at one temperature: give T as a scalar")
        self.dt = timestep / TIMEFACTOR
        self.systems = systems
        self.forces = forces
        self.device = device
        if gamma is not None:
            gamma = gamma / PICOSEC2TIMEU
        self.gamma = gamma
        self.T = T
        # mass source: the system's if any is set, else the force field's (integrator.py:92-99)
        if torch.any(systems.masses != 0):
            self.masses = systems.masses
        else:
            self.masses = (
                forces.par.masses.clone().detach().to(device=device, dtype=systems.pos.dtype).view(-1, 1)
            )
        self._ladder = None  # (R,) int32 device ladder of a sequence T: replica r reads vcoeff row _ladder[r]
        if self.temperatures is not None:
            # one row per temperature, each the expression of the scalar case
            self.vcoeff = torch.stack([torch.sqrt(2.0 * gamma / self.masses * BOLTZMAN * t * self.dt) for t in self.temperatures]).to(device)
            self._ladder = torch.arange(nrep, dtype=torch.int32, device=systems.pos.device)
        elif T:
            self.vcoeff = torch.sqrt(2.0 * gamma / self.masses * BOLTZMAN * T * self.dt).to(device)
        self.batch = batch
        if batch is not None:
            self.natoms = torch.bincount(batch).cpu().numpy()
        else:
            self.natoms = len(self.masses)
        # Philox key for the in-kernel Langevin noise: drawn from torch's generator so
        # torch.manual_seed (torchmd/run.py:231) makes runs reproducible
        self.seed = int(torch.randint(0, 2**62, (1,)).item())
        self._step_index = 0
        self._own_ctx = None
        self._own_dtype = None  # precision the private context was set up for
        self._out = None  # (ke, energies) device buffers, kept between calls: the captured steps hold their addresses
        self.constraints = constraints
        self._projected = False  # the start state has been projected onto the constraints
        if constraints is not None:
            if constraints.natoms != len(self.masses):
                raise ValueError(f"constraints are for {constraints.natoms} atoms, the system has {len(self.masses)}")
            self.ndof = constraints.ndof(batch=batch.cpu().numpy() if batch is not None else None)
        self.barostat = barostat
        if barostat is not None:
            box = systems.box
            diag = torch.diagonal(box, dim1=1, dim2=2)
            off = box - torch.diag_embed(diag)
            if not bool((diag > 0).all()) or bool((off != 0).any()):
                raise RuntimeError("MonteCarloBarostat needs a periodic orthorhombic box on every replica")
            barostat._bind(self)
        self.replica_exchange = replica_exchange
        if replica_exchange is not None:
            replica_exchange._bind(self)

    def __del__(self):
        try:
            if self._own_ctx is not None:
                _lib.lib().tmd_destroy(self._own_ctx)
        except Exception:
            pass

    def _require_cuda(self):
        """The state's dtype is the run's precision (float32 or float64); masses and vcoeff follow it."""
        s = self.systems
        dtype = s.pos.dtype
        for name in ("pos", "vel", "forces"):
            t = getattr(s, name)
            if not _lib.on_device(t):
                raise RuntimeError(f"systems.{name} must live on a CUDA device: torchmd_b200 has no CPU path")
            if t.dtype not in (torch.float32, torch.float64) or not t.is_contiguous():
                raise NotImplementedError(f"systems.{name} must be contiguous float32 or float64")
            if t.dtype != dtype:
                raise RuntimeError(f"systems.{name} is {t.dtype} but systems.pos is {dtype}: one precision per run")
        m = self.masses
        if not _lib.on_device(m) or m.dtype != dtype or not m.is_contiguous():
            self.masses = m.to(device=s.pos.device, dtype=dtype).contiguous()
        if self.T and (not _lib.on_device(self.vcoeff) or self.vcoeff.dtype != dtype or not self.vcoeff.is_contiguous()):
            self.vcoeff = self.vcoeff.to(device=s.pos.device, dtype=dtype).contiguous()

    def _ctx(self):
        """Context for the integrator kernels: the Forces object's, or a private one."""
        s = self.systems
        if isinstance(self.forces, Forces):
            return self.forces._ensure_ctx(s.pos)
        if self._own_ctx is None:
            handle = C.c_void_p()
            dev = s.pos.device.index if s.pos.device.index is not None else torch.cuda.current_device()
            _lib.check(_lib.lib().tmd_create(C.byref(handle), dev, s.pos.shape[1], s.pos.shape[0]))
            self._own_ctx = handle
            self._own_dtype = None
        if self._own_dtype != s.pos.dtype:
            if self._own_dtype is not None:  # the precision is fixed at set-up: a new context
                _lib.lib().tmd_destroy(self._own_ctx)
                self._own_ctx = None
                return self._ctx()
            if s.pos.dtype == torch.float64:
                _lib.check(_lib.lib().tmd_set_precision(self._own_ctx, 64))
            self._own_dtype = s.pos.dtype
        return self._own_ctx

    def _constrained_ctx(self):
        """``_ctx()`` holding this integrator's constraint tables, or none.  The tables live in the context, which a
        ``Forces`` object shares between the integrators built on it: the handle records which ``Constraints`` it
        holds, and the tables are handed over (or cleared) whenever that is not this integrator's."""
        ctx = self._ctx()
        if getattr(ctx, "_tmd_constraints", None) is not self.constraints:
            if self.constraints is not None:
                self.constraints.upload(ctx)
            else:
                _lib.check(_lib.lib().tmd_set_constraints(ctx, 0, None, None, 0, None, None, None))
            ctx._tmd_constraints = self.constraints
        # the temperature ladder, shared the same way: an integrator with one temperature must not run on another's
        if getattr(ctx, "_tmd_ladder", None) is not self._ladder:
            if self._ladder is not None:
                temps = np.ascontiguousarray(self.temperatures, dtype=np.float64)
                _lib.check(_lib.lib().tmd_set_temperature_ladder(ctx, len(temps), temps.ctypes.data, self._ladder.data_ptr()))
            else:
                _lib.check(_lib.lib().tmd_set_temperature_ladder(ctx, 0, None, None))
            ctx._tmd_ladder = self._ladder
        return ctx

    def step(self, niter=1, noise=None):
        """Advance ``niter`` steps.  ``noise`` (niter, R, N, 3) injects the N(0,1) Langevin
        draws (parity tests); by default they come from Philox4x32-10 inside the kernel."""
        s = self.systems
        self._require_cuda()
        L = _lib.lib()
        ctx = self._constrained_ctx()
        stream = torch.cuda.current_stream(s.pos.device).cuda_stream
        nrep = s.pos.shape[0]
        f64 = s.pos.dtype == torch.float64
        sfx = "_f64" if f64 else ""
        thermostat = bool(self.T)
        gamma = float(self.gamma) if thermostat else -1.0
        vcoeff = self.vcoeff.data_ptr() if thermostat else None
        if noise is not None:
            if tuple(noise.shape) != (niter,) + tuple(s.vel.shape):
                raise RuntimeError("noise must have shape (niter, nreplicas, natoms, 3)")
            noise = noise.to(device=s.pos.device, dtype=s.pos.dtype).contiguous()
        if self._out is None or self._out[0].shape[0] != nrep or self._out[0].device != s.pos.device:
            self._out = (torch.empty(nrep, dtype=torch.float64, device=s.pos.device),
                         torch.empty((nrep, _lib.NUM_ENERGIES), dtype=torch.float64, device=s.pos.device))
        ke = self._out[0]
        if self.constraints is not None and not self._projected:
            # a start state (maxwell_boltzmann velocities above all) has components along the constrained bonds
            _lib.check(getattr(L, "tmd_constrain" + sfx)(ctx, s.pos.data_ptr(), s.vel.data_ptr(), self.masses.data_ptr(), stream))
            self._projected = True
        native = isinstance(self.forces, Forces) and not self.forces.external
        rex = self.replica_exchange
        exchanged = False  # the call ended with an exchange: the kinetic energy is that of the scaled velocities
        pot = None
        if native and niter > 0:
            f = self.forces
            f._ensure_box(s.box)
            if f._exact_gradient:  # left behind by an autograd-path compute(): MD uses the reference's explicit forces
                _lib.check(L.tmd_set_force_convention(ctx, 0))
                f._exact_gradient = False
            ene = self._out[1]
            bar = self.barostat
            period = bar.frequency if bar is not None else (rex.frequency if rex is not None else None)
            done = 0
            while done < niter:
                # with a barostat or replica exchange the steps run in chunks that end where a move is due
                n = niter - done if period is None else min(niter - done, period - self._step_index % period)
                chunk_noise = noise[done:done + n] if noise is not None and period is not None else noise
                # A neighbour list that outgrows its reserved capacity inside the fused call invalidates the call (the
                # kernels truncate, the library grows the capacity at the stats() check).  The state is three small
                # tensors: keep a copy and run the call again from it instead of giving up.  Everything else a step reads
                # is either rebuilt by the re-finalised context (lists, their reference positions, the captured steps) or
                # rewritten by the step before it is read (constraint reference positions, energy outputs).
                saved = (s.pos.clone(), s.vel.clone(), s.forces.clone())
                for attempt in range(6):
                    _lib.check(
                        getattr(L, "tmd_md_steps" + sfx)(
                            ctx, n, s.pos.data_ptr(), s.vel.data_ptr(), s.forces.data_ptr(), self.masses.data_ptr(),
                            self.dt, gamma, vcoeff, _lib.ptr(chunk_noise), self.seed, 0,
                            ene.data_ptr(), ke.data_ptr(), stream,
                        )
                    )
                    try:
                        f.stats()
                        break
                    except _lib.TmdError as err:
                        if err.code != _lib.ERR_OVERFLOW:
                            raise
                        if attempt == 5:
                            raise RuntimeError("the neighbour lists kept overflowing during Integrator.step") from err
                        s.pos.copy_(saved[0])
                        s.vel.copy_(saved[1])
                        s.forces.copy_(saved[2])
                        # the discarded steps advanced the device's Philox position: step s draws the noise of step s again
                        _lib.check(L.tmd_rewind_noise(ctx, n, stream))
                        ctx = self._constrained_ctx()  # (re-finalised with the grown capacity on the next call)
                self._step_index += n
                done += n
                pot = None
                exchanged = False
                if bar is not None and self._step_index % bar.frequency == 0:
                    pot = [float(e) for e in bar.attempt(ctx, ene)]
                if rex is not None and self._step_index % rex.frequency == 0:  # (after the chunk's overflow check)
                    rex.attempt(ctx, ene, _lib.NUM_ENERGIES, _lib.NUM_ENERGIES)
                    exchanged = True
            if pot is None:
                pot = f._format(ene, None, s.pos.dtype, False, True)
        else:
            for it in range(niter):
                _lib.check(
                    getattr(L, "tmd_vv_first" + sfx)(ctx, s.pos.data_ptr(), s.vel.data_ptr(), s.forces.data_ptr(), self.masses.data_ptr(), self.dt, stream)
                )
                pot = self.forces.compute(s.pos, s.box, s.forces)
                last = it == niter - 1
                _lib.check(
                    getattr(L, "tmd_vv_second" + sfx)(
                        ctx, s.vel.data_ptr(), s.forces.data_ptr(), self.masses.data_ptr(), self.dt, gamma, vcoeff,
                        noise[it].data_ptr() if noise is not None else None, self.seed, 0,
                        ke.data_ptr() if last else None, stream,
                    )
                )
                self._step_index += 1
                exchanged = rex is not None and self._step_index % rex.frequency == 0
                if exchanged:  # from this step's potential energies, the external term included
                    pot_dev = torch.as_tensor(np.asarray(pot, dtype=np.float64).reshape(nrep, 1)).to(s.pos.device)
                    rex.attempt(ctx, pot_dev, 1, 1)
            if niter <= 0:
                _lib.check(getattr(L, "tmd_kinetic_energy" + sfx)(ctx, s.vel.data_ptr(), self.masses.data_ptr(), ke.data_ptr(), stream))
            elif self.constraints is not None:  # (the fused path learns of a failed constraint group from f.stats())
                _lib.check(L.tmd_get_stats(ctx, C.byref(_lib.Stats()), stream))
        if exchanged:
            _lib.check(getattr(L, "tmd_kinetic_energy" + sfx)(ctx, s.vel.data_ptr(), self.masses.data_ptr(), ke.data_ptr(), stream))

        if self.batch is None:
            Ekin = ke.cpu().numpy().astype(np.float64 if f64 else np.float32)  # the state's dtype, like integrator.py:122-125
        else:
            # summed in fp64 like the kernels' ke, then given the state's dtype
            Ekin = kinetic_energy(self.masses.double(), s.vel.double(), self.batch).flatten().cpu().numpy()
            Ekin = Ekin.astype(np.float64 if f64 else np.float32)
        if self.constraints is None:
            T = kinetic_to_temp(Ekin, self.natoms)
        else:
            T = 2.0 / (self.ndof * BOLTZMAN) * Ekin
        return Ekin, pot, T
