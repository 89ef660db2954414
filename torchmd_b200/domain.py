"""Decomposed (multi-GPU) MD step: one process per GPU, NCCL over NVLink.

The reference is single-device; this is the multi-GPU mode for ONE large
system (BASELINE.json config 4).  Decomposition:

* every rank holds all positions (16 B/atom: 1.6 MB at 100k atoms -- the halo of a
  50 A brick with a 10 A list radius would already be 1.5x its own volume, SURVEY.md
  section 8e) and the same cell list / sorted order;
* rank r OWNS a contiguous range of atoms -- a slab of the box for the generator's
  lattice ordering -- and computes the complete force on exactly those atoms (their
  neighbour rows, their bonded terms), integrates exactly those atoms, and
* ONE collective per step: an all-gather of the new positions between the first
  half-kick and the force evaluation.  No force reduction (full neighbour rows), no
  velocity exchange (ownership is static).  Energies / kinetic energy are summed
  across ranks only when ``step()`` returns.

Because each atom's neighbour row is built from the same sorted order by whichever
rank owns it, forces -- and with the counter-based Langevin noise keyed on the global
atom index, whole trajectories -- are bitwise identical to the single-GPU run.

One MD step (kernels + the all-gather) is captured once as a CUDA graph and replayed:
every per-step quantity that changes (rebuild flag parity, Philox step) lives on the
device, so the graph is replayable and the host issues one launch per step.

``exchange="p2p"`` (or TMD_B200_EXCHANGE=p2p) replaces the all-gather by the fused
integrate + exchange kernel of the library (include/tmd_b200.h, tmd_dd_*): the first
half-kick of every rank stores its new positions directly into all ranks' position
buffers through NVLink peer memory and raises a flag; a one-warp kernel waits for the
flags.  Positions then live in two library-owned buffers per rank (read / write buffer
alternate every step) and ``system.pos`` is synchronised at the ends of ``step()``.
Opt-in until validated on a multi-GPU H100 machine.
"""
import ctypes as C
import os

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .integrator import Integrator, kinetic_to_temp


class SlabDecomposition:
    """Static ownership of atom ranges and the padded gather layout (pure host logic)."""

    def __init__(self, natoms, world, rank):
        self.natoms, self.world, self.rank = natoms, world, rank
        self.chunk = -(-natoms // world)  # atoms per rank, last rank may own fewer
        self.padded = self.chunk * world
        self.lo = min(natoms, rank * self.chunk)
        self.hi = min(natoms, self.lo + self.chunk)

    @property
    def count(self):
        return self.hi - self.lo

    def ranges(self):
        return [(min(self.natoms, r * self.chunk), min(self.natoms, (r + 1) * self.chunk)) for r in range(self.world)]

    def rehome(self, pos):
        """Move a (1,N,3) position tensor into a buffer padded to world*chunk atoms and
        return (buffer, view): the view has the original shape and aliases the buffer, so an
        all-gather into the buffer updates the positions in place."""
        buf = torch.zeros(self.padded * 3, dtype=pos.dtype, device=pos.device)
        buf[: self.natoms * 3] = pos.reshape(-1)
        return buf, buf[: self.natoms * 3].view(1, self.natoms, 3)

    def gather(self, buf, send, group=None):
        """All-gather every rank's owned slice of ``buf`` (flattened xyz) into ``buf``."""
        c3 = self.chunk * 3
        send.copy_(buf[self.rank * c3 : (self.rank + 1) * c3])
        if dist.get_backend(group) == "nccl":
            dist.all_gather_into_tensor(buf, send, group=group)
        else:  # gloo (CPU tests)
            parts = [torch.empty_like(send) for _ in range(self.world)]
            dist.all_gather(parts, send, group=group)
            for r, p in enumerate(parts):
                buf[r * c3 : (r + 1) * c3] = p


class DecomposedIntegrator:
    """``Integrator.step`` semantics for one system spread over the ranks of ``group``.

    ``system`` must hold identical data on every rank (same generator, same seed); after
    construction ``system.pos`` aliases a padded gather buffer.  Single replica only.
    """

    def __init__(self, system, forces, timestep, device, gamma=None, T=None, group=None, use_graph=True, exchange=None, constraints=None,
                 barostat=None):
        if barostat is not None:
            raise NotImplementedError("the Monte Carlo barostat runs on one GPU: use Integrator(..., barostat=...)")
        if constraints is not None:
            raise NotImplementedError("constraints run on one GPU: use Integrator(..., constraints=...)")
        if T is not None and np.ndim(T) > 0:
            raise NotImplementedError("per-replica temperatures run on one GPU: use Integrator(..., T=[...])")
        if getattr(forces, "pme", False):
            raise NotImplementedError("particle-mesh Ewald runs on one GPU: use Integrator with Forces(..., pme=True)")
        if getattr(forces, "implicit_solvent", None):
            raise NotImplementedError("implicit solvent runs on one GPU: use Integrator with Forces(..., implicit_solvent=...)")
        if system.pos.dtype == torch.float64:
            raise NotImplementedError("decomposed runs are fp32 only: run 'precision: double' on one GPU")
        if system.pos.shape[0] != 1:
            raise NotImplementedError("decomposed runs take one replica; shard replicas across ranks instead")
        self.exchange = (exchange or os.environ.get("TMD_B200_EXCHANGE", "allgather")).lower()
        if self.exchange not in ("allgather", "p2p"):
            raise ValueError(f"unknown exchange {self.exchange!r}: 'allgather' or 'p2p'")
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        self.system, self.forces = system, forces
        n = system.pos.shape[1]
        self.dec = SlabDecomposition(n, self.world, self.rank)
        self.buf, system.pos = self.dec.rehome(system.pos)
        self.send = torch.empty(self.dec.chunk * 3, dtype=system.pos.dtype, device=system.pos.device)
        self.integ = Integrator(system, forces, timestep, device, gamma=gamma, T=T)
        seed = torch.tensor([self.integ.seed], dtype=torch.int64, device=system.pos.device)
        dist.broadcast(seed, 0, group=group)  # one noise stream, independent of the rank count
        self.integ.seed = int(seed.item())
        self.integ._require_cuda()
        self.ctx = forces._ensure_ctx(system.pos)
        forces._ensure_box(system.box)
        _lib.check(_lib.lib().tmd_set_owned_atoms(self.ctx, self.dec.lo, self.dec.count))
        nrep = 1
        self.ene = torch.zeros((nrep, _lib.NUM_ENERGIES), dtype=torch.float64, device=system.pos.device)
        self.ke = torch.zeros(nrep, dtype=torch.float64, device=system.pos.device)
        self.use_graph = use_graph
        self._graphs = {}
        self._parity = 0  # p2p: which of the two position buffers holds the current positions
        self._marks = None  # bench.py: list that collects the phase events of eagerly issued steps
        if self.exchange == "p2p" and not self._connect_peers():
            self.exchange = "allgather"

    def _all_ok(self, err, what):
        """Every rank must take the same path: True iff the local step ``what`` worked on all ranks."""
        ok = torch.tensor([0 if err else 1], dtype=torch.int32, device=self.system.pos.device)
        if self.world > 1:
            dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
        if int(ok.item()) == 1:
            return True
        if self.rank == 0 or err is not None:
            import sys

            print(f"[domain] rank {self.rank}: peer-to-peer exchange unavailable ({what}: {err if err else 'failed on another rank'}); "
                  "using the NCCL all-gather exchange", file=sys.stderr)
        return False

    def _connect_peers(self):
        """Allocate this rank's exchange buffers and map every peer's (CUDA IPC handles travel
        through one all-gather at set-up; nothing else does).  Returns False -- on every rank --
        if any rank could not (CUDA IPC not permitted, no peer access between two GPUs ...)."""
        L = _lib.lib()
        if self.world > _lib.MAX_PEERS:
            raise NotImplementedError(f"peer-to-peer exchange supports up to {_lib.MAX_PEERS} ranks")
        dev = self.system.pos.device
        handle = (C.c_ubyte * _lib.IPC_HANDLE_BYTES)()
        err = None
        try:
            _lib.check(L.tmd_dd_create(self.ctx, self.rank, self.world, handle))
        except _lib.TmdError as e:
            err = e
        if not self._all_ok(err, "allocating the exchange buffers"):
            return False
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=dev)
        everyone = torch.empty(self.world * _lib.IPC_HANDLE_BYTES, dtype=torch.uint8, device=dev)
        if self.world > 1:
            dist.all_gather_into_tensor(everyone, mine, group=self.group)
        else:
            everyone.copy_(mine)
        raw = bytes(everyone.cpu().numpy().tobytes())
        table = (C.c_ubyte * len(raw)).from_buffer_copy(raw)
        try:
            _lib.check(L.tmd_dd_connect(self.ctx, table))
        except _lib.TmdError as e:
            err = e
        # (also the barrier: every rank has mapped every buffer before anyone stores into one)
        return self._all_ok(err, "mapping the peers' buffers")

    # one MD step on the current stream; with_energy: also this rank's energy / KE share
    def _mark(self, marks):
        """Phase boundary of an eagerly issued step (bench.py's per-phase breakdown): a CUDA event on the stream."""
        if marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append(ev)

    def _enqueue_step_p2p(self, with_energy, parity, marks=None):
        s, ig, L = self.system, self.integ, _lib.lib()
        stream = torch.cuda.current_stream(s.pos.device).cuda_stream
        thermostat = bool(ig.T)
        gamma = float(ig.gamma) if thermostat else -1.0
        vcoeff = ig.vcoeff.data_ptr() if thermostat else None
        self._mark(marks)
        _lib.check(L.tmd_dd_vv_first_push(self.ctx, parity, s.vel.data_ptr(), s.forces.data_ptr(), ig.masses.data_ptr(), ig.dt, stream))
        self._mark(marks)
        _lib.check(L.tmd_dd_wait(self.ctx, stream))
        self._mark(marks)
        _lib.check(L.tmd_dd_forces(self.ctx, 1 - parity, s.forces.data_ptr(), self.ene.data_ptr() if with_energy else None, stream))
        self._mark(marks)
        _lib.check(
            L.tmd_vv_second(self.ctx, s.vel.data_ptr(), s.forces.data_ptr(), ig.masses.data_ptr(), ig.dt, gamma, vcoeff,
                            None, ig.seed, 0, self.ke.data_ptr() if with_energy else None, stream)
        )
        self._mark(marks)

    def _enqueue_step(self, with_energy, parity=0, marks=None):
        if self.exchange == "p2p":
            return self._enqueue_step_p2p(with_energy, parity, marks)
        s, ig, L = self.system, self.integ, _lib.lib()
        stream = torch.cuda.current_stream(s.pos.device).cuda_stream
        thermostat = bool(ig.T)
        gamma = float(ig.gamma) if thermostat else -1.0
        vcoeff = ig.vcoeff.data_ptr() if thermostat else None
        self._mark(marks)
        _lib.check(L.tmd_vv_first(self.ctx, s.pos.data_ptr(), s.vel.data_ptr(), s.forces.data_ptr(), ig.masses.data_ptr(), ig.dt, stream))
        self._mark(marks)
        self.dec.gather(self.buf, self.send, self.group)  # the exchange step: new positions to everyone
        self._mark(marks)
        _lib.check(L.tmd_forces(self.ctx, s.pos.data_ptr(), s.forces.data_ptr(), self.ene.data_ptr() if with_energy else None, stream))
        self._mark(marks)
        _lib.check(
            L.tmd_vv_second(self.ctx, s.vel.data_ptr(), s.forces.data_ptr(), ig.masses.data_ptr(), ig.dt, gamma, vcoeff,
                            None, ig.seed, 0, self.ke.data_ptr() if with_energy else None, stream)
        )
        self._mark(marks)

    def _graph(self, with_energy, parity=0):
        """Capture one step (kernels + exchange) once per variant; None if capture is not possible.
        A p2p step reads one position buffer and writes the other, so each parity is its own graph."""
        key = (with_energy, parity) if self.exchange == "p2p" else with_energy
        if key in self._graphs:
            return self._graphs[key]
        g = None
        if self.use_graph:
            try:
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                # the library edits the graph under capture (conditional node for the rebuild kernels, body
                # captured from a helper stream) -- relaxed mode permits that
                mode = "relaxed"  # (the library turns the rebuild into a conditional node of the graph under capture)
                with torch.cuda.graph(g, capture_error_mode=mode):
                    self._enqueue_step(with_energy, parity)
                # the capture only records; state was not advanced
            except Exception as err:  # pragma: no cover - depends on the NCCL build
                if self.rank == 0:
                    import sys

                    print(f"[domain] CUDA graph capture unavailable ({type(err).__name__}: {err}); stepping eagerly", file=sys.stderr)
                g = None
                self.use_graph = False
                torch.cuda.synchronize()
        self._graphs[key] = g
        return g

    def step(self, niter=1):
        """niter MD steps; returns (Ekin, pot, T) of the whole system like Integrator.step."""
        p2p = self.exchange == "p2p"
        L = _lib.lib()
        if p2p:  # the caller may have edited system.pos since the last call
            stream = torch.cuda.current_stream(self.system.pos.device).cuda_stream
            _lib.check(L.tmd_dd_load(self.ctx, self._parity, self.system.pos.data_ptr(), stream))
        for it in range(niter):
            last = it == niter - 1
            g = self._graph(last, self._parity)
            if g is not None:
                g.replay()
            else:
                self._enqueue_step(last, self._parity, self._marks)
            if p2p:
                self._parity ^= 1
        if p2p:
            stream = torch.cuda.current_stream(self.system.pos.device).cuda_stream
            _lib.check(L.tmd_dd_store(self.ctx, self._parity, self.system.pos.data_ptr(), stream))
        tot = torch.cat([self.ene.sum(dim=1), self.ke])  # this rank's shares
        dist.all_reduce(tot, group=self.group)
        self.forces.stats()  # raises on neighbour-row overflow / far positions
        host = tot.cpu().numpy()
        n = self.system.pos.shape[1]
        ekin = host[1:].astype("float32")
        return ekin, [float(host[0])], kinetic_to_temp(ekin, n)


def bench_decomposed(args, world, rank, local, config):
    """bench.py body for N > 1 (same workload as the single-GPU arm, strong scaling)."""
    import ctypes as C
    import json
    import os

    from . import Forces, System, maxwell_boltzmann, testsystems
    import bench as B

    dev = B.DEVICE_OVERRIDE or f"cuda:{local}"  # (the override: tests/test_domain_host.py dry-runs this function over gloo)
    wl = getattr(args, "workload", "water100k")
    sysd = testsystems.water_box(266664 if wl == "water800k" else B.N_WATERS, seed=0)
    n = len(sysd["coords"])
    par = testsystems.water_parameters(sysd, device=dev)
    system = System(n, 1, torch.float32, dev)
    system.set_positions(sysd["coords"])
    system.set_box(sysd["box"])
    torch.manual_seed(1)
    system.set_velocities(maxwell_boltzmann(par.masses, B.TEMPERATURE, 1))
    forces = Forces(par, terms=B.TERMS, **B.CFG)

    eq = DecomposedIntegrator(system, forces, B.TIMESTEP_FS, dev, gamma=10.0, T=B.TEMPERATURE, use_graph=False)
    forces.compute(system.pos, system.box, system.forces)  # sizes the neighbour rows (owned atoms)
    eq.step(niter=args.equil)
    integ = DecomposedIntegrator.__new__(DecomposedIntegrator)
    integ.__dict__.update(eq.__dict__)  # same buffers, production thermostat
    integ.integ = Integrator(system, forces, B.TIMESTEP_FS, dev, gamma=B.GAMMA_PS, T=B.TEMPERATURE)
    integ.integ.seed = eq.integ.seed
    integ.integ._require_cuda()
    integ.use_graph, integ._graphs = True, {}
    sampler = B.ClockSampler(local) if rank == 0 else None  # samples the warm-up too: same load
    st_a = forces.stats()
    # warm-up: at least 5000 steps (>= 0.4 s under load for the clock sampler); a FIXED count, the
    # same on every rank -- a wall-clock criterion could give ranks different numbers of collectives
    ekin, pot, T = integ.step(niter=max(3, args.warmup, B.MIN_DECOMPOSED_WARMUP))
    launches_per_step = None
    if integ.use_graph:  # kernels of one captured step (the capture itself went through the counting path)
        st_b = forces.stats()
        launches_per_step = (st_b["kernel_launches"] - st_a["kernel_launches"]) // max(1, len(integ._graphs))  # one step per captured graph

    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    st0 = forces.stats()
    dist.barrier()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    ekin, pot, T = integ.step(niter=args.steps)
    ev1.record()
    torch.cuda.synchronize()
    dist.barrier()
    clocks = sampler.stop() if sampler else None
    st1 = forces.stats()
    # pair-kernel duration: graph replays cannot be bracketed by host-recorded events, so the
    # same step is run eagerly for a short stretch right after the timed region
    eager = DecomposedIntegrator.__new__(DecomposedIntegrator)
    eager.__dict__.update(integ.__dict__)
    eager.use_graph, eager._graphs = False, {}
    nprof = min(100, args.steps)
    _lib.check(L.tmd_profile_begin(forces._ctx, nprof))
    eager._marks = []
    eager.step(niter=nprof)
    pair_ms, pair_n = C.c_double(), C.c_int()
    _lib.check(L.tmd_profile_end(forces._ctx, C.byref(pair_ms), C.byref(pair_n), stream))
    # phases of the eagerly issued steps (5 events per step): this rank's averages, then the slowest rank of each
    phase_names = ["integrate_first_half" + ("+push" if integ.exchange == "p2p" else ""), "exchange_wait" if integ.exchange == "p2p" else "exchange_allgather",
                   "forces_total(prepare+rebuild+pair+bonded)", "integrate_second_half"]
    phases = torch.zeros(4, dtype=torch.float64, device=dev)
    mk = eager._marks
    if B.DEVICE_OVERRIDE is None and len(mk) == 5 * nprof:
        for k in range(nprof):
            for q in range(4):
                phases[q] += mk[5 * k + q].elapsed_time(mk[5 * k + q + 1])
        phases /= nprof
    dist.all_reduce(phases, op=dist.ReduceOp.MAX)
    t = torch.tensor([ev0.elapsed_time(ev1), pair_ms.value / max(1, pair_n.value)], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)  # slowest rank
    ms_total, pair_avg_ms = float(t[0]), float(t[1])
    nl = launches_per_step * args.steps if launches_per_step else st1["kernel_launches"] - st0["kernel_launches"]
    launches = torch.tensor([nl], dtype=torch.int64, device=dev)
    dist.all_reduce(launches)

    # in-cutoff pairs of the whole system, each counted once: a rank evaluates every pair that touches one of its
    # atoms (pairs across a boundary on both sides), and counts those whose lower atom index it owns
    count = torch.zeros(1, dtype=torch.int64, device=dev)
    dummy = torch.zeros(2, dtype=torch.int32, device=dev)
    _lib.check(L.tmd_export_pairs(forces._ctx, system.pos.data_ptr(), 0, dummy.data_ptr(), 0, count.data_ptr(), stream))
    evaluated = int(count.item())
    buf = torch.empty((max(evaluated, 1), 2), dtype=torch.int32, device=dev)
    _lib.check(L.tmd_export_pairs(forces._ctx, system.pos.data_ptr(), 0, buf.data_ptr(), buf.shape[0], count.data_ptr(), stream))
    first = buf[: int(count.item()), 0]
    count = ((first >= integ.dec.lo) & (first < integ.dec.hi)).sum().to(torch.int64).reshape(1)
    dist.all_reduce(count)
    evaluated_t = torch.tensor([evaluated], dtype=torch.int64, device=dev)
    dist.all_reduce(evaluated_t)

    # end to end: host-resident positions in and out every step
    e2e_steps = min(args.steps, args.e2e_steps)
    hpos = torch.empty(system.pos.shape, dtype=torch.float32, pin_memory=B.DEVICE_OVERRIDE is None)
    hpos.copy_(system.pos)
    for k in range(3 + e2e_steps):
        if k == 3:
            dist.barrier()
            torch.cuda.synchronize()
            import time

            t0 = time.perf_counter()
        system.pos.copy_(hpos, non_blocking=True)
        integ.step(niter=1)
        hpos.copy_(system.pos, non_blocking=True)
        torch.cuda.synchronize()
    t_e2e = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device=dev)
    dist.all_reduce(t_e2e, op=dist.ReduceOp.MAX)

    if rank != 0:
        return
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(B.ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    peak = float(peaks.get("hbm_gbs", B.FALLBACK_HBM_GBS))
    ms_per_step = ms_total / args.steps
    # cross-rank pairs are seen from both owners: halve them out of the per-rank byte model by
    # using the single-GPU definition on the whole system, divided over the ranks
    p_rc_total = None
    alg_bytes_rank = None
    achieved = None
    line = {
        "metric": B.METRICS[wl],
        "value": 1e3 / ms_per_step,
        "unit": "steps/s",
        "n_gpus": world,
        "steps": args.steps,
        "warmup": max(3, args.warmup),
        "ms_per_step": ms_per_step,
        "higher_is_better": True,
        "scaling": "weak" if wl == "water800k" else "strong",
        "vs_baseline": None,
        "dtype": "f32",
        "data": "synthetic",
        "config": config,
        "clocks": clocks,
        "e2e": {
            "value": e2e_steps / float(t_e2e[0]),
            "unit": "steps/s",
            "h2d_bytes_per_step": system.pos.numel() * 4,
            "d2h_bytes_per_step": system.pos.numel() * 4 + 16,
            "steps": e2e_steps,
            "api": "DecomposedIntegrator.step(1) with pinned host positions copied in and out every step",
        },
        "gpu_launches": int(launches.item()),
        "roofline": {
            "kernel": "non-bonded pair kernel %s, slowest rank; timed over %d eager steps after the graph-replayed timed region" % (_lib.PAIR_KERNEL_NAMES[int(L.tmd_pair_kernel(forces._ctx))], nprof),
            "bound": "hbm",
            "achieved": (32.0 * n / world + 4.0 * int(count.item()) / world) / (pair_avg_ms * 1e-3) / 1e9 if pair_avg_ms > 0 else 0.0,
            "peak": peak,
            "unit": "GB/s",
            "frac": ((32.0 * n / world + 4.0 * int(count.item()) / world) / (pair_avg_ms * 1e-3) / 1e9 / peak) if pair_avg_ms > 0 else 0.0,
            "peak_source": "MEASURED_PEAKS.json hbm_gbs (measured)" if "hbm_gbs" in peaks else "H100 SXM data sheet, 3350 GB/s (not measured)",
            "algorithmic_bytes": 32.0 * n / world + 4.0 * int(count.item()) / world,
            "pairs_in_cutoff": int(count.item()),
            "pair_entries_counted": int(count.item()),
            "pairs_evaluated_all_ranks": int(evaluated_t.item()),
            "avg_kernel_ms": pair_avg_ms,
            "share_of_step": pair_avg_ms / ms_per_step,
            "traffic": None,
        },
        "cpu_baseline": None,
        "state": {
            "temperature_K": float(T[0]),
            "epot": float(pot[0]),
            "rebuilds_in_timed_region": int(st1["rebuilds"] - st0["rebuilds"]),
            "cuda_graph": bool(integ.use_graph),
            "phase_ms_eager_slowest_rank": {k: float(v) for k, v in zip(phase_names, phases.tolist())},
            "phase_note": "CUDA events between the calls of %d steps issued kernel by kernel after the timed region (the timed steps are graph replays); per phase the maximum over ranks, so the sum exceeds one step of the slowest rank" % nprof,
            "collective": "one all-gather of positions per step (NCCL)" if integ.exchange == "allgather"
            else "none: positions stored into every rank's buffer by the integration kernel (NVLink peer memory) + flag wait",
        },
    }
    print(json.dumps(line), flush=True)
