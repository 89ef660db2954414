"""``ReplicaExchange``: parallel tempering (temperature replica exchange) for ``Integrator``.

``Integrator(systems, forces, dt, device, gamma=g, T=[T0 < T1 < ... < T_{R-1}], replica_exchange=ReplicaExchange(...))``
runs R replicas on a ladder of R temperatures.  ``ladder()[r]`` is the temperature index of replica r (the identity at
the start); replica r's Langevin noise scale is row ``ladder()[r]`` of the integrator's (R, N, 1) ``vcoeff`` table.

After every ``frequency``-th step (counted on the integrator's step index across ``step`` calls) the device tries
swaps between neighbouring temperatures, alternating the even pairs (0,1), (2,3), ... and the odd ones (1,2), (3,4),
...: slots k and k+1, held by replicas i and j, swap with probability min(1, exp((beta_k - beta_{k+1}) (U_i - U_j))),
beta = 1 / (kB T), U the replica's potential energy.  A replica that changes temperature has its velocities scaled by
sqrt(T_new / T_old).  The decision and the scaling run on the GPU in stream order (``tmd_replica_exchange``,
csrc/remd.cuh): no read-back, and the captured MD steps stay valid.  The uniforms come from Philox4x32-10 keyed on
``seed`` in a counter domain of their own (``oracle/remd.py`` restates the rule).
"""
import numpy as np
import torch

from . import _lib


class ReplicaExchange:
    """Temperature replica exchange for ``Integrator(..., T=[...], replica_exchange=...)``.

    frequency : an attempt after every ``frequency``-th step.  seed : of the exchange draws, by default drawn from
    torch's generator (``torch.manual_seed`` makes runs reproducible).
    """

    def __init__(self, frequency=1000, seed=None):
        if int(frequency) < 1 or int(frequency) != frequency:
            raise ValueError("ReplicaExchange: frequency must be an integer >= 1")
        self.frequency = int(frequency)
        self.seed = int(torch.randint(0, 2**62, (1,)).item()) if seed is None else int(seed)
        self.attempts = 0  # attempts made so far; attempt a tries the pairs (k, k+1) with k = a (mod 2)
        self._integ = None
        self._counts = None

    def _bind(self, integ):
        """Checks the integrator can run a ladder (called by Integrator, after it has checked T)."""
        temps = integ.temperatures
        if integ.gamma is None or temps is None:
            raise RuntimeError("ReplicaExchange needs a thermostat: give the Integrator gamma and a list of temperatures")
        if len(temps) < 2:
            raise ValueError("ReplicaExchange needs at least two replicas")
        if any(b <= a for a, b in zip(temps, temps[1:])):
            raise ValueError("ReplicaExchange: the temperatures must be strictly increasing")
        self._integ = integ
        self._counts = torch.zeros((len(temps) - 1, 2), dtype=torch.int64, device=integ.systems.pos.device)

    def attempt(self, ctx, energies, stride, nterms):
        """Enqueue one attempt on the current stream from the (R, stride) fp64 device ``energies`` (the first
        ``nterms`` columns summed per replica), scaling ``systems.vel`` of the replicas that change temperature."""
        s = self._integ.systems
        f64 = s.pos.dtype == torch.float64
        fn = _lib.lib().tmd_replica_exchange_f64 if f64 else _lib.lib().tmd_replica_exchange
        stream = torch.cuda.current_stream(s.pos.device).cuda_stream
        _lib.check(fn(ctx, energies.data_ptr(), stride, nterms, self.seed, self.attempts, s.vel.data_ptr(),
                      self._counts.data_ptr(), stream))
        self.attempts += 1

    # ------------------------------------------------------------------ read-outs (one device-to-host copy each)
    def ladder(self):
        """(R,) int: the temperature index of each replica."""
        return self._integ._ladder.cpu().numpy().astype(np.int64)

    def temperatures(self):
        """(R,) float: the current temperature of each replica (K)."""
        return np.asarray(self._integ.temperatures, dtype=np.float64)[self.ladder()]

    def acceptance(self):
        """(R-1,) float: accepted / attempted swaps of each neighbour pair of temperatures (nan before an attempt)."""
        c = self._counts.cpu().numpy().astype(np.float64)
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(c[:, 0] > 0, c[:, 1] / c[:, 0], np.nan)

    def counts(self):
        """(R-1, 2) int: attempted and accepted swaps of each neighbour pair of temperatures."""
        return self._counts.cpu().numpy()
