"""H100-native MD inner loop behind torchmd's System / Forces.compute / Integrator.step.

Host classes mirror the reference interface (``torchmd/systems.py``,
``torchmd/forces.py``, ``torchmd/integrator.py``); the arithmetic runs in
hand-written sm_90a CUDA kernels reached through the C ABI of
``include/tmd_b200.h`` (``libtmd_b200.so``, built in-tree by
``__graft_entry__.build()``).  There is no CPU or stock-PyTorch fallback.
"""
from .systems import System  # noqa: F401
from .forces import Forces  # noqa: F401
from .integrator import Integrator, kinetic_energy, kinetic_to_temp, maxwell_boltzmann  # noqa: F401
from .parameters import TopologyParameters  # noqa: F401
from .constraints import Constraints  # noqa: F401
from .wrapper import Wrapper  # noqa: F401
from .barostat import MonteCarloBarostat  # noqa: F401

__version__ = "0.1.0"
