"""ctypes binding of ``libtmd_b200.so`` (C ABI declared in ``include/tmd_b200.h``).

There is no CPU fallback: if the shared library has not been built
(``python -c 'import __graft_entry__ as g; g.build()'``) importing anything that
computes raises immediately.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TMD_B200_LIB", os.path.join(_HERE, "libtmd_b200.so"))  # override: tuning builds only

OK = 0
ERR_OVERFLOW = -4

# energy slots, same order as include/tmd_b200.h
ENERGY_SLOTS = (
    "bonds",
    "angles",
    "dihedrals",
    "impropers",
    "1-4",
    "electrostatics",
    "lj",
    "repulsion",
    "repulsioncg",
)
NUM_ENERGIES = len(ENERGY_SLOTS)


# tmd_pair_kernel() ids (include/tmd_b200.h): the non-bonded pair kernel the last force call ran
PAIR_ROWS, PAIR_ROWS_FX, PAIR_ROWS_FX2, PAIR_OPEN_FX2, PAIR_CLUSTER, PAIR_F64 = 0, 1, 2, 3, 4, 5
PAIR_EWALD, PAIR_EWALD_FX, PAIR_EWALD_F64, PAIR_EWALD_FX2, PAIR_EWALD_CLUSTER = 6, 7, 8, 9, 10
PAIR_KERNEL_NAMES = {
    PAIR_ROWS: "k_pair (full rows)",
    PAIR_ROWS_FX: "k_pair_fx (full rows, fixed point)",
    PAIR_ROWS_FX2: "k_pair_fx2 (full rows, fixed point, fp32x2)",
    PAIR_OPEN_FX2: "k_pair2_open (full rows without a box, fp32x2)",
    PAIR_CLUSTER: "k_cpair (cluster half list)",
    PAIR_F64: "k_pair_f64 (full rows, fp64)",
    PAIR_EWALD: "k_pair (full rows, real-space Ewald)",
    PAIR_EWALD_FX: "k_pair_fx (full rows, fixed point, real-space Ewald)",
    PAIR_EWALD_F64: "k_ewpair64 (full rows, fp64, real-space Ewald)",
    PAIR_EWALD_FX2: "k_pair_fx2_ew (full rows, fixed point, fp32x2, real-space Ewald)",
    PAIR_EWALD_CLUSTER: "k_cpair_ew (cluster half list, real-space Ewald)",
}


def term_mask(terms):
    m = 0
    for t in terms:
        m |= 1 << ENERGY_SLOTS.index(t)
    return m


class Stats(C.Structure):
    _fields_ = [
        ("rebuilds", C.c_int64),
        ("force_calls", C.c_int64),
        ("max_neighbours", C.c_int32),
        ("row_capacity", C.c_int32),
        ("overflow", C.c_int32),
        ("ncells", C.c_int32 * 3),
        ("kernel_launches", C.c_int64),
    ]


_P = C.c_void_p
IPC_HANDLE_BYTES = 64  # TMD_IPC_HANDLE_BYTES
MAX_PEERS = 16  # TMD_MAX_PEERS
_SIGNATURES = {
    "tmd_last_error": (C.c_char_p, []),
    "tmd_version": (C.c_int, []),
    "tmd_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.c_int]),
    "tmd_destroy": (C.c_int, [_P]),
    "tmd_set_atoms": (C.c_int, [_P, _P, _P, C.c_int, _P, _P]),
    "tmd_set_exclusions": (C.c_int, [_P, _P, _P]),
    "tmd_set_nonbonded": (C.c_int, [_P, C.c_uint32, C.c_double, C.c_double, C.c_int, C.c_double, C.c_double, C.c_double]),
    "tmd_set_bonds": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_angles": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_torsions": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, C.c_int]),
    "tmd_set_pairs14": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_box": (C.c_int, [_P, _P]),
    "tmd_forces": (C.c_int, [_P, _P, _P, _P, _P]),
    "tmd_vv_first": (C.c_int, [_P, _P, _P, _P, _P, C.c_double, _P]),
    "tmd_vv_second": (C.c_int, [_P, _P, _P, _P, C.c_double, C.c_double, _P, _P, C.c_uint64, C.c_uint64, _P, _P]),
    "tmd_kinetic_energy": (C.c_int, [_P, _P, _P, _P, _P]),
    "tmd_md_steps": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_double, C.c_double, _P, _P, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "tmd_md_steps_host": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, _P, C.c_double, C.c_double, _P, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "tmd_export_pairs": (C.c_int, [_P, _P, C.c_int, _P, C.c_int64, _P, _P]),
    "tmd_get_stats": (C.c_int, [_P, C.POINTER(Stats), _P]),
    "tmd_set_owned_atoms": (C.c_int, [_P, C.c_int, C.c_int]),
    "tmd_set_force_convention": (C.c_int, [_P, C.c_int]),
    "tmd_pair_kernel": (C.c_int, [_P]),
    "tmd_dd_create": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "tmd_dd_connect": (C.c_int, [_P, _P]),
    "tmd_dd_load": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_dd_store": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_dd_vv_first_push": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_double, _P]),
    "tmd_dd_wait": (C.c_int, [_P, _P]),
    "tmd_dd_forces": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "tmd_wrapper_create": (C.c_int, [C.POINTER(_P), C.c_int, C.c_int, C.c_int, _P, _P]),
    "tmd_wrapper_wrap": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    "tmd_wrapper_destroy": (C.c_int, [_P]),
    "tmd_profile_begin": (C.c_int, [_P, C.c_int]),
    "tmd_profile_end": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_int), _P]),
    # "precision: double" (library version >= 101)
    "tmd_set_precision": (C.c_int, [_P, C.c_int]),
    "tmd_set_atoms_f64": (C.c_int, [_P, _P, _P, C.c_int, _P, _P]),
    "tmd_set_bonds_f64": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_angles_f64": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_torsions_f64": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, C.c_int]),
    "tmd_set_pairs14_f64": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_box_f64": (C.c_int, [_P, _P]),
    "tmd_forces_f64": (C.c_int, [_P, _P, _P, _P, _P]),
    "tmd_vv_first_f64": (C.c_int, [_P, _P, _P, _P, _P, C.c_double, _P]),
    "tmd_vv_second_f64": (C.c_int, [_P, _P, _P, _P, C.c_double, C.c_double, _P, _P, C.c_uint64, C.c_uint64, _P, _P]),
    "tmd_kinetic_energy_f64": (C.c_int, [_P, _P, _P, _P, _P]),
    "tmd_md_steps_f64": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_double, C.c_double, _P, _P, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "tmd_export_pairs_f64": (C.c_int, [_P, _P, C.c_int, _P, C.c_int64, _P, _P]),
    "tmd_wrapper_wrap_f64": (C.c_int, [_P, _P, _P, C.c_int, _P]),
    # constraints (library version >= 102)
    "tmd_set_constraints": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, _P, _P, _P]),
    "tmd_constrain": (C.c_int, [_P, _P, _P, _P, _P]),
    "tmd_constrain_f64": (C.c_int, [_P, _P, _P, _P, _P]),
    # particle-mesh Ewald (library version >= 103)
    "tmd_set_pme": (C.c_int, [_P, C.c_double]),
    "tmd_get_pme": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_int32 * 3)]),
    # box rescale and molecule scaling (library version >= 104)
    "tmd_rescale_box": (C.c_int, [_P, _P, _P]),
    "tmd_rescale_box_f64": (C.c_int, [_P, _P, _P]),
    "tmd_set_molecules": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "tmd_scale_molecules": (C.c_int, [_P, _P, _P, _P]),
    "tmd_scale_molecules_f64": (C.c_int, [_P, _P, _P, _P]),
    "tmd_step_captures": (C.c_int64, [_P]),
    "tmd_rewind_noise": (C.c_int, [_P, C.c_int, _P]),
    # CMAP correction maps (library version >= 105)
    "tmd_set_cmap": (C.c_int, [_P, C.c_int, _P, _P, C.c_int, _P, _P]),
    # Urey-Bradley terms (library version >= 106)
    "tmd_set_urey_bradley": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_set_urey_bradley_f64": (C.c_int, [_P, C.c_int, _P, _P]),
    # temperature ladder and replica exchange (library version >= 107)
    "tmd_set_temperature_ladder": (C.c_int, [_P, C.c_int, _P, _P]),
    "tmd_replica_exchange": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "tmd_replica_exchange_f64": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_uint64, C.c_uint64, _P, _P, _P]),
    # OBC2 implicit solvent (library version >= 108)
    "tmd_set_gb": (C.c_int, [_P, C.c_int, _P, _P, C.c_double, C.c_double]),
}
ERR_UNSUPPORTED = -5
EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


def lib():
    """The loaded library; raises if it is missing (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: the CUDA extension is not built. Run "
                "`python -c \"import __graft_entry__ as g; g.build()\"` in the repository root. "
                "torchmd_b200 has no CPU or PyTorch fallback."
            )
        handle = C.CDLL(LIB_PATH)
        if not hasattr(handle, "tmd_set_gb"):
            raise ImportError(f"{LIB_PATH} predates the implicit-solvent entry point: rebuild it (__graft_entry__.build())")
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        if handle.tmd_version() < 100:
            raise ImportError(
                f"{LIB_PATH} is the host SIMT-interpreter build of the kernels (tests/simt, a unit-test tool): "
                "torchmd_b200 runs on the CUDA library only"
            )
        if handle.tmd_version() < 101:
            raise ImportError(f"{LIB_PATH} predates the fp64 entry points: rebuild it (__graft_entry__.build())")
        _lib = handle
    return _lib


def on_device(t):
    """True for a tensor in CUDA memory -- the one definition the host classes use for "must be a CUDA tensor"."""
    return bool(t.is_cuda)


class TmdError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"tmd_b200 error {code}: {msg}")
        self.code = code


def check(code):
    if code != OK:
        raise TmdError(code, lib().tmd_last_error().decode())
    return code


def ptr(t):
    """Raw device/host pointer of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data
