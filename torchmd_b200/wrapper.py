"""``Wrapper`` -- molecules back into the periodic box (mirror of torchmd/wrapper.py).

Same constructor and ``wrap(pos, box, wrapidx=None)`` call as the reference
(wrapper.py:4-30; used by run.py:242,266 every output period).  The reference loops over
the molecule groups in Python -- 33,333 iterations of ~5 torch ops for the 100k-atom water
box; here the groups are a CSR and one CUDA kernel (csrc/wrap.cuh) moves every group of
every replica, one warp per group.  CUDA fp32 or fp64 tensors, no fallback.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib


def calculate_molecule_groups(natoms, bonds, device="cpu"):
    """Connected components of the bond graph (wrapper.py:33-55): ``(molgroups, nongrouped)``
    with ``molgroups`` a list of index tensors (components of two or more atoms, atoms in
    ascending order, components ordered by their smallest atom) and ``nongrouped`` the atoms
    that belong to no bond.  Union-find on the host instead of networkx."""
    groups, single = _components(natoms, bonds)
    molgroups = [torch.tensor(g, dtype=torch.int64, device=device) for g in groups]
    nongrouped = torch.tensor(single, dtype=torch.int64, device=device)
    return molgroups, nongrouped


def _components(natoms, bonds):
    if bonds is None or len(bonds) == 0:
        return [], list(range(natoms))
    b = np.asarray(bonds).astype(np.int64).reshape(-1, 2)
    if b.min() < 0 or b.max() >= natoms:
        raise ValueError("bond index outside the system")
    parent = np.arange(natoms)

    def find(x):
        root = x
        while parent[root] != root:
            root = parent[root]
        while parent[x] != root:  # path compression
            parent[x], x = root, parent[x]
        return root

    for i, j in b:
        ri, rj = find(int(i)), find(int(j))
        if ri != rj:
            if ri < rj:
                parent[rj] = ri
            else:
                parent[ri] = rj
    roots = np.fromiter((find(i) for i in range(natoms)), dtype=np.int64, count=natoms)
    order = np.argsort(roots, kind="stable")  # members ascending inside a component, components by smallest atom
    sroots = roots[order]
    starts = np.flatnonzero(np.r_[True, sroots[1:] != sroots[:-1]])
    ends = np.r_[starts[1:], natoms]
    groups, single = [], []
    for s, e in zip(starts, ends):
        if e - s == 1:
            single.append(int(order[s]))
        else:
            groups.append(order[s:e].tolist())
    return groups, single


class Wrapper:
    def __init__(self, natoms, bonds, device):
        self.natoms = int(natoms)
        self.device = torch.device(device)
        groups, single = _components(self.natoms, bonds)
        self.groups = [torch.tensor(g, dtype=torch.int64, device=device) for g in groups]
        self.nongrouped = torch.tensor(single, dtype=torch.int64, device=device)
        # CSR over all atoms: the bonded components first, then one-atom groups
        members = [a for g in groups for a in g] + single
        sizes = [len(g) for g in groups] + [1] * len(single)
        self._ptr = np.zeros(len(sizes) + 1, dtype=np.int32)
        np.cumsum(sizes, out=self._ptr[1:])
        self._atoms = np.asarray(members, dtype=np.int32)
        self._handle = None

    def _ensure(self, pos):
        if self._handle is None:
            if not _lib.on_device(pos):
                raise RuntimeError("torchmd_b200.Wrapper runs on CUDA tensors only (no CPU fallback)")
            h = C.c_void_p()
            _lib.check(_lib.lib().tmd_wrapper_create(C.byref(h), pos.device.index or 0, self.natoms, len(self._ptr) - 1,
                                                     self._ptr.ctypes.data, self._atoms.ctypes.data))
            self._handle, self._device = h, pos.device
        return self._handle

    def wrap(self, pos, box, wrapidx=None):
        """In place on ``pos`` (R,N,3); ``box`` (R,3,3), diagonal used (wrapper.py:8-30)."""
        if wrapidx is not None:
            # wrapper.py:17-21 rebinds the local name `pos` to a new tensor: everything after it
            # acts on that temporary and the caller's tensor is left untouched.  Same here.
            return
        if pos.dtype not in (torch.float32, torch.float64) or box.dtype != pos.dtype:
            raise RuntimeError("torchmd_b200.Wrapper needs positions and box of one dtype, float32 or float64")
        if pos.dim() != 3 or pos.shape[1] != self.natoms or pos.shape[2] != 3 or tuple(box.shape) != (pos.shape[0], 3, 3):
            raise RuntimeError("wrap: pos must be (nreplicas, natoms, 3) and box (nreplicas, 3, 3)")
        if not pos.is_contiguous() or not box.is_contiguous():
            raise RuntimeError("wrap: pos and box must be contiguous")
        h = self._ensure(pos)
        if not _lib.on_device(pos) or not _lib.on_device(box) or pos.device != self._device or box.device != pos.device:
            raise RuntimeError(f"wrap: pos and box must both live on {self._device} (got {pos.device} and {box.device})")
        stream = torch.cuda.current_stream(pos.device).cuda_stream
        fn = _lib.lib().tmd_wrapper_wrap_f64 if pos.dtype == torch.float64 else _lib.lib().tmd_wrapper_wrap
        _lib.check(fn(h, pos.data_ptr(), box.data_ptr(), pos.shape[0], stream))

    def __del__(self):
        h, self._handle = getattr(self, "_handle", None), None
        if h is not None:
            try:
                _lib.lib().tmd_wrapper_destroy(h)
            except Exception:
                pass
