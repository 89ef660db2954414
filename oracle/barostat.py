"""numpy fp64 reference of the barostat's molecule move (torchmd_b200/csrc/barostat.cuh, k_scale_molecules).

For every molecule of every replica: unwrap along its bond tree (u = u_parent + minimum image of r - r_parent), take the
centroid c of the unwrapped atoms, and move each atom to r + (s - 1) c + n (s L - L), n = rint((r - u) / L) its image
in the molecule's unwrapped frame.  Same operations in the same order as the kernel, so that with contraction off the
two agree to the final rounding.
"""
import numpy as np


def image(d, L):
    return d - L * np.rint(d / L)


def scale_molecules(pos, L, s, ptr, atoms, parent):
    """pos (R,N,3) positions (any float dtype, read as fp64), L (R,3) box lengths, s (R,3) scale factors; ptr / atoms /
    parent the molecule CSR of tmd_set_molecules.  Returns the moved positions in fp64 (round them to the state's
    dtype once)."""
    x = np.asarray(pos, dtype=np.float64)
    L = np.asarray(L, dtype=np.float64)
    s = np.asarray(s, dtype=np.float64)
    out = x.copy()
    R = x.shape[0]
    for r in range(R):
        u = np.zeros_like(x[r])
        for m in range(len(ptr) - 1):
            k0, k1 = int(ptr[m]), int(ptr[m + 1])
            c = np.zeros(3)
            for k in range(k0, k1):
                a, p = int(atoms[k]), int(parent[k])
                if a == p:
                    u[a] = x[r, a]
                else:
                    u[a] = u[p] + image(x[r, a] - x[r, p], L[r])
                c += u[a]
            shift = (s[r] - 1.0) * (c * (1.0 / (k1 - k0)))
            dL = s[r] * L[r] - L[r]
            for k in range(k0, k1):
                a = int(atoms[k])
                n = np.rint((x[r, a] - u[a]) / L[r])
                out[r, a] = x[r, a] + (shift + n * dL)
    return out
