"""The in-kernel Langevin noise restated in numpy: Philox4x32-10 and the two Box-Muller transforms of the kernels.

Written from the definition of Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2,
3", SC'11) and from the device code (``torchmd_b200/csrc/integrate.cuh`` ``normal3`` on float and on double),
with vectorised uint64 arithmetic: the draw of every (seed, step, slot) can be computed on the host, exactly, and the
kernels compared with it draw for draw.

The stream a run draws (``langevin_noise``): the noise of atom ``i`` of replica ``r`` at the k-th step (k = 1, 2, ...)
of a context is ``normal3(seed, first_step + position + k, r * N + i)``.  ``position`` is the context's Philox position
(device ``counters[1]``): zero when the context is created and advanced by one at every first half-kick, so the first
step of a fresh context draws with step 1; ``first_step`` is the offset the C entry points take (``Integrator`` passes
0).  Step and slot are 64-bit and wrap modulo 2**64 like the device's ``uint64_t``.

Agreement with the device:

* The Philox words and the uniforms built from them are integer or exactly rounded fp32 / fp64 operations: bitwise.
* ``normal3_f32``: ``logf``, ``sqrtf``, ``sincosf`` and ``cosf`` are evaluated here in fp64 and rounded to fp32
  (the correctly rounded value).  The CUDA library (built without fast math) has ``logf`` within 1 ulp and
  ``sincosf`` / ``cosf`` within 2 ulp, so a device draw is within about 4 ulp of |xi| of this one:
  ``|xi_dev - xi| <= F32_BOUND * max(1, |xi|)`` with ``F32_BOUND = 2e-6``.  A host build of the kernels against a
  libm with sub-ulp ``logf`` / ``sinf`` / ``cosf`` agrees to about 1 ulp.
* ``normal3_f64``: fp64 Box-Muller with numpy's ``log`` / ``sin`` / ``cos``; the device functions are within 1-2 ulp,
  so ``|xi_dev - xi| <= F64_BOUND * max(1, |xi|)`` with ``F64_BOUND = 1e-14`` (observed: about 1e-15).
"""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)  # round multipliers
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)  # Weyl increments of the key
MASK32 = np.uint64(0xFFFFFFFF)
TOP_BIT = np.uint64(0x80000000)  # counter word 1 of the second block of the fp64 normal3

F32_BOUND = 2e-6
F64_BOUND = 1e-14

TWO_PI_F32 = np.float32(6.283185307179586)
TWO_PI_F64 = 6.283185307179586


def _u64(x):
    return np.asarray(x, dtype=np.uint64) if not isinstance(x, int) else np.uint64(x)


def philox4x32_10(counter, key):
    """Ten Philox4x32 rounds.  ``counter``: four arrays (or ints) of 32-bit words c0..c3, ``key``: two (k0, k1); they
    broadcast against each other.  Returns the four output words as uint64 arrays holding 32-bit values.

    Round: (hi(M1*c2) ^ c1 ^ k0, lo(M1*c2), hi(M0*c0) ^ c3 ^ k1, lo(M0*c0)), then the key takes the Weyl increments."""
    c0, c1, c2, c3 = (np.asarray(_u64(c), dtype=np.uint64) & MASK32 for c in counter)
    k0, k1 = (np.asarray(_u64(k), dtype=np.uint64) & MASK32 for k in key)
    shape = np.broadcast_shapes(c0.shape, c1.shape, c2.shape, c3.shape, k0.shape, k1.shape)
    c0, c1, c2, c3, k0, k1 = (np.broadcast_to(a, shape).copy() for a in (c0, c1, c2, c3, k0, k1))
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c0  # 32 x 32 -> 64 bits: no overflow in uint64
            p1 = M1 * c2
            c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & MASK32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & MASK32
            k0 = (k0 + W0) & MASK32
            k1 = (k1 + W1) & MASK32
    return c0, c1, c2, c3


def _words(seed, step, slot):
    """The counter (slot lo, slot hi, step lo, step hi) and key (seed lo, seed hi) of one draw."""
    seed, step, slot = (np.asarray(_u64(x), dtype=np.uint64) for x in (seed, step, slot))
    s32 = np.uint64(32)
    return (slot & MASK32, slot >> s32, step & MASK32, step >> s32), (seed & MASK32, seed >> s32)


def _uniform_f32(u):
    """((float)(u >> 8) + 0.5f) * 2^-24, each operation rounded to fp32 (the sum needs 25 bits at the top of the range)."""
    return ((u >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0)


def _f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32)


def normal3_f32(seed, step, slot):
    """The three fp32 N(0,1) draws of ``normal3`` (integrate.cuh) for each (seed, step, slot): array (..., 3) float32."""
    counter, key = _words(seed, step, slot)
    return box_muller_f32(philox4x32_10(counter, key))


def box_muller_f32(u):
    """``normal3``'s transform of one Philox block (four 32-bit words): array (..., 3) float32."""
    u0, u1, u2, u3 = (_uniform_f32(np.asarray(w, np.uint64)) for w in u)
    # sqrtf(-2.0f * logf(u)): log rounded to fp32, the product by -2 is exact, sqrt of an fp32 rounded to fp32
    r0 = _f32(np.sqrt((np.float32(-2.0) * _f32(np.log(u0.astype(np.float64)))).astype(np.float64)))
    r1 = _f32(np.sqrt((np.float32(-2.0) * _f32(np.log(u2.astype(np.float64)))).astype(np.float64)))
    a1 = TWO_PI_F32 * u1  # fp32 product
    a3 = TWO_PI_F32 * u3
    s, c = _f32(np.sin(a1.astype(np.float64))), _f32(np.cos(a1.astype(np.float64)))
    c3 = _f32(np.cos(a3.astype(np.float64)))
    return np.stack([r0 * c, r0 * s, r1 * c3], axis=-1).astype(np.float32)


def u53(hi, lo):
    """53-bit uniform in (0, 1) from two 32-bit words: (((hi >> 5) << 26 | lo >> 6) + 0.5) * 2^-53 (exact in fp64)."""
    hi, lo = np.asarray(hi, np.uint64), np.asarray(lo, np.uint64)
    m = ((hi >> np.uint64(5)) << np.uint64(26)) | (lo >> np.uint64(6))
    return (m.astype(np.float64) + 0.5) * (1.0 / 9007199254740992.0)


def normal3_f64(seed, step, slot):
    """The three fp64 N(0,1) draws of ``normal3`` on double (integrate.cuh): two Philox blocks, the second with the top bit of
    counter word 1 set, four 53-bit uniforms, Box-Muller in fp64.  Array (..., 3) float64."""
    (c0, c1, c2, c3), key = _words(seed, step, slot)
    return box_muller_f64(philox4x32_10((c0, c1, c2, c3), key), philox4x32_10((c0, c1 | TOP_BIT, c2, c3), key))


def box_muller_f64(u, w):
    """``normal3_f64``'s transform of its two Philox blocks ``u`` and ``w``: array (..., 3) float64."""
    r0 = np.sqrt(-2.0 * np.log(u53(u[0], u[1])))
    r1 = np.sqrt(-2.0 * np.log(u53(w[0], w[1])))
    a = TWO_PI_F64 * u53(u[2], u[3])
    b = TWO_PI_F64 * u53(w[2], w[3])
    return np.stack([r0 * np.cos(a), r0 * np.sin(a), r1 * np.cos(b)], axis=-1)


def langevin_noise(seed, nsteps, nrep, natoms, dtype=np.float32, position=0, first_step=0):
    """The (nsteps, nrep, natoms, 3) draws of ``nsteps`` steps of a run: step k (1-based) of the call draws with
    Philox step ``first_step + position + k`` (mod 2**64), atom i of replica r with slot ``r * natoms + i``.
    ``position``: the context's Philox position before the call (the number of steps it has run, for a context that
    ``Integrator`` drives); ``dtype``: float32 for ``normal3``, float64 for ``normal3_f64``."""
    f64 = str(dtype) == "torch.float64" or (not str(dtype).startswith("torch.") and np.dtype(dtype) == np.float64)
    fn = normal3_f64 if f64 else normal3_f32
    base = (int(first_step) + int(position)) % (1 << 64)
    steps = np.array([(base + k) % (1 << 64) for k in range(1, nsteps + 1)], dtype=np.uint64)
    slots = np.arange(nrep * natoms, dtype=np.uint64).reshape(nrep, natoms)
    out = fn(seed, steps[:, None, None], slots[None])
    return out.reshape(nsteps, nrep, natoms, 3)
