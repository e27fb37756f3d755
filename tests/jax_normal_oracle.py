"""NumPy restatement of ``jax.random.normal`` in fp32 (jax 0.4.x ``_normal_real``), test infrastructure for
``normal_from_bits`` / ``normal_scalar`` in ``purejaxql_b200/csrc/threefry.cuh`` and ``pqn_random_normal``.

It extends ``oracle/jax_prng.py`` (threefry, ``random_bits``, ``uniform``), which it reuses unchanged, and lives
beside the other test oracles so that the ``oracle`` package stays as it is.

    u = uniform(key, shape, lo = nextafter(-1, 0), hi = 1)
    normal = sqrt(2) * erf_inv(u)                      sqrt(2) rounded to fp32

``erf_inv`` is XLA's fp32 form of M. Giles' single-precision approximation ("Approximating the erfinv function", GPU
Computing Gems Jade Edition, 2011), as ``chlo.erf_inv`` lowers it:

    w = -log1p(-x * x)
    w < 5:  t = w - 2.5,      p = Horner over CENTRAL in t
    else:   t = sqrt(w) - 3,  p = Horner over TAIL in t
    erf_inv(x) = x * inf where |x| == 1, else p * x

PARITY UNPINNED: no jax is installable here.  Recollected points, each checked by
``tests/golden/make_gaussian_bandit_golden_from_ref.py`` once it has run:

(J1) ``_normal_real``'s formula and bounds above; ``uniform`` clamps with ``max(lo, .)`` (never active here: the
     uniform is 2 f - (1 - 2^-24) for f = (bits >> 9) * 2^-23, exact in fp32, never 0 and never +-1).
(J2) Giles' coefficients and the w < 5 split, as XLA restates them (the constants below).
(J3) On a CUDA device XLA calls libdevice's ``log1pf`` on the rounded product x * x (no fma into log1pf's internals).
(J4) On a CUDA device each Horner step p * t + c is one fma (LLVM's NVPTX backend contracts the fmul / fadd pair);
     ``FMA = False`` restates the uncontracted form of jax on the CPU.

The log1p is the one point where NumPy cannot restate libdevice: ``log1p`` defaults to the fp64 log1p rounded to fp32
(correctly rounded but for rare double roundings), and tests pass the platform's own log1pf (the host C library's, or
libdevice's through torch on the GPU) where they check bits.  A log1pf within 1 ulp of the exact value gives a w
within 1 ulp of this one, and ``NORMAL_ULP_BOUND`` is the most that a 1-ulp change of w moves the normal: 3 ulps,
found by trying both neighbours of w at all 2^23 inputs (tests/test_gaussian_bandit_host.py asserts it).  The
polynomial part itself (``erf_inv_from_w``) restates the C++ bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import jax_prng as jr

F32 = np.float32
LO = np.nextafter(F32(-1), F32(0))                      # -(1 - 2^-24)
SQRT2 = F32(np.sqrt(2.0))
CENTRAL = np.array([2.81022636e-08, 3.43273939e-07, -3.5233877e-06, -4.39150654e-06, 0.00021858087, -0.00125372503,
                    -0.00417768164, 0.246640727, 1.50140941], F32)
TAIL = np.array([-0.000200214257, 0.000100950558, 0.00134934322, -0.00367342844, 0.00573950773, -0.0076224613,
                 0.00943887047, 1.00167406, 2.83297682], F32)
FMA = True                                              # (J4)
NORMAL_ULP_BOUND = 3                                    # see the module docstring; asserted by the host tests


def fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: the product is exact in fp64, the fp64 sum is rounded to odd (TwoSum
    error term), and rounding that to fp32 rounds the exact sum once (53 >= 2 * 24 + 2)."""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    e = (p - (s - bp)) + (c - bp)
    fix = (e != 0) & ((s.view(np.int64) & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def log1p_f64(x):
    """log1p in fp64 rounded to fp32."""
    return np.log1p(np.asarray(x, F32).astype(np.float64)).astype(F32)


def erf_inv_w(x, log1p=log1p_f64):
    x = np.asarray(x, F32)
    return (-log1p((-(x * x)).astype(F32))).astype(F32)


def erf_inv_from_w(x, w, fma=None):
    """(J2), given w = -log1p(-x * x)."""
    fma = FMA if fma is None else fma
    x, w = np.asarray(x, F32), np.asarray(w, F32)
    lt = w < F32(5)
    with np.errstate(invalid="ignore", over="ignore"):
        t = np.where(lt, (w - F32(2.5)).astype(F32), (np.sqrt(w) - F32(3)).astype(F32)).astype(F32)
        p = np.where(lt, CENTRAL[0], TAIL[0]).astype(F32)
        for i in range(1, 9):
            c = np.where(lt, CENTRAL[i], TAIL[i]).astype(F32)
            p = fma32(p, t, c) if fma else ((p * t).astype(F32) + c).astype(F32)
        return np.where(np.abs(x) == F32(1), x * F32(np.inf), (p * x).astype(F32)).astype(F32)


def erf_inv(x, log1p=log1p_f64, fma=None):
    return erf_inv_from_w(x, erf_inv_w(x, log1p), fma)


def uniform_from_bits(bits):
    """(J1): ``uniform(key, shape, lo, 1)`` of the random bits."""
    f = ((np.asarray(bits, np.uint32) >> np.uint32(9)) | np.uint32(0x3F800000)).view(F32) - F32(1)
    return np.maximum(LO, (f * (F32(1) - LO)).astype(F32) + LO).astype(F32)


def normal_from_bits(bits, log1p=log1p_f64, fma=None):
    return (SQRT2 * erf_inv(uniform_from_bits(bits), log1p, fma)).astype(F32)


def normal(key, shape=(), partitionable=None, log1p=log1p_f64, fma=None):
    """``jax.random.normal(key, shape)`` float32, vectorised over leading key axes as ``oracle/jax_prng.py``."""
    return normal_from_bits(jr.random_bits(key, shape, partitionable), log1p, fma)


def all_bits():
    """The 2^23 distinct inputs: every value of bits >> 9."""
    return (np.arange(1 << 23, dtype=np.uint32) << np.uint32(9)).astype(np.uint32)


def ulp_distance(a, b):
    """|a - b| in fp32 ulps (the distance in the ordered integer line of the bit patterns)."""
    def ordered(v):
        i = np.asarray(v, F32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))
