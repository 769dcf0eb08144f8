"""ORACLE (test infrastructure, never imported by the product package).

Plain-numpy, batched restatement of MPS sampling,

  MatrixProductState.sample / sample_configuration   quimb/tensor/tn1d/core.py:3871-3990

Sites are (l, p, r) numpy arrays.  The reference draws one
``rng.choice(d, p=p)`` per site and sample, and each such call consumes
exactly one ``rng.random()`` double and returns
``searchsorted(cumsum(p) / cumsum(p)[-1], u, side='right')``.  So the
reference's draws are the doubles of ``rng.random((C, L))`` in row-major
order, and this restatement (all samples at once, host uniforms, the
selected row renormalised at each site) reproduces its configurations
sample for sample, except for a uniform within rounding of a cdf boundary:
``margin`` (the least |u - cdf[s]| over every draw and every s) says how far
from that the run was.  Pinned against the reference itself by
oracle/make_golden_sample.py (tests/golden/sample.*).
"""

import numpy as np

from . import tebd_np


def prepare(sites):
    """Right-canonical copy (centre at site 0) with the centre at unit norm."""
    psi = [np.array(a, dtype=np.result_type(a.dtype, np.float64)) for a in sites]
    cplx = any(np.iscomplexobj(a) for a in psi)
    if cplx:
        psi = [a.astype(np.complex128) for a in psi]
    tebd_np.canonicalize(psi, 0)
    psi[0] = psi[0] / np.linalg.norm(psi[0])
    return psi


def sample_uniforms(psi, u):
    """Configurations (C, L), probabilities (C,) and the margin for the
    uniforms ``u`` (C, L) of a prepared MPS ``psi``."""
    C, L = u.shape
    V = np.ones((C, 1), dtype=psi[0].dtype)
    configs = np.empty((C, L), dtype=np.int64)
    omegas = np.ones(C)
    margin = np.inf
    for i, A in enumerate(psi):
        l, d, r = A.shape
        W = (V @ A.reshape(l, d * r)).reshape(C, d, r)
        pi = np.sum(np.abs(W) ** 2, axis=2)
        p = pi / pi.sum(axis=1, keepdims=True)
        cdf = np.cumsum(p, axis=1)
        cdf /= cdf[:, -1:]
        x = np.sum(cdf <= u[:, i:i + 1], axis=1)
        margin = min(margin, float(np.min(np.abs(cdf - u[:, i:i + 1]))))
        rows = np.arange(C)
        configs[:, i] = x
        omegas *= p[rows, x]
        V = W[rows, x, :] / np.sqrt(pi[rows, x])[:, None]
    return configs, omegas, margin


def sample(sites, C, seed=None):
    """``(configs, omegas, margin)`` of ``C`` samples; ``seed`` as
    ``np.random.default_rng`` takes it (a Generator is advanced by C * L
    doubles)."""
    rng = np.random.default_rng(seed)
    psi = prepare(sites)
    u = rng.random((C, len(psi)))
    return sample_uniforms(psi, u)
