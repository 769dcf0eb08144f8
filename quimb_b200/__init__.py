"""quimb_b200 -- an H100-native array backend for quimb's hot path.

The module *is* the backend: arrays are :class:`quimb_b200.Array`, so
``autoray.infer_backend(x) == "quimb_b200"`` and
``autoray.do("tensordot", a, b, axes)`` resolves to
:func:`quimb_b200.tensordot`, ``do("linalg.svd", x)`` to
:func:`quimb_b200.linalg.svd`, and so on (SURVEY.md section 8b).  With quimb
installed, ``quimb_b200.register_with_quimb()`` additionally installs the
fused overrides of quimb's composed split drivers (``svd_truncated``,
``qr_stabilized``, ``fuse`` ...), exactly as quimb itself does for its numpy
backend (quimb/tensor/decomp.py:1058, :2198).

All arithmetic on the hot path runs in hand-written sm_90a CUDA kernels
behind a C ABI (``include/quimb_b200.h``); there is no CPU fallback.
"""

from . import _lib
from .array import Array
from .ops import *  # noqa: F401,F403  (the autoray-visible function surface)
from .ops import (abs, all, any, max, min, sum)  # noqa: F401,A004
from . import linalg  # noqa: F401
from .contract import (contract_batched, contract_pair, feed_pair, plan_pair,  # noqa: F401
                       route_pair, schedule_pair)
from . import dist  # noqa: F401
from .tree import (ContractExpression, GraphedContraction, Tree,  # noqa: F401
                   array_contract, find_sliced_tree, find_slices, find_tree,
                   gen_output_inds, tensor_contract)
from .mps import (ChainPlan, MovingEnvironment, compute_left_environments,  # noqa: F401
                  compute_right_environments, env_left_step, env_right_step,
                  mpo_ham_heis, mps_expec, mps_expec2, mps_norm, mps_norm2)
from .split import (array_split, array_svals, cholesky_regularized,  # noqa: F401
                    eigh_truncated, lddiv, ldmul, lu_truncated, polar_left, polar_right,
                    qr_stabilized, qr_via_cholesky, rddiv, rdmul, safe_inverse, sgn, svd_rand_truncated, svd_truncated,
                    svd_via_eig, svd_via_eig_truncated, tensor_canonize_bond,
                    tensor_compress_bond, tensor_split)
from .lanczos import eigh_lanczos  # noqa: F401
from . import boundary, linop, tebd, treeopt  # noqa: F401
from .linop import TNLinearOperator  # noqa: F401
from .tebd import (TEBD, LocalHam1D, gate_split, gate_with_auto_swap,  # noqa: F401
                   mps_sample, mps_sample_configuration)
from .boundary import (BoundaryContractor2D, contract_boundary,  # noqa: F401
                       contract_boundary_two_sided, peps_norm_tensors)
from .dmrg import DMRG1, DMRG2  # noqa: F401
from .dmrgx import DMRGX  # noqa: F401
from . import peps_expec  # noqa: F401
from .peps_expec import (calc_plaquette_map, calc_plaquette_sizes,  # noqa: F401
                         peps_compute_local_expectation, peps_normalize, plaquette_to_sites)
from . import observables  # noqa: F401
from .observables import (mps_calc_current_orthog_center, mps_canonicalize,  # noqa: F401
                          mps_compute_local_expectation, mps_correlation,
                          mps_count_canonized, mps_entropy,
                          mps_local_expectation_canonical, mps_magnetization,
                          mps_partial_trace_to_dense_canonical, mps_schmidt_gap,
                          mps_schmidt_values, mps_singular_values)
from . import mpo_compress  # noqa: F401
from .mpo_compress import mps_gate_with_mpo  # noqa: F401
from . import fit  # noqa: F401
from .fit import mps_fit, mps_gate_with_mpo_fit  # noqa: F401
from . import successive  # noqa: F401
from .successive import mps_gate_with_mpo_successive  # noqa: F401
from . import nonlocal_gates  # noqa: F401
from .nonlocal_gates import (mpo_from_dense, mps_gate_controlled,  # noqa: F401
                             mps_gate_nonlocal, mps_gate_with_submpo)
from .compressed import contract_compressed, path_to_sequence  # noqa: F401
from .integration import register_with_quimb  # noqa: F401



class _Namespace:
    """attribute bag so that dotted autoray names resolve
    (``do("scipy.linalg.solve_triangular", like="quimb_b200")``)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _random_array(shape, dist="normal", dtype="float64", rng=None, seed=None,
                  loc=0.0, scale=1.0, **kwargs):
    """``xp.random.array`` as quimb's builders call it (tensor_builder.py:4129,
    tn1d/compress.py:1283): values drawn on the host from a numpy Generator
    (``rng`` / ``seed``: reproducible, same stream as the numpy backend) and
    placed on the device."""
    return asarray(_random_host(shape, dist, dtype, rng, seed, loc, scale))  # noqa: F405


def _random_host(shape, dist="normal", dtype="float64", rng=None, seed=None, loc=0.0,
                scale=1.0):
    """The host draw of ``random.array``: a numpy array, not yet uploaded."""
    import numpy as _np
    if rng is None:
        if seed is None:
            # follow numpy's global state like the numpy backend does, so that
            # ``np.random.seed(...)`` makes quimb's randomized drivers repeatable
            seed = int(_np.random.randint(0, 2 ** 31 - 1))
        rng = _np.random.default_rng(seed)
    elif hasattr(rng, "_rng"):
        rng = rng._rng                      # a _DeviceGenerator from random.default_rng
    elif not isinstance(rng, _np.random.Generator):
        rng = _np.random.default_rng(rng)
    if isinstance(shape, int):
        shape = (shape,)
    dt = _np.dtype(dtype)

    def draw():
        if dist == "normal":
            return rng.standard_normal(shape)
        if dist == "uniform":
            return rng.uniform(-1.0, 1.0, size=shape)
        if dist == "rademacher":
            return rng.choice([-1.0, 1.0], size=shape)
        if dist == "exp":
            return rng.exponential(size=shape)
        raise ValueError(f"unknown distribution {dist!r}")
    x = draw()
    if dt.kind == "c":
        x = (x + 1j * draw()) / 2 ** 0.5 if dist != "rademacher" else x + 0j
    x = x * scale + loc
    return _np.asarray(x, dtype=dt)


class _DeviceGenerator:
    """``xp.random.default_rng(seed)`` as quimb's randomized drivers use it
    (decomp.py:1796-1824, tn1d/compress.py:1768): a numpy Generator whose
    draws are placed on the device."""

    def __init__(self, seed=None):
        import numpy as _np
        if isinstance(seed, _np.random.Generator):
            self._rng = seed
        else:
            if seed is None:
                seed = int(_np.random.randint(0, 2 ** 31 - 1))
            self._rng = _np.random.default_rng(seed)

    def normal(self, loc=0.0, scale=1.0, size=None, dtype="float64"):
        return _random_array(() if size is None else size, "normal", dtype, rng=self._rng,
                             loc=loc, scale=scale)

    def standard_normal(self, size=None, dtype="float64"):
        return self.normal(size=size, dtype=dtype)

    def uniform(self, low=0.0, high=1.0, size=None, dtype="float64"):
        return _random_array(() if size is None else size, "uniform", dtype, rng=self._rng,
                             loc=(low + high) / 2, scale=(high - low) / 2)

    def random(self, size=None, dtype="float64"):
        return self.uniform(0.0, 1.0, size, dtype)

    def integers(self, *args, **kwargs):
        return self._rng.integers(*args, **kwargs)

    def choice(self, *args, **kwargs):
        return self._rng.choice(*args, **kwargs)


random = _Namespace(
    default_rng=_DeviceGenerator,
    array=_random_array,
    normal=lambda loc=0.0, scale=1.0, size=(), dtype="float64", **kw: _random_array(
        size, "normal", dtype, loc=loc, scale=scale, **kw),
    uniform=lambda low=0.0, high=1.0, size=(), dtype="float64", **kw: _random_array(
        size, "uniform", dtype, loc=(low + high) / 2, scale=(high - low) / 2, **kw),
)

scipy = _Namespace(linalg=_Namespace(solve_triangular=linalg.solve_triangular,
                                     expm=linalg.expm, lu=linalg.lu))

__version__ = "0.1.0"


def launch_count():
    """Number of CUDA kernels this library has launched in this process."""
    return _lib.launch_count()
