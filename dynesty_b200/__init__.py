"""dynesty_b200 -- H100 (sm_90a) implementation of dynesty's bounding-and-proposal
hot path behind dynesty's own ``bound=`` / ``sample=`` / ``pool=`` plug-in surface.

Layout (only what the path needs):
  csrc/            hand-written CUDA kernels + the C ABI (include/b200nest.h)
  _lib.py, ops.py  ctypes binding / array-level wrappers (one C call each)
  likelihoods.py   device models (in-kernel prior transform + log-likelihood)
  torchmodel.py    models written as batched PyTorch functions (stepped random-walk chains)
  bounding.py      B200Ellipsoid / B200MultiEllipsoid   (mirror of dynesty.bounding.Bound)
  samplers.py      B200RWalkSampler / ...               (mirror of dynesty InternalSampler)
  pool.py          B200Pool                              (the pool= duck-type)
  nested.py        host mirror of Sampler's proposal dispatch (propose_live/_fill_queue/...)
There is no CPU fallback: without libb200nest.so + a CUDA device the ops raise.
"""
from ._lib import B200Unavailable  # noqa: F401
from .torchmodel import TorchModel  # noqa: F401

__version__ = '0.1.0'
