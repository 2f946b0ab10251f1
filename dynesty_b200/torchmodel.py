"""Models written as batched PyTorch functions.

A ``TorchModel`` goes where a ``DeviceModel`` goes (``NestedSampler(model, ...)``, ``DynamicNestedSampler(model,
...)``) when the likelihood is easier to write in PyTorch than as a warp-cooperative CUDA device function: a linear
solve, an FFT, an interpolation table, a neural emulator.  The random-walk chains then run as one launch of the
stepped kernel per step (csrc/b2n_rwalk_step.cu), with the two callables between the launches on the same stream:

    prior_transform(u: (B, n) float64 CUDA tensor) -> (B, n)
    loglike(v: (B, n) float64 CUDA tensor)         -> (B,)

Row i of an output may depend on row i of the input only; B changes from call to call (the queue size, the round
size, the initial draws).  The first call for a given B checks each output's shape, dtype and device once; after that
no host-side check runs, so that a fill never waits for the GPU.  A NaN log-likelihood rejects the proposal, as in the
in-kernel chains and in dynesty (``logl > loglstar`` is false).

Only the random walk is stepped: ``sample='auto'`` resolves to ``'rwalk'``; the slice and uniform samplers, whose
number of evaluations per chain depends on the data, refuse a ``TorchModel``.  The live points are drawn on the host
(``live_init='host'``) and evaluated in one batched call, and ``run_nested(loop='device')`` runs the phase before the
first bound in the host loop.
"""
import numpy as np

from . import _lib


class TorchModel:
    """A prior transform and a log-likelihood as batched torch functions of (B, ndim) float64 tensors on the
    context's device.  ``evaluate`` / ``prior_transform`` / ``loglikelihood`` are the numpy-level callables a
    ``DeviceModel`` has."""

    def __init__(self, ndim, loglike, prior_transform, name='torch'):
        if not callable(loglike) or not callable(prior_transform):
            raise TypeError('TorchModel needs callable loglike and prior_transform')
        self.ndim = int(ndim)
        if self.ndim < 1:
            raise ValueError('ndim must be >= 1')
        self.loglike = loglike
        self.prior_transform_fn = prior_transform
        self.name = name
        self.nblob = 0
        self._checked = set()       # (callable, batch size) pairs whose output has been checked

    @staticmethod
    def model_id(ctx=None):
        """-1: no in-kernel model.  The in-kernel chain entry points refuse it; the stepped ones need none."""
        return -1

    @staticmethod
    def device(ctx=None):
        import torch
        ctx = ctx if ctx is not None else _lib.default_context()
        return torch.device('cuda', ctx.device)

    def _check(self, fn, out, shape, device):
        import torch
        key = (fn, shape[0])
        if key in self._checked:
            return
        what = '%s of TorchModel %r' % (getattr(fn, '__name__', repr(fn)), self.name)
        if not isinstance(out, torch.Tensor):
            raise ValueError('%s returned %s, not a torch.Tensor' % (what, type(out).__name__))
        if tuple(out.shape) != shape:
            raise ValueError('%s returned shape %s for a batch of %d rows; expected %s'
                             % (what, tuple(out.shape), shape[0], shape))
        if out.dtype != torch.float64:
            raise ValueError('%s returned dtype %s; expected torch.float64' % (what, out.dtype))
        if out.device != device:
            raise ValueError('%s returned a tensor on %s; expected %s' % (what, out.device, device))
        self._checked.add(key)

    def _eval(self, u):
        """(v, logl) of the (B, ndim) float64 tensor u, contiguous, on the current stream."""
        B = u.shape[0]
        v = self.prior_transform_fn(u)
        self._check(self.prior_transform_fn, v, (B, self.ndim), u.device)
        logl = self.loglike(v)
        self._check(self.loglike, logl, (B,), u.device)
        return v.contiguous(), logl.contiguous()

    # -- host callables (numpy in, numpy out) -------------------------------------
    def evaluate(self, u, ctx=None):
        """(v, logl) of unit-cube points u (M, ndim), numpy arrays."""
        import torch
        u = np.ascontiguousarray(np.atleast_2d(u), dtype=np.float64)
        v, logl = self._eval(torch.as_tensor(u, device=self.device(ctx)))
        return v.cpu().numpy(), logl.cpu().numpy()

    def prior_transform(self, u):
        u = np.asarray(u, dtype=float)
        v, _ = self.evaluate(u.reshape(-1, self.ndim))
        return v.reshape(u.shape)

    def loglikelihood(self, v):
        import torch
        v = np.asarray(v, dtype=float)
        vt = torch.as_tensor(np.ascontiguousarray(v.reshape(-1, self.ndim)), device=self.device())
        logl = self.loglike(vt)
        self._check(self.loglike, logl, (vt.shape[0],), vt.device)
        logl = logl.cpu().numpy()
        return float(logl[0]) if v.ndim == 1 else logl
