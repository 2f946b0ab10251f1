"""Device models: the prior-transform / log-likelihood pairs the proposal kernels
can evaluate in-kernel ("device-side likelihood callback").

The reference accepts arbitrary Python callables (dynesty.py:584-614) and calls
them once per proposal on the host.  Here a model is a descriptor from a closed
registry (include/b200nest.h, ``b2n_model_desc``) whose parameters live in HBM.
A ``DeviceModel`` is ALSO a pair of host callables (``prior_transform`` /
``loglikelihood``), evaluated on the GPU through ``b2n_model_eval`` -- so the
same object can be handed to dynesty's own ``NestedSampler`` as
``loglikelihood=model.loglikelihood, prior_transform=model.prior_transform``
(unit-cube warm-up phase, initial live points) while the B200 samplers pick up
the descriptor for the in-kernel evaluation.

``DeviceModel.from_cuda`` opens the registry: the log-likelihood, and optionally the prior transform, is then user
CUDA code compiled into the same kernels at run time (NVRTC, ``usermodel.py``).
"""
import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import ModelDesc, ptr, f64


class DeviceModel:
    def __init__(self, ndim, prior_kind, like_kind, prior_p0=None, prior_p1=None, like_vec0=None,
                 like_vec1=None, like_mat=None, s0=0.0, s1=0.0, s2=0.0, name='model'):
        self.ndim = int(ndim)
        self.name = name
        self.prior_kind, self.like_kind = int(prior_kind), int(like_kind)
        opt = lambda a, shape: None if a is None else f64(np.broadcast_to(a, shape))
        n = self.ndim
        self.prior_p0, self.prior_p1 = opt(prior_p0, (n,)), opt(prior_p1, (n,))
        self.like_vec0, self.like_vec1 = opt(like_vec0, (n,)), opt(like_vec1, (n,))
        self.like_mat = opt(like_mat, (n, n))
        self.s = (float(s0), float(s1), float(s2))
        self.nblob = 0          # doubles of derived quantities per point (from_cuda(nblob=)); registry models have none
        self._ids = {}          # ctx -> (full id, likelihood-only id)

    # -- pickling: device handles are per-process, re-created lazily ------------
    def __getstate__(self):
        d = self.__dict__.copy()
        d['_ids'] = {}
        return d

    def _desc(self, prior_kind):
        d = ModelDesc()
        d.ndim, d.prior_kind, d.like_kind = self.ndim, prior_kind, self.like_kind
        d.prior_p0, d.prior_p1 = ptr(self.prior_p0), ptr(self.prior_p1)
        d.like_vec0, d.like_vec1, d.like_mat = ptr(self.like_vec0), ptr(self.like_vec1), ptr(self.like_mat)
        d.like_s0, d.like_s1, d.like_s2 = self.s
        return d

    @classmethod
    def from_cuda(cls, ndim, source, params=None, prior_kind=_lib.PRIOR_IDENTITY, prior_p0=None, prior_p1=None,
                  prior_source=None, prior_params=None, name='user', nblob=0):
        """A model whose log-likelihood (and optionally prior transform) is user CUDA code, compiled into the
        proposal kernels at run time.

        ``source`` defines ONE warp-cooperative device function::

            __device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane);

        * all 32 lanes of a warp call it (``lane`` = 0..31) and it must return the same value on every lane;
        * ``v``: the prior-transformed point, ``n`` = ndim doubles in warp-private shared memory (read only);
        * ``work``: ``n`` doubles of warp-private shared scratch;
        * ``p``: ``params`` (float64) in device memory, or NULL when ``params`` is None;
        * ``b2n_warp_sum`` / ``b2n_warp_prod`` / ``b2n_warp_max`` / ``b2n_warp_min`` reduce over the warp.

        A sum over dimensions is split over the lanes and reduced::

            __device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
                double s = 0.0;
                for (int i = lane; i < n; i += 32) s += (v[i] - p[i]) * (v[i] - p[i]);
                return -0.5 * b2n_warp_sum(s);
            }

        A scalar formula is computed by lane 0 and broadcast::

            __device__ double b2n_user_loglike(const double* v, double* work, int n, const double* p, int lane) {
                double l = 0.0;
                if (lane == 0) l = -0.5 * (v[0] * v[0] + 100.0 * (v[1] - v[0] * v[0]) * (v[1] - v[0] * v[0]));
                return __shfl_sync(0xffffffffu, l, 0);
            }

        The prior is one of the registry's (``prior_kind`` with per-dimension ``prior_p0`` / ``prior_p1``), or
        user code: ``prior_source`` defines a second warp-cooperative device function (the prior is then
        ``PRIOR_USER``)::

            __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane);

        * all 32 lanes call it; it writes ``v[0, n)`` from ``u[0, n)`` and may read ANY component of ``u``, so
          joint transforms (correlated Gaussians, ordered parameters, simplex weights) are allowed;
        * ``u``: read only (warp-private shared memory in the chain kernels, global memory in ``evaluate``);
        * ``v``, ``work``: ``n`` doubles each of warp-private shared memory; ``work`` is undefined on entry;
        * ``p``: ``prior_params`` (float64) in device memory, or NULL when ``prior_params`` is None;
        * the caller synchronises the warp before and after the call; inside it, ``__syncwarp()`` between one lane
          writing ``work`` and another reading it.  The ``b2n_warp_*`` reductions are available;
        * it must be deterministic (the same ``u`` gives the same bits of ``v``).  Only proposals inside the unit
          cube are transformed.

        Per dimension -- log-uniform on ``[p[i], p[n + i]]``::

            __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
                for (int i = lane; i < n; i += 32) v[i] = p[i] * exp(u[i] * log(p[n + i] / p[i]));
            }

        Joint -- a correlated Gaussian ``mu + L ndtri(u)`` (``mu`` = ``p[0, n)``, lower-triangular ``L``
        column-major at ``p + n``), with ``ndtri(u)`` staged in ``work``::

            __device__ void b2n_user_prior(const double* u, double* v, double* work, int n, const double* p, int lane) {
                for (int i = lane; i < n; i += 32) work[i] = normcdfinv(u[i]);
                __syncwarp();
                for (int i = lane; i < n; i += 32) {
                    double s = p[i];
                    for (int j = 0; j <= i; j++) s = fma(p[n + (size_t)j * n + i], work[j], s);
                    v[i] = s;
                }
            }

        ``prior_source`` excludes ``prior_kind`` / ``prior_p0`` / ``prior_p1``, and ``prior_params`` needs
        ``prior_source`` (``ValueError`` otherwise).  ``loglikelihood(v)`` stays prior-free.

        With ``nblob > 0`` the model has a blob: ``nblob`` derived quantities per point, which the samplers save with
        every sample (``NestedSampler(..., blob=True)``, ``results['blob']``).  ``source`` then also defines a third
        warp-cooperative device function::

            __device__ void b2n_user_blob(const double* v, double* work, int n, const double* p, int lane,
                                          double* blob, int nblob);

        * all 32 lanes call it; ``v`` (read only), ``work``, ``n``, ``p`` and ``lane`` are those of
          ``b2n_user_loglike``, which it may call (a blob may hold the log-likelihood or its parts);
        * ``blob``: ``nblob`` doubles of warp-private shared memory, NaN on entry; what it writes there is the point's
          row of the blob, and an element it leaves unwritten stays NaN;
        * the caller synchronises the warp before and after the call; inside it, ``__syncwarp()`` between one lane
          writing ``work`` or ``blob`` and another reading it;
        * it must be deterministic: the blob of a saved sample is computed from its ``v`` after the run, in one launch
          (``blob(v)``), not carried through the chains.

        A source without ``b2n_user_blob`` raises ``usermodel.UserModelCompileError`` naming it when the model is first
        used.  ``blob(v)`` evaluates the blob of any points.

        The model is accepted wherever a registry model is: every sampler, the device-resident rounds, the dynamic
        sampler, replicas; random walks run on the warp-per-chain kernel.  The source is compiled with NVRTC for
        sm_90a (once per process, ``usermodel.compile_user``); a compile error raises
        ``usermodel.UserModelCompileError`` carrying NVRTC's log.  Pickling keeps ``source``, ``params``,
        ``prior_source``, ``prior_params`` and ``nblob``.
        """
        if isinstance(nblob, bool) or int(nblob) != nblob or nblob < 0:
            raise ValueError('nblob must be a non-negative integer')
        if prior_source is not None:
            if prior_kind not in (_lib.PRIOR_IDENTITY, _lib.PRIOR_USER) or prior_p0 is not None or prior_p1 is not None:
                raise ValueError('prior_source defines the prior: prior_kind / prior_p0 / prior_p1 do not apply')
            prior_kind = _lib.PRIOR_USER
        elif prior_params is not None:
            raise ValueError('prior_params are the parameters of a user prior: give prior_source as well')
        elif prior_kind == _lib.PRIOR_USER:
            raise ValueError('prior_kind PRIOR_USER needs prior_source')
        m = cls(ndim, prior_kind, _lib.LIKE_USER, prior_p0=prior_p0, prior_p1=prior_p1, name=name)
        m.source = str(source)
        m.params = None if params is None else f64(np.ravel(params))
        m.prior_source = None if prior_source is None else str(prior_source)
        m.prior_params = None if prior_params is None else f64(np.ravel(prior_params))
        m.nblob = int(nblob)
        m.logz_truth = None
        return m

    def ids(self, ctx=None):
        ctx = ctx if ctx is not None else _lib.default_context()
        key = ctx.serial           # (not id(ctx): an address can be reused after a Context is freed)
        if key not in self._ids:
            out = []
            for pk in (self.prior_kind, _lib.PRIOR_IDENTITY):
                mid = C.c_int32(-1)
                if self.like_kind == _lib.LIKE_USER:
                    self._create_user(ctx, pk, mid)
                else:
                    ctx.check(ctx.lib.b2n_model_create(ctx.h, C.byref(self._desc(pk)), C.byref(mid)))
                out.append(mid.value)
            self._ids[key] = tuple(out)
        return self._ids[key]

    def _create_user(self, ctx, prior_kind, mid):
        from . import usermodel
        prior_source = getattr(self, 'prior_source', None)
        cm = usermodel.compile_user(self.source, prior_source, blob=getattr(self, 'nblob', 0) > 0)
        names = (C.c_char_p * len(cm.lowered))(*[s.encode() for s in cm.lowered])
        prm = self.params
        nprm = 0 if prm is None else prm.size
        if prior_source is None:
            ctx.check(ctx.lib.b2n_model_create_user(ctx.h, C.byref(self._desc(prior_kind)), ptr(prm), nprm,
                                                    cm.cubin, len(cm.cubin), names, C.byref(mid)))
            return
        # the user prior and the likelihood-only (identity prior) model share the one image
        pp = self.prior_params if prior_kind == _lib.PRIOR_USER else None
        ctx.check(ctx.lib.b2n_model_create_user_ex(ctx.h, C.byref(self._desc(prior_kind)), ptr(prm), nprm, ptr(pp),
                                                   0 if pp is None else pp.size, cm.cubin, len(cm.cubin), names,
                                                   C.byref(mid)))

    def model_id(self, ctx=None):
        return self.ids(ctx)[0]

    # -- host callables (GPU-evaluated) ------------------------------------------
    def evaluate(self, u, ctx=None):
        """(v, logl) of unit-cube points u (M, ndim) in one launch."""
        from . import ops
        return ops.model_eval(self.ids(ctx)[0], u, ctx=ctx)

    def blob(self, v, ctx=None):
        """The blob (M, nblob) of the physical points v (M, ndim) in one launch (``b2n_model_blob``)."""
        from . import ops
        if getattr(self, 'nblob', 0) < 1:
            raise ValueError('the model %r has no blob: DeviceModel.from_cuda(..., nblob=k) with a source that '
                             'defines b2n_user_blob' % self.name)
        v = np.asarray(v, dtype=float).reshape(-1, self.ndim)
        return ops.model_blob(self.ids(ctx)[0], v, self.nblob, ctx=ctx)

    def prior_transform(self, u):
        from . import ops
        u = np.asarray(u, dtype=float)
        v, _ = ops.model_eval(self.ids()[0], u.reshape(-1, self.ndim))
        return v.reshape(u.shape)

    def loglikelihood(self, v):
        from . import ops
        v = np.asarray(v, dtype=float)
        _, l = ops.model_eval(self.ids()[1], v.reshape(-1, self.ndim), want_v=False)
        return float(l[0]) if v.ndim == 1 else l


# ---- the BASELINE.json problem families -------------------------------------------
def gauss_corr(ndim, rho=0.4, halfwidth=5.0):
    """C2: correlated normal, prior U(-h, h)^n (demos/Examples -- 25-D Correlated Normal.ipynb)."""
    Cm = np.full((ndim, ndim), float(rho))
    np.fill_diagonal(Cm, 1.0)
    prec = np.linalg.inv(Cm)
    lnorm = -0.5 * (math.log(2 * math.pi) * ndim + np.linalg.slogdet(Cm)[1])
    m = DeviceModel(ndim, _lib.PRIOR_UNIFORM, _lib.LIKE_GAUSS_PREC, prior_p0=-halfwidth,
                    prior_p1=2 * halfwidth, like_vec0=0.0, like_mat=prec, s0=lnorm,
                    name='gauss_corr%d' % ndim)
    m.logz_truth = -ndim * math.log(2 * halfwidth)
    return m


def gauss_test3d():
    """C1: tests/test_gau.py:67-102."""
    n = 3
    Cm = np.full((n, n), 0.95)
    np.fill_diagonal(Cm, 1.0)
    lnorm = -0.5 * (math.log(2 * math.pi) * n + np.linalg.slogdet(Cm)[1])
    m = DeviceModel(n, _lib.PRIOR_UNIFORM, _lib.LIKE_GAUSS_PREC, prior_p0=-10., prior_p1=20.,
                    like_vec0=np.linspace(-1, 1, n), like_mat=np.linalg.inv(Cm), s0=lnorm,
                    name='gauss_test3d')
    m.logz_truth = n * (-math.log(20.))
    return m


def iid_normal_ppf(ndim):
    """C4: iid N(0,1) likelihood with a standard-normal ppf prior
    (demos/Examples -- 200-D Multivariate Normal.ipynb)."""
    lnorm = -0.5 * math.log(2 * math.pi) * ndim
    m = DeviceModel(ndim, _lib.PRIOR_NORMAL_PPF, _lib.LIKE_GAUSS_DIAG, prior_p0=0., prior_p1=1.,
                    like_vec0=0., like_vec1=1., s0=lnorm, name='iid_normal%d' % ndim)
    m.logz_truth = lnorm - 0.5 * ndim * math.log(2)
    return m


def eggbox(ndim, tmax=5.0 * math.pi, power=5.0):
    """C3: demos/Examples -- Eggbox.ipynb generalised to ndim."""
    m = DeviceModel(ndim, _lib.PRIOR_IDENTITY, _lib.LIKE_EGGBOX, s0=tmax, s1=power,
                    name='eggbox%d' % ndim)
    m.logz_truth = 235.856 if ndim == 2 else None      # tests/test_egg.py:29-46
    return m


def shells(ndim, r=2.0, w=0.1, c=3.5, halfwidth=6.0):
    """C5: demos/Examples -- Gaussian Shells.ipynb."""
    c1 = np.zeros(ndim)
    c1[0] = -c
    c2 = np.zeros(ndim)
    c2[0] = c
    m = DeviceModel(ndim, _lib.PRIOR_UNIFORM, _lib.LIKE_SHELLS, prior_p0=-halfwidth,
                    prior_p1=2 * halfwidth, like_vec0=c1, like_vec1=c2, s0=r, s1=w,
                    name='shells%d' % ndim)
    m.logz_truth = {2: -1.75, 5: -5.67, 10: -14.59}.get(ndim)
    return m


def region2d(shape='diamond', ndim=2):
    """The hard-edged regions of the reference's sampler-uniformity harness (tests/test_sampling.py:8-23):
    ``diamond_logl`` / ``checker_logl`` on the first two coordinates, identity prior, the remaining
    dimensions free.  Used with loglstar = 0: the samplers must leave the uniform distribution on
    {logl > 0} invariant."""
    m = DeviceModel(ndim, _lib.PRIOR_IDENTITY, _lib.LIKE_REGION2D, s0={'diamond': 0.0, 'checkerboard': 1.0}[shape],
                    name='region2d_%s%d' % (shape, ndim))
    m.logz_truth = None
    return m
