"""B200 inner samplers: drop-in mirrors of dynesty's ``RWalkSampler`` / ``RSliceSampler`` /
``SliceSampler`` / ``UniformBoundSampler`` (internal_samplers.py:206-863).

The reference maps a *static* ``sample(args)`` over the queue, one task per chain
(sampler.py:708-717).  Here ``prepare_sampler`` -- which the reference calls once with ALL
queue slots -- launches ONE kernel for the whole queue and returns the finished
``SamplerReturn`` tuples as the "arguments"; the static ``sample`` is then the identity,
so ``mapper(self.internal_sampler.sample, args)`` (sampler.py:717) works unchanged with
any mapper (``map``, ``B200Pool.map``, a real pool).

The likelihood is evaluated in-kernel, so each sampler is constructed with a
``DeviceModel`` (``model=``); dynesty's ``_new_from_template`` re-instantiates with the
same kwargs (internal_samplers.py:96-109), so the model travels with it.
"""
import math
import warnings

import numpy as np

from . import ops, _lib
from ._compat import InternalSamplerBase, SamplerReturn
from .bounding import TaggedAxes
from .torchmodel import TorchModel

__all__ = ['B200RWalkSampler', 'B200RSliceSampler', 'B200SliceSampler', 'B200UniformSampler']


# The queue's ``SamplerReturn`` list (one per slot; what Sampler._fill_queue maps ``sample`` over) is built positionally
# through ``tuple.__new__`` when the field order is the one written here (dynesty's own and the mirror's): building 2000
# namedtuples by keyword was 4 ms of a 6.6 ms plug-in fill at C2, this way it is 2 ms.
_SR_FAST = SamplerReturn._fields == ('u', 'v', 'logl', 'ncalls', 'evaluation_history', 'tuning_info', 'proposal_stats')
_new_tuple = tuple.__new__


def _seed_of(seeds, fallback_rstate=None):
    """One 64-bit Philox seed per queue fill from what Sampler passes as `seeds`
    (SeedSequence children when queue_size > 1, else the master Generator itself,
    sampler.py:695-699)."""
    s = seeds[0]
    if isinstance(s, np.random.Generator):
        return int(s.integers(0, 2**63 - 1))
    if isinstance(s, np.random.SeedSequence):
        w = s.generate_state(2, dtype=np.uint32)
        return (int(w[0]) | (int(w[1]) << 32)) & (2**63 - 1)
    return int(s) & (2**63 - 1)


def _announce(axes, nested_sampler, u):
    """The end points of a queue are the live points -- hence the ``bound.contains`` queries of
    Sampler.propose_live (sampler.py:485) -- of the near future: evaluate their membership in one launch."""
    b = getattr(nested_sampler, 'bound', None)
    if b is None and len(axes) and isinstance(axes[0], TaggedAxes):
        b = axes[0].bound
    if b is not None and hasattr(b, 'prefetch_contains'):
        b.prefetch_contains(u)


class _Resident:
    """Keeps the device copy of the current bound's ellipsoids in sync.  Which bound is resident is
    recorded ONCE per context (``Context.resident_key``, set by ``ops.bound_set``), not per sampler:
    anything else that uploads a bound to the same ctx invalidates it for everybody."""

    def ensure(self, axes_list, ctx):
        """Returns the int32 ellipsoid index of every chain."""
        a0 = axes_list[0]
        if isinstance(a0, TaggedAxes) and a0.bound is not None and hasattr(a0.bound, 'make_resident'):
            b = a0.bound
            c = ctx if ctx is not None else b.ctx
            if c.resident_key is None or c.resident_key != b.version:
                b.make_resident(c)
            return np.fromiter((a.ell for a in axes_list), dtype=np.int32, count=len(axes_list))
        # foreign Bound (e.g. the reference's own classes or a user Box bound,
        # tests/test_bound_interface.py:20-49): upload the distinct matrices of this fill
        uniq, ell = {}, np.empty(len(axes_list), dtype=np.int32)
        mats = []
        for i, a in enumerate(axes_list):
            k = id(a)
            if k not in uniq:
                uniq[k] = len(mats)
                mats.append(np.asarray(a, dtype=float))
            ell[i] = uniq[k]
        ops.bound_set(np.array(mats), ctx=ctx)          # anonymous upload: resident_key = None
        return ell


class _B200Sampler(InternalSamplerBase):
    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.model = kwargs.get('model')
        if self.model is None:
            raise ValueError("B200 samplers evaluate the likelihood in-kernel: pass model=<DeviceModel>")
        self._ctx = kwargs.get('ctx')
        self.ncdim = kwargs.get('ncdim')
        self._res = _Resident()
        self.chain_counter = 0
        self.last_batch = None

    def __getstate__(self):
        d = self.__dict__.copy()
        d['_ctx'] = None
        d['_res'] = _Resident()
        d['last_batch'] = None
        if 'input_kwargs' in d:
            d['input_kwargs'] = {k: v for k, v in d['input_kwargs'].items() if k != 'ctx'}
        return d

    def _flags(self):
        per, ref = self.sampler_kwargs.get('periodic'), self.sampler_kwargs.get('reflective')
        return ops.dimflags_from(self.ndim or self.model.ndim, per, ref)

    @staticmethod
    def sample(args):
        """The chain already ran inside ``prepare_sampler``'s launch."""
        return args


class B200RWalkSampler(_B200Sampler):
    """internal_samplers.py:444-565."""

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        walks = max(2, kwargs.get('walks', 25) or 25)
        self.facc = min(1., max(1. / walks, kwargs.get('facc', 0.5) or 0.5))
        self.rwalk_history = {'n_accept': 0, 'n_reject': 0}
        self.sampler_kwargs['walks'] = walks
        self.sampler_kwargs['ncdim'] = self.ncdim

    @property
    def update_bound_interval_ratio(self):
        return self.sampler_kwargs['walks']

    def run_batch(self, loglstar, points, ell, seed, chain0=0, peer=None):
        walks = self.sampler_kwargs['walks']
        if isinstance(self.model, TorchModel):       # the likelihood runs between the launches of the stepped walk
            if peer is not None:
                raise NotImplementedError("a TorchModel's chains run on one GPU")
            return ops.rwalk_stepped(self.model, points, loglstar, self.scale, walks, seed, chain0=chain0, ell=ell,
                                     dimflags=self._flags(), ncdim=self.ncdim or self.model.ndim, ctx=self._ctx)
        return ops.rwalk_batch(self.model.model_id(self._ctx), points, loglstar, self.scale, walks, seed,
                               chain0=chain0, ncdim=self.ncdim or self.model.ndim, ell=ell,
                               dimflags=self._flags(), ctx=self._ctx, peer=peer)

    def prepare_sampler(self, loglstar=None, points=None, axes=None, seeds=None, prior_transform=None,
                        loglikelihood=None, nested_sampler=None):
        ell = self._res.ensure(axes, self._ctx)
        o = self.run_batch(loglstar, np.asarray(points), ell, _seed_of(seeds))
        self.last_batch = o
        _announce(axes, nested_sampler, o['u'])
        sc = self.scale
        # (one .tolist() per array instead of a numpy scalar conversion per field: the list is built once per
        # queue fill and its cost, not the kernel's, is what dynesty sees per fill)
        ll, nc = o['logl'].tolist(), o['ncall'].tolist()
        na, nr = o['n_accept'].tolist(), o['n_reject'].tolist()
        SR = SamplerReturn
        if _SR_FAST:
            return [_new_tuple(SR, (u, v, l, c, [], {'accept': a, 'reject': r, 'scale': sc}, {'n_accept': a, 'n_reject': r}))
                    for u, v, l, c, a, r in zip(list(o['u']), list(o['v']), ll, nc, na, nr)]
        return [SR(u=u, v=v, logl=l, ncalls=c, evaluation_history=[],
                   tuning_info={'accept': a, 'reject': r, 'scale': sc},
                   proposal_stats={'n_accept': a, 'n_reject': r})
                for u, v, l, c, a, r in zip(o['u'], o['v'], ll, nc, na, nr)]

    def tune(self, tuning_info, update=True):
        """internal_samplers.py:460-493."""
        self.scale = tuning_info['scale']
        h = self.rwalk_history
        h['n_accept'] += tuning_info['accept']
        h['n_reject'] += tuning_info['reject']
        if not update:
            return
        facc = h['n_accept'] / (h['n_accept'] + h['n_reject'])
        self.scale *= math.exp((facc - self.facc) / self.ncdim / self.facc)
        h['n_accept'] = h['n_reject'] = 0

    @property
    def citations(self):
        return [("Skilling (2006)", "projecteuclid.org/euclid.ba/1340370944")]


class _B200SliceBase(_B200Sampler):
    _fn = None

    def __init__(self, **kwargs):
        super().__init__(**kwargs)
        self.sampler_kwargs['slices'] = kwargs.get('slices', 5) or 5
        self.slice_history = {'n_contract': 0, 'n_expand': 0}

    def run_batch(self, loglstar, points, ell, seed, chain0=0, peer=None):
        fn = getattr(ops, self._fn)
        return fn(self.model.model_id(self._ctx), points, loglstar, self.scale, self.sampler_kwargs['slices'],
                  seed, chain0=chain0, doubling=bool(self.sampler_kwargs.get('slice_doubling', False)),
                  ell=ell, ctx=self._ctx, peer=peer)

    def prepare_sampler(self, loglstar=None, points=None, axes=None, seeds=None, prior_transform=None,
                        loglikelihood=None, nested_sampler=None):
        ell = self._res.ensure(axes, self._ctx)
        o = self.run_batch(loglstar, np.asarray(points), ell, _seed_of(seeds))
        self.last_batch = o
        _announce(axes, nested_sampler, o['u'])
        ll, ncl = o['logl'].tolist(), o['ncall'].tolist()
        nes, ncs = o['n_expand'].tolist(), o['n_contract'].tolist()
        warns = ((o['flags'] & _lib.WARN_DOUBLING) != 0).tolist()
        SR = SamplerReturn
        if _SR_FAST:
            return [_new_tuple(SR, (u, v, l, c, [], {'n_expand': ne, 'n_contract': nc, 'expansion_warning_set': w},
                                    {'n_expand': ne, 'n_contract': nc}))
                    for u, v, l, c, ne, nc, w in zip(list(o['u']), list(o['v']), ll, ncl, nes, ncs, warns)]
        return [SR(u=u, v=v, logl=l, ncalls=c, evaluation_history=[],
                   tuning_info={'n_expand': ne, 'n_contract': nc, 'expansion_warning_set': w},
                   proposal_stats={'n_expand': ne, 'n_contract': nc})
                for u, v, l, c, ne, nc, w in zip(o['u'], o['v'], ll, ncl, nes, ncs, warns)]

    def tune(self, tuning_info, update=True):
        """tune_slice (internal_samplers.py:1209-1239)."""
        h = self.slice_history
        h['n_expand'] += tuning_info['n_expand']
        h['n_contract'] += tuning_info['n_contract']
        if tuning_info['expansion_warning_set']:
            if not self.sampler_kwargs.get('slice_doubling'):
                warnings.warn('Enabling doubling strategy of slice sampling from Neal(2003)')
            self.sampler_kwargs['slice_doubling'] = True
        if not update:
            return
        ne, nc = max(h['n_expand'], 1), h['n_contract']
        self.scale = self.scale * min(max(ne * 2. / (ne + nc), 0.5), 2.)
        h['n_expand'] = h['n_contract'] = 0

    @property
    def citations(self):
        return [("Neal (2003)", "projecteuclid.org/euclid.aos/1056562461"),
                ("Handley, Hobson & Lasenby (2015a)", "ui.adsabs.harvard.edu/abs/2015MNRAS.450L..61H"),
                ("Handley, Hobson & Lasenby (2015b)", "ui.adsabs.harvard.edu/abs/2015MNRAS.453.4384H")]


class B200RSliceSampler(_B200SliceBase):
    """internal_samplers.py:720-863."""
    _fn = 'rslice_batch'

    @property
    def update_bound_interval_ratio(self):
        return self.sampler_kwargs['slices']


class B200SliceSampler(_B200SliceBase):
    """internal_samplers.py:568-717."""
    _fn = 'slice_batch'

    @property
    def update_bound_interval_ratio(self):
        return self.sampler_kwargs['slices'] * (self.ndim or self.model.ndim)


class B200UniformSampler(_B200Sampler):
    """internal_samplers.py:206-340; needs a B200 bound (the kernel draws from the
    device-resident ellipsoids)."""

    def run_batch(self, loglstar, nchain, bound, seed, chain0=0, ncdim=None, peer=None):
        if getattr(bound, 'kind', None) in ('balls', 'cubes'):          # RadFriends / SupFriends: their own draw
            if peer is not None:
                raise NotImplementedError("fused multi-GPU gather is not wired for the friends bounds")
            n = self.ndim or self.model.ndim
            c = bound._resident()
            return ops.friends_unif_batch(self.model.model_id(c), nchain, n, loglstar, seed, chain0=chain0,
                                          dimflags=self._flags(), ctx=c)
        c = self._ctx if self._ctx is not None else bound.ctx
        if c.resident_key is None or c.resident_key != bound.version:
            bound.make_resident(c)
        n = self.ndim or self.model.ndim
        flags = self._flags()
        return ops.unif_batch(self.model.model_id(self._ctx), nchain, n, loglstar, seed, chain0=chain0,
                              ncdim=ncdim or self.ncdim or n, dimflags=flags, ctx=self._ctx, peer=peer)

    def prepare_sampler(self, loglstar=None, points=None, axes=None, seeds=None, prior_transform=None,
                        loglikelihood=None, nested_sampler=None):
        bound = nested_sampler.bound
        if not hasattr(bound, 'make_resident'):
            raise TypeError("B200UniformSampler needs one of the B200 bounds (ellipsoids or friends)")
        o = self.run_batch(loglstar, len(points), bound, _seed_of(seeds), ncdim=nested_sampler.ncdim)
        self.last_batch = o
        SR = SamplerReturn
        if _SR_FAST:
            return [_new_tuple(SR, (u, v, l, c, [], None, {'n_proposals': npr}))
                    for u, v, l, c, npr in zip(list(o['u']), list(o['v']), o['logl'].tolist(), o['ncall'].tolist(), o['nprop'].tolist())]
        return [SR(u=u, v=v, logl=l, ncalls=c, evaluation_history=[], tuning_info=None,
                   proposal_stats={'n_proposals': npr})
                for u, v, l, c, npr in zip(o['u'], o['v'], o['logl'].tolist(), o['ncall'].tolist(), o['nprop'].tolist())]
