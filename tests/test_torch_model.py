"""TorchModel on the CPU tier: the checks of the callables' outputs and the options a TorchModel refuses (no GPU:
the callables run on CPU tensors, and the refusals come before any device work)."""
import numpy as np
import pytest
import torch

from dynesty_b200 import TorchModel, nested


def _model(like=None, prior=None, n=3):
    return TorchModel(n, like or (lambda v: v.sum(1)), prior or (lambda u: 2.0 * u), name='m')


def test_outputs_pass_and_are_checked_once_per_batch_size():
    m = _model()
    u = torch.rand(5, 3, dtype=torch.float64)
    v, l = m._eval(u)
    assert torch.equal(v, 2.0 * u) and torch.equal(l, (2.0 * u).sum(1))
    assert (m.prior_transform_fn, 5) in m._checked and (m.loglike, 5) in m._checked
    m._eval(torch.rand(7, 3, dtype=torch.float64))
    assert (m.loglike, 7) in m._checked


def bad_loglike_shape(v):
    return v.sum(1, keepdim=True)


def bad_prior_dtype(u):
    return u.float()


def bad_loglike_device(v):
    return torch.empty(v.shape[0], dtype=torch.float64, device='meta')


@pytest.mark.parametrize('kw,match', [
    (dict(like=bad_loglike_shape), r'bad_loglike_shape of TorchModel .*shape \(4, 1\)'),
    (dict(prior=bad_prior_dtype), r'bad_prior_dtype of TorchModel .*dtype torch.float32'),
    (dict(like=bad_loglike_device), r'bad_loglike_device of TorchModel .*meta'),
    (dict(like=lambda v: v.sum(1).numpy()), r'not a torch.Tensor'),
])
def test_wrong_outputs_raise_naming_the_callable(kw, match):
    m = _model(**kw)
    with pytest.raises(ValueError, match=match):
        m._eval(torch.rand(4, 3, dtype=torch.float64))


def test_constructor_checks():
    with pytest.raises(TypeError):
        TorchModel(3, None, lambda u: u)
    with pytest.raises(ValueError):
        TorchModel(0, lambda v: v, lambda u: u)
    assert TorchModel.model_id() == -1


@pytest.mark.parametrize('sample', ['unif', 'slice', 'rslice'])
def test_samplers_without_a_stepped_form_refuse(sample):
    with pytest.raises(NotImplementedError, match='rwalk'):
        nested.NestedSampler(_model(), nlive=20, sample=sample)


def test_blob_and_comm_refused():
    with pytest.raises(ValueError, match='blob'):
        nested.NestedSampler(_model(), nlive=20, blob=True)
    with pytest.raises(ValueError, match='comm'):
        nested.NestedSampler(_model(), nlive=20, comm=object())


def test_checkpoint_refused_and_defaults():
    rng = np.random.default_rng(0)
    u = rng.random((20, 3))
    s = nested.NestedSampler(_model(), nlive=20, live_points=(u, 2 * u, (2 * u).sum(1)))
    assert s.sample_name == 'rwalk' and s.device_init is False
    with pytest.raises(ValueError, match='checkpoint_file'):
        s.run_nested(loop='device', checkpoint_file='x.pkl')
