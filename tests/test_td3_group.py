"""K7 group launch and the sweep driver without a GPU: the shapes train_group refuses to group, the per-run generator swap
and the runs a Sweep refuses."""
import os
import random
import types

import numpy as np
import pytest
import torch



def test_train_group_refuses_shapes_it_cannot_group():
    """train_group refuses learners of different actor shapes before it reads their replays or launches, unless
    mixed_shapes or prioritized lets one launch train them; serl_td3_learn's own refusals are in test_td3_oracle.py"""
    from serl_b200 import _native, rollout, td3_fused
    learner = lambda *shape: types.SimpleNamespace(shape=rollout.actor_shape(*shape), state=torch.zeros(1))
    for bad in ((64,), (72, 2), (72, 3, 'elu')):
        learners = [learner(72), learner(72), learner(*bad)]
        with pytest.raises(_native.NativeError, match=r"train_group: learner 2: actor shape differs from learner 0's"):
            td3_fused.train_group(learners, [None] * 3, [10] * 3, [1] * 3, [False] * 3)
    learners = [learner(72), learner(256)]
    for kw in (dict(mixed_shapes=True), dict(prioritized=True)):
        with pytest.raises(AssertionError):          # past the shape check: the CPU rows are refused
            td3_fused.train_group(learners, [torch.zeros(100, 19)] * 2, [10] * 2, [1] * 2, [False] * 2, **kw)


def _draws():
    return random.random(), np.random.rand(3).tolist(), torch.rand(2).tolist()


def test_rng_scope_swaps_the_global_generators_exactly():
    from serl_b200.sweep import RNGState, rng_scope
    random.seed(1); np.random.seed(1); torch.manual_seed(1)
    a = RNGState.capture()
    random.seed(2); np.random.seed(2); torch.manual_seed(2)
    b = RNGState.capture()
    random.seed(99); np.random.seed(99); torch.manual_seed(99)
    outer = RNGState.capture()
    expect_outer = _draws()
    outer.restore()
    # run a, run b, run a: each continues its own streams; the caller's streams are untouched
    with rng_scope(a):
        a1 = _draws()
    with rng_scope(b):
        b1 = _draws()
    with rng_scope(a):
        a2 = _draws()
    assert _draws() == expect_outer
    random.seed(1); np.random.seed(1); torch.manual_seed(1)
    assert [_draws(), _draws()] == [a1, a2]
    random.seed(2); np.random.seed(2); torch.manual_seed(2)
    assert _draws() == b1
    # the state is restored even when the block raises
    with pytest.raises(KeyError):
        with rng_scope(b):
            raise KeyError
    random.seed(5)
    x = random.getstate()
    with rng_scope(a):
        _draws()
    assert random.getstate() == x


def _params(tmp_path, **kw):
    from serl_b200.parameters import Parameters
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=4, mut_type='normal', test_ea=False,
                                             fused_td3=True))
    finally:
        os.chdir(cwd)
    p.state_dim, p.action_dim = 7, 3
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_sweep_refuses_runs_it_cannot_group(tmp_path):
    from serl_b200.sweep import Sweep
    with pytest.raises(ValueError, match='no runs'):
        Sweep([])
    with pytest.raises(ValueError, match='fused_td3'):
        Sweep([(_params(tmp_path), None), (_params(tmp_path, fused_td3=False), None)])
    for kw in (dict(hidden_size=64), dict(num_layers=2), dict(activation_actor='elu')):
        with pytest.raises(ValueError, match='actor shape'):
            Sweep([(_params(tmp_path), None), (_params(tmp_path, **kw), None)])
