"""K7's group launch of prioritized and uniform learners without a GPU: Sweep(per=True)'s admission of `per` runs and the
runs examples/sweep.py makes of a `per` grid."""
import importlib.util
import os
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def test_per_sweep_admits_per_runs_before_building_an_agent(tmp_path, monkeypatch):
    from serl_b200 import build
    from serl_b200.core import agent as agent_mod
    from serl_b200.sweep import Sweep
    build.build()

    def no_agent(*a, **k):
        raise AssertionError('an Agent was built')
    monkeypatch.setattr(agent_mod, 'Agent', no_agent)
    env = types.SimpleNamespace(seed=lambda s: None)
    # per runs beside uniform ones, of one shape or (mixed_shapes) of several, pass every check and reach the Agent
    with pytest.raises(AssertionError, match='an Agent was built'):
        Sweep([(_params(tmp_path, per=True), env), (_params(tmp_path), env)], per=True)
    with pytest.raises(AssertionError, match='an Agent was built'):
        Sweep([(_params(tmp_path, per=True), env), (_params(tmp_path, hidden_size=256, per=True), env),
               (_params(tmp_path), env)], mixed_shapes=True, per=True)
    # without per=True the refusal stands, and points at per=True
    with pytest.raises(ValueError, match=r'Sweep: run 1 sets per \(prioritized experience replay\).*per=True'):
        Sweep([(_params(tmp_path), None), (_params(tmp_path, per=True), None)], mixed_shapes=True)
    # the other refusals are unchanged with per=True
    with pytest.raises(ValueError, match='run 1 flies incremental control'):
        Sweep([(_params(tmp_path, per=True), None), (_params(tmp_path, per=True, state_dim=10), None)], per=True)
    with pytest.raises(ValueError, match='run 1 flies symmetric control'):
        Sweep([(_params(tmp_path, per=True), None), (_params(tmp_path, per=True, state_dim=2, action_dim=1), None)], per=True)
    with pytest.raises(ValueError, match='run 1 does not set fused_td3'):
        Sweep([(_params(tmp_path, per=True), None), (_params(tmp_path, per=True, fused_td3=False), None)], per=True)
    with pytest.raises(ValueError, match='actor shape'):
        Sweep([(_params(tmp_path, per=True), None), (_params(tmp_path, hidden_size=96), None)], per=True)


def _example(tmp_path, monkeypatch):
    """examples/sweep.py under a private name; it adds its flags to train.py's parser, so it imports a fresh `train`
    module, which is dropped again: no parser with those flags is left behind, and a `train` imported before is kept"""
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(ROOT, 'examples'))
    had_train = sys.modules.pop('train', None)
    try:
        spec = importlib.util.spec_from_file_location('sweep_example', os.path.join(ROOT, 'examples', 'sweep.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        if had_train is None:
            sys.modules.pop('train', None)
        else:
            sys.modules['train'] = had_train
    assert sys.modules.get('sweep_example') is None
    return mod


def test_example_per_grid_makes_a_uniform_and_a_per_run(tmp_path, monkeypatch):
    mod = _example(tmp_path, monkeypatch)
    runs = mod.make_runs(mod.parser.parse_args(['-frames', '1000', '-grid', 'per=0,1']))
    assert [p.per for _, p, _ in runs] == [False, True]
    assert all(p.fused_td3 for _, p, _ in runs)
    runs = mod.make_runs(mod.parser.parse_args(['-frames', '1000', '-seeds', '7', '8', '-grid', 'per=0,1']))
    assert [(p.seed, p.per) for _, p, _ in runs] == [(7, False), (7, True), (8, False), (8, True)]
    runs = mod.make_runs(mod.parser.parse_args(['-frames', '1000', '-per', '-seeds', '7', '8', '9']))
    assert len(runs) == 3 and all(p.per for _, p, _ in runs)
    text = open(os.path.join(ROOT, 'examples', 'sweep.py')).read()
    assert 'mixed_shapes=True, per=True' in text
