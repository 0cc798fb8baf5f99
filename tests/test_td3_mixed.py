"""K7 for learners of different actor shapes in one launch, without a GPU: the runs a mixed-shape Sweep refuses before it
builds any Agent, and the runs examples/sweep.py makes of a shape grid."""
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


def test_mixed_sweep_refuses_runs_before_building_an_agent(tmp_path, monkeypatch):
    from serl_b200 import build
    from serl_b200.core import agent as agent_mod
    from serl_b200.sweep import Sweep
    build.build()

    def no_agent(*a, **k):
        raise AssertionError('an Agent was built before the runs were checked')
    monkeypatch.setattr(agent_mod, 'Agent', no_agent)
    with pytest.raises(ValueError, match='run 1 does not set fused_td3'):
        Sweep([(_params(tmp_path), None), (_params(tmp_path, fused_td3=False), None)], mixed_shapes=True)
    for kw in (dict(hidden_size=48), dict(hidden_size=400), dict(hidden_size=256, num_layers=9)):
        with pytest.raises(ValueError, match=r'run 2 has actor shape .* which K7 does not train'):
            Sweep([(_params(tmp_path), None), (_params(tmp_path, hidden_size=256), None), (_params(tmp_path, **kw), None)],
                  mixed_shapes=True)
    # shapes inside K7's domain pass the checks and reach the Agent; without mixed_shapes the refusal is today's
    env = types.SimpleNamespace(seed=lambda s: None)
    with pytest.raises(AssertionError, match='an Agent was built'):
        Sweep([(_params(tmp_path), env), (_params(tmp_path, hidden_size=256, activation_actor='relu'), env)], mixed_shapes=True)
    with pytest.raises(ValueError, match='actor shape'):
        Sweep([(_params(tmp_path), None), (_params(tmp_path, hidden_size=96), None)])


def test_example_shape_grid_makes_one_run_per_shape(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    monkeypatch.syspath_prepend(os.path.join(ROOT, 'examples'))
    spec = importlib.util.spec_from_file_location('sweep_example', os.path.join(ROOT, 'examples', 'sweep.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    cla = mod.parser.parse_args(['-frames', '1000', '-grid', 'hidden_size=72,96', 'activation_actor=tanh,relu'])
    runs = mod.make_runs(cla)
    from serl_b200.sweep import _shape
    assert len(runs) == 4
    assert len({_shape(p) for _, p, _ in runs}) == 4
    assert {(p.hidden_size, p.activation_actor) for _, p, _ in runs} == {(72, 'tanh'), (72, 'relu'), (96, 'tanh'), (96, 'relu')}
    assert all(p.fused_td3 for _, p, _ in runs)
    assert 'mixed_shapes=True' in open(os.path.join(ROOT, 'examples', 'sweep.py')).read()
    assert sys.modules.get('sweep_example') is None
