"""K7 for learners of different actor shapes in one launch, without a GPU: the binding of include/serl_td3_mixed.h, the
argument checks serl_td3_train_mixed makes before any CUDA call, the runs a mixed-shape Sweep refuses before it builds any
Agent, and the runs examples/sweep.py makes of a shape grid."""
import ctypes
import importlib.util
import os
import re
import subprocess
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_binding_matches_the_mixed_header(tmp_path):
    from serl_b200 import _native
    text = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'serl_td3_mixed.h')).read(), flags=re.S)
    protos = {n: (r.strip(), [p.strip() for p in ps.split(',')])
              for r, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', text)}
    assert sorted(protos) == sorted(_native.TD3_MIXED_SIGNATURES) == ['serl_td3_train_mixed']
    assert '#include "serl_td3_mixed.h"' in open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    restype, argtypes = _native.TD3_MIXED_SIGNATURES['serl_td3_train_mixed']
    ret, params = protos['serl_td3_train_mixed']
    assert ret == 'int' and restype is ctypes.c_int
    assert params == ['const serl_td3_desc* descs', 'int n', 'void* stream']
    assert len(argtypes) == 3
    assert argtypes[0]._type_ is _native.TD3Desc and argtypes[1] is ctypes.c_int32 and argtypes[2] is ctypes.c_void_p
    src = tmp_path / 'c.c'
    src.write_text('#include "serl_b200.h"\n'
                   'int (*f)(const serl_td3_desc*, int, void*) = serl_td3_train_mixed;\n')
    subprocess.check_call(['gcc', '-fsyntax-only', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src)])
    # the K7 headers still stand on their own, whichever is included first
    for h in ('serl_td3.h', 'serl_td3_group.h', 'serl_td3_mixed.h'):
        src.write_text('#include "%s"\n#include "serl_td3_mixed.h"\n'
                       'int (*f)(const serl_td3_desc*, int, void*) = serl_td3_train_mixed;\n' % h)
        subprocess.check_call(['gcc', '-fsyntax-only', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src)])
    from serl_b200 import build
    build.build()
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), 'serl_td3_train_mixed')


def _desc(shape=None, **kw):
    from serl_b200 import _native, rollout
    d = _native.TD3Desc()
    d.shape = shape or rollout.actor_shape(72)
    d.d_state, d.d_replay, d.d_losses = 0x10000, 0x20000, 0x30000          # non-null, never read
    d.replay_cols, d.n_valid, d.batch, d.n_steps, d.policy_update_freq = 19, 1000, 86, 10, 3
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _mixed(descs, n=None):
    from serl_b200 import _native
    arr = (_native.TD3Desc * max(len(descs), 1))(*descs)
    rc = _native.lib().serl_td3_train_mixed(arr, len(descs) if n is None else n, None)
    return rc, _native.lib().serl_last_error().decode()


def _shapes():
    from serl_b200 import rollout
    return [rollout.actor_shape(32, 1, 'tanh'), rollout.actor_shape(72, 3, 'elu'), rollout.actor_shape(256, 3, 'relu')]


def test_mixed_group_is_rejected_before_any_cuda_call():
    """every failure is SERL_ERR_ARG with a message, and no kernel is launched; the device pointers are never read"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    before = L.serl_launch_count()
    ok = [_desc(s, seed=k) for k, s in enumerate(_shapes())]
    rc, msg = _mixed(ok, 0)
    assert rc == -1 and msg == 'serl_td3_train_mixed: n must be 1..SERL_TD3_MAX_GROUP (64)'
    rc, msg = _mixed([_desc()] * (_native.TD3_MAX_GROUP + 1))
    assert rc == -1 and msg.startswith('serl_td3_train_mixed: n must be')
    rc = L.serl_td3_train_mixed(None, 2, None)
    assert rc == -1 and L.serl_last_error().decode() == 'serl_td3_train_mixed: null descriptors'
    rc, msg = _mixed(ok[:2] + [_desc(rollout.actor_shape(256), cluster_size=4)])
    assert rc == -1 and msg.startswith('serl_td3_train_mixed: learner 2:') and 'cluster_size' in msg
    # every check of serl_td3_train, per learner, naming it
    for kw in (dict(batch=129), dict(batch=0), dict(n_valid=85), dict(replay_cols=18), dict(policy_update_freq=0),
               dict(cluster_size=3), dict(flags=2), dict(d_state=None), dict(d_replay=None), dict(d_losses=None),
               dict(n_steps=-1), dict(first_iteration=-1), dict(critic_adam_steps=-1), dict(actor_adam_steps=-1),
               dict(shape=rollout.actor_shape(48)), dict(shape=rollout.actor_shape(400, 3)),
               dict(shape=rollout.actor_shape(256, 9)), dict(shape=rollout.actor_shape(72, 0)),
               dict(shape=rollout.actor_shape(72, 3, 'tanh', state_dim=6))):
        for i in range(3):
            descs = list(ok)
            descs[i] = _desc(**dict(dict(shape=_shapes()[i]), **kw))
            rc, msg = _mixed(descs)
            assert rc == -1 and msg.startswith('serl_td3_train_mixed: learner %d: ' % i), (kw, i, rc, msg)
    assert L.serl_launch_count() == before


def test_mixed_group_without_steps_makes_no_launch():
    from serl_b200 import build, _native
    build.build()
    L = _native.lib()
    before = L.serl_launch_count()
    # different shapes, both hidden classes, cluster_size 0 and 8 agreeing, and nothing to do
    assert _mixed([_desc(s, n_steps=0, cluster_size=c) for s, c in zip(_shapes(), (0, 8, 0))])[0] == 0
    assert L.serl_launch_count() == before
    # the uniform entry point still refuses the same group for its shapes
    arr = (_native.TD3Desc * 3)(*[_desc(s, n_steps=0) for s in _shapes()])
    assert L.serl_td3_train_group(arr, 3, None) == -1
    assert L.serl_last_error().decode().startswith('serl_td3_train_group: learner 1: actor shape differs')


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
