"""K7's group launch of prioritized and uniform learners without a GPU: the binding of include/serl_td3_group_per.h, the
checks serl_td3_train_group_per makes before any CUDA call, Sweep(per=True)'s admission of `per` runs and the runs
examples/sweep.py makes of a `per` grid."""
import ctypes
import importlib.util
import os
import re
import subprocess
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = 'serl_td3_train_group_per'


def test_binding_matches_the_group_per_header(tmp_path):
    from serl_b200 import _native
    text = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'serl_td3_group_per.h')).read(), flags=re.S)
    protos = {n: (r.strip(), [p.strip() for p in ps.split(',')])
              for r, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', text)}
    assert sorted(protos) == sorted(_native.TD3_GROUP_PER_SIGNATURES) == [NAME]
    restype, argtypes = _native.TD3_GROUP_PER_SIGNATURES[NAME]
    ret, params = protos[NAME]
    assert ret == 'int' and restype is ctypes.c_int
    assert len(params) == len(argtypes) == 4
    for decl, t in zip(params, argtypes):
        assert ('*' in decl) == (t is ctypes.c_void_p or issubclass(t, ctypes._Pointer)), decl
        if '*' not in decl:
            assert decl.split()[0] == 'int' and t is ctypes.c_int32, decl
    assert argtypes[0]._type_ is _native.TD3Desc and argtypes[1]._type_ is _native.TD3PerDesc
    src = tmp_path / 'c.c'
    src.write_text('#include "serl_td3_group_per.h"\n'
                   'int (*f)(const serl_td3_desc*, const serl_td3_per_desc*, int, void*) = serl_td3_train_group_per;\n'
                   'int g = SERL_TD3_MAX_GROUP;\n')
    subprocess.check_call(['gcc', '-fsyntax-only', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src)])
    from serl_b200 import build
    build.build()
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), NAME)


def _desc(shape=None, **kw):
    from serl_b200 import _native, rollout
    d = _native.TD3Desc()
    d.shape = shape or rollout.actor_shape(72)
    d.d_state, d.d_replay, d.d_losses = 0x10000, 0x20000, 0x30000          # non-null, never read
    d.replay_cols, d.n_valid, d.batch, d.n_steps, d.policy_update_freq = 19, 1000, 86, 10, 3
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _per(tree=0x40000, **kw):
    from serl_b200 import _native
    p = _native.TD3PerDesc()
    p.d_tree, p.capacity, p.n_valid = tree, 1000, 1000                    # non-null, never read
    p.alpha, p.beta0, p.beta_frames = 0.6, 0.4, 1e5
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _group(descs, pers, n=None):
    from serl_b200 import _native
    a = (_native.TD3Desc * max(len(descs), 1))(*descs)
    b = (_native.TD3PerDesc * max(len(pers), 1))(*pers)
    rc = _native.lib().serl_td3_train_group_per(a, b, len(descs) if n is None else n, None)
    return rc, _native.lib().serl_last_error().decode()


def test_group_per_is_rejected_before_any_cuda_call():
    """every failure is SERL_ERR_ARG with a message naming the learner; the device pointers are never dereferenced"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    ok = [_desc(seed=s) for s in range(3)]
    pers = [_per(), _per(tree=None), _per()]
    assert L.serl_td3_train_group_per(None, (_native.TD3PerDesc * 1)(_per()), 1, None) == -1
    assert L.serl_last_error().decode() == NAME + ': null descriptors'
    assert L.serl_td3_train_group_per((_native.TD3Desc * 1)(_desc()), None, 1, None) == -1
    assert L.serl_last_error().decode() == NAME + ': null descriptors'
    rc, msg = _group(ok, pers, 0)
    assert rc == -1 and msg.startswith(NAME + ': n must be')
    rc, msg = _group([_desc()] * (_native.TD3_MAX_GROUP + 1), [_per()] * (_native.TD3_MAX_GROUP + 1))
    assert rc == -1 and msg.startswith(NAME + ': n must be')
    rc, msg = _group(ok[:2] + [_desc(cluster_size=4)], pers)
    assert rc == -1 and msg.startswith(NAME + ': learner 2:') and 'cluster_size' in msg
    # every check of serl_td3_train, for a prioritized and for a uniform learner, naming it
    for kw in (dict(batch=129), dict(batch=0), dict(n_valid=85), dict(replay_cols=18), dict(policy_update_freq=0),
               dict(cluster_size=3), dict(flags=2), dict(d_state=None), dict(d_replay=None), dict(d_losses=None),
               dict(n_steps=-1), dict(first_iteration=-1), dict(critic_adam_steps=-1),
               dict(shape=rollout.actor_shape(48)), dict(shape=rollout.actor_shape(400, 3)),
               dict(shape=rollout.actor_shape(256, 9))):
        for j in (0, 1):                  # learner 0 is prioritized, learner 1 uniform
            descs = list(ok)
            descs[j] = _desc(**kw)
            rc, msg = _group(descs, pers)
            assert rc == -1 and msg.startswith('%s: learner %d:' % (NAME, j)), (kw, j, rc, msg)
    # every check of serl_td3_train_per, for a learner with a tree
    for kw in (dict(capacity=0), dict(capacity=(1 << 30) + 1), dict(n_valid=999), dict(capacity=999, n_valid=1000),
               dict(alpha=0.0), dict(alpha=1.5), dict(alpha=float('nan')), dict(beta0=-0.1), dict(beta0=1.1),
               dict(beta_frames=0.0), dict(beta_frames=float('nan'))):
        rc, msg = _group(ok, pers[:2] + [_per(**kw)])
        assert rc == -1 and msg.startswith(NAME + ': learner 2:'), (kw, rc, msg)
        # ...which a learner without a tree ignores: its other fields are not read
        ok_pers = pers[:2] + [_per(tree=None, **kw)]
        before = L.serl_launch_count()
        assert _group([_desc(n_steps=0, seed=s) for s in range(3)], ok_pers)[0] == 0, kw
        assert L.serl_launch_count() == before


def test_group_without_steps_makes_no_launch():
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    shapes = [rollout.actor_shape(72), rollout.actor_shape(256), rollout.actor_shape(72, 2), rollout.actor_shape(320, 8)]
    before = L.serl_launch_count()
    # prioritized and uniform, narrow and wide, cluster_size 0 and 8 agreeing, and nothing to do
    rc, msg = _group([_desc(s, n_steps=0, cluster_size=c) for s, c in zip(shapes, (0, 8, 0, 8))],
                     [_per(), _per(tree=None), _per(tree=None), _per()])
    assert rc == 0, msg
    assert L.serl_launch_count() == before


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
