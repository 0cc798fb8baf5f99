"""K7 group launch and the sweep driver without a GPU: the binding of include/serl_td3_group.h, the argument checks
serl_td3_train_group makes before any CUDA call, the per-run generator swap and the runs a Sweep refuses."""
import ctypes
import os
import random
import re
import subprocess
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_binding_matches_the_group_header(tmp_path):
    from serl_b200 import _native
    text = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'serl_td3_group.h')).read(), flags=re.S)
    protos = {n: (r.strip(), [p.strip() for p in ps.split(',')])
              for r, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', text)}
    assert sorted(protos) == sorted(_native.TD3_GROUP_SIGNATURES) == ['serl_td3_train_group']
    assert '#include "serl_td3_group.h"' in open(os.path.join(ROOT, 'include', 'serl_td3.h')).read()
    restype, argtypes = _native.TD3_GROUP_SIGNATURES['serl_td3_train_group']
    ret, params = protos['serl_td3_train_group']
    assert ret == 'int' and restype is ctypes.c_int
    assert len(params) == len(argtypes) == 3
    assert argtypes[0]._type_ is _native.TD3Desc and argtypes[1] is ctypes.c_int32 and argtypes[2] is ctypes.c_void_p
    src = tmp_path / 'c.c'
    src.write_text('#include "serl_b200.h"\n'
                   'int (*f)(const serl_td3_desc*, int, void*) = serl_td3_train_group;\n')
    subprocess.check_call(['gcc', '-fsyntax-only', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src)])
    out = subprocess.check_output(['gcc', '-E', '-dM', '-I', os.path.join(ROOT, 'include'), str(src)], text=True)
    assert '#define SERL_TD3_MAX_GROUP %d' % _native.TD3_MAX_GROUP in out
    from serl_b200 import build
    build.build()
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), 'serl_td3_train_group')


def _desc(**kw):
    from serl_b200 import _native, rollout
    d = _native.TD3Desc()
    d.shape = rollout.actor_shape(72)
    d.d_state, d.d_replay, d.d_losses = 0x10000, 0x20000, 0x30000          # non-null, never read
    d.replay_cols, d.n_valid, d.batch, d.n_steps, d.policy_update_freq = 19, 1000, 86, 10, 3
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _group(descs, n=None):
    from serl_b200 import _native
    arr = (_native.TD3Desc * max(len(descs), 1))(*descs)
    rc = _native.lib().serl_td3_train_group(arr, len(descs) if n is None else n, None)
    return rc, _native.lib().serl_last_error().decode()


def test_group_is_rejected_before_any_cuda_call():
    """every failure is SERL_ERR_ARG with a message; the device pointers are never dereferenced"""
    from serl_b200 import build, _native, rollout
    build.build()
    ok = [_desc(seed=s) for s in range(3)]
    rc, msg = _group(ok, 0)
    assert rc == -1 and 'n must be' in msg
    rc, msg = _group([_desc()] * (_native.TD3_MAX_GROUP + 1))
    assert rc == -1 and 'n must be' in msg
    rc = _native.lib().serl_td3_train_group(None, 2, None)
    assert rc == -1 and 'null' in _native.lib().serl_last_error().decode()
    rc, msg = _group(ok[:2] + [_desc(shape=rollout.actor_shape(64))])
    assert rc == -1 and 'learner 2' in msg and 'shape' in msg
    rc, msg = _group(ok[:1] + [_desc(shape=rollout.actor_shape(72, 2))])
    assert rc == -1 and 'learner 1' in msg and 'shape' in msg
    rc, msg = _group(ok[:1] + [_desc(cluster_size=4)])
    assert rc == -1 and 'learner 1' in msg and 'cluster_size' in msg
    # every check of serl_td3_train, per learner, naming it
    for kw in (dict(batch=129), dict(batch=0), dict(n_valid=85), dict(replay_cols=18), dict(policy_update_freq=0),
               dict(cluster_size=3), dict(flags=2), dict(d_state=None), dict(d_losses=None), dict(n_steps=-1),
               dict(first_iteration=-1), dict(shape=rollout.actor_shape(48)), dict(shape=rollout.actor_shape(400, 3))):
        rc, msg = _group(ok[:1] + [_desc(**kw)] + ok[1:])
        assert rc == -1 and msg.startswith('serl_td3_train_group: learner 1:'), (kw, rc, msg)
    rc, msg = _group([_desc(shape=rollout.actor_shape(100))] * 2)
    assert rc == -1 and 'learner 0' in msg and 'shape' in msg
    # the same shape everywhere, cluster_size 0 and 8 agreeing, and nothing to do: no launch
    before = _native.lib().serl_launch_count()
    assert _group([_desc(n_steps=0, cluster_size=c) for c in (0, 8, 0)])[0] == 0
    assert _native.lib().serl_launch_count() == before


def test_solo_entry_point_keeps_its_messages():
    from serl_b200 import build, _native
    build.build()
    L = _native.lib()
    assert L.serl_td3_train(ctypes.byref(_desc(batch=129)), None) == -1
    assert L.serl_last_error().decode() == 'serl_td3_train: batch must be 1..128'
    assert L.serl_td3_train(ctypes.byref(_desc(cluster_size=3)), None) == -1
    assert L.serl_last_error().decode() == 'serl_td3_train: cluster_size must be 0, 1, 2, 4 or 8'


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
