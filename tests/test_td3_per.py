"""Prioritized experience replay (include/serl_td3_per.h, csrc/per.cu, K7's PER learner) on the CPU: the priority tree
restated in numpy against the reference's PrioritizedReplayMemory, the weight and beta formulas against its arithmetic, the
ctypes mirror of the header, the tree entry points' refusals, and the weighted oracle (tests/td3_per_oracle.py) against
oracle/td3.py and the torch TD3's weighted path.  serl_td3_learn's refusals of a prioritized learner are in
test_td3_oracle.py."""
import copy
import ctypes
import importlib.util
import os
import re
import subprocess
import types

import numpy as np
import pytest
import torch

import td3_per_oracle as P
from oracle import td3 as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_BUFFER = '/root/reference/base/core/replay_memory.py'


def reference_buffer_module():
    spec = importlib.util.spec_from_file_location('reference_replay_memory', REF_BUFFER)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- the tree -------------------------------------------------------------------------------------------------------------

def check_tree(tree):
    t, L = tree.t, tree.leaves
    for v in range(1, L):
        assert t[v, 0] == t[2 * v, 0] + t[2 * v + 1, 0] and t[v, 1] == min(t[2 * v, 1], t[2 * v + 1, 1])
    p = tree.priorities()
    assert np.all(t[L + tree.n_valid:, 0] == 0) and np.all(np.isinf(t[L + tree.n_valid:, 1]))
    if p.size:
        assert t[1, 1] == p.min()
        assert abs(t[1, 0] - p.sum()) <= 1e-12 * p.sum()


@pytest.mark.skipif(not os.path.exists(REF_BUFFER), reason='needs the reference tree')
def test_tree_follows_the_reference_buffer_through_adds_updates_and_wraps():
    """the same adds (single, bulk, past the capacity) and update_priorities calls (with a row drawn twice) on the
    reference's PrioritizedReplayMemory and on the tree: the same priorities, max and min"""
    R = reference_buffer_module()
    cap = 37
    ref = R.PrioritizedReplayMemory(cap, 'cpu')
    tree = P.NumpyTree(cap)
    rng = np.random.RandomState(0)
    z = lambda: (np.zeros(7), np.zeros(3), np.zeros(7), 0.0, 0.0)
    for step, n in enumerate([1, 5, 12, 30, 3, 50, 9, 37, 1]):
        for _ in range(n):
            ref.add(*z())
        tree.add(n)
        check_tree(tree)
        assert tree.n_valid == len(ref)
        rows = rng.randint(0, len(ref), size=8)
        rows[-1] = rows[0]                                   # drawn twice: the later TD error wins
        td = rng.rand(8) * 3
        ref.update_priorities(rows, td)
        tree.update(rows, td)
        check_tree(tree)
        want = ref.priorities[:len(ref)].astype(np.float64)
        np.testing.assert_allclose(tree.priorities(), want, rtol=1e-6, err_msg=str(step))
        assert tree.priorities()[rows[-1]] == pytest.approx((td[-1] + 1e-5) ** 0.6, rel=1e-12)
        np.testing.assert_allclose([tree.t[1, 1], tree.priorities().max()], [want.min(), ref.priorities.max()], rtol=1e-6)


def test_bulk_add_equals_sequential_adds():
    """a bulk add of n rows gives every new or overwritten row the max stored before it: n single adds give the same"""
    rng = np.random.RandomState(1)
    bulk, single = P.NumpyTree(20), P.NumpyTree(20)
    for n in (3, 11, 25, 7):
        bulk.add(n)
        for _ in range(n):
            single.add(1)
        rows, td = rng.randint(0, bulk.n_valid, size=6), rng.rand(6)
        bulk.update(rows, td)
        single.update(rows, td)
        assert np.array_equal(bulk.t, single.t)


@pytest.mark.skipif(not os.path.exists(REF_BUFFER), reason='needs the reference tree')
def test_beta_and_weights_follow_the_reference_arithmetic():
    R = reference_buffer_module()
    ref = R.PrioritizedReplayMemory(100, 'cpu', beta_frames=5000)
    for f in (1, 2, 17, 2999, 3000, 4999, 5000, 9000):
        assert P.beta_by_frame(f, 0.4, 5000) == ref.beta_by_frame(f)
    from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory
    buf = DevicePrioritizedReplayMemory(100, 'cpu', beta_frames=5000)
    assert all(buf.beta_by_frame(f) == ref.beta_by_frame(f) for f in (1, 2999, 5000, 9000))
    # the weight of row i: the reference's float32 arithmetic (replay_memory.py:147-157) against the fp64 formula the
    # device uses (csrc/per.cuh per_weight)
    rng = np.random.RandomState(2)
    prios = ((rng.rand(77) * 4 + 1e-5) ** 0.6).astype(np.float32)
    probs = prios / prios.sum()
    for beta in (0.4, 0.73, 1.0):
        want = (len(prios) * probs) ** (-beta) / (probs.min() * len(prios)) ** (-beta)
        p = prios.astype(np.float64)
        got = (len(p) * (p / p.sum())) ** -beta / (len(p) * (p.min() / p.sum())) ** -beta
        np.testing.assert_allclose(got, want, rtol=2e-6)
        assert got.max() == pytest.approx(1.0) and got.min() > 0


# ---- the header and its binding ---------------------------------------------------------------------------------------------

def header_text(name):
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', name)).read(), flags=re.S)


def test_binding_matches_the_per_header():
    from serl_b200 import _native
    protos = {n: [p.strip() for p in ps.split(',')]
              for _, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', header_text('serl_td3_per.h'))}
    assert sorted(protos) == sorted(_native.PER_SIGNATURES)
    for name, params in protos.items():
        restype, argtypes = _native.PER_SIGNATURES[name]
        assert len(argtypes) == len(params), name
        for decl, t in zip(params, argtypes):
            assert ('*' in decl) == (t is ctypes.c_void_p or issubclass(t, ctypes._Pointer)), (name, decl)
            if '*' not in decl:
                kind = decl.split()[0]
                assert {'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64, 'uint64_t': ctypes.c_uint64,
                        'double': ctypes.c_double}[kind] is t, (name, decl)
    assert _native.PER_SIGNATURES['serl_per_tree_doubles'][0] is ctypes.c_int64


def test_ctypes_mirror_of_the_per_descriptor_matches_the_header(tmp_path):
    from serl_b200 import _native
    fields = [f for f, _ in _native.TD3PerDesc._fields_]
    src = tmp_path / 'layout.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "serl_td3_per.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(serl_td3_per_desc));\n' +
                   ''.join('  printf("%%zu\\n", offsetof(serl_td3_per_desc, %s));\n' % f for f in fields) +
                   '  printf("%lld\\n", (long long)SERL_PER_MAX_CAPACITY);\n  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert out[0] == ctypes.sizeof(_native.TD3PerDesc)
    assert out[1:1 + len(fields)] == [getattr(_native.TD3PerDesc, f).offset for f in fields]
    assert out[-1] == _native.PER_MAX_CAPACITY


def test_tree_entry_points_refuse_bad_arguments():
    """the tree's entry points refuse bad sizes, rows and parameters with SERL_ERR_ARG; the device pointers are never
    dereferenced"""
    from serl_b200 import build, _native
    build.build()
    L = _native.lib()
    assert L.serl_per_tree_doubles(800_000) == 4 * (1 << 20) and L.serl_per_tree_doubles(1) == 4
    assert L.serl_per_tree_doubles(0) == -1 and L.serl_per_tree_doubles(-5) == -1
    assert L.serl_per_insert(0x40000, 100, 101, 0, 1, None) == -1
    assert L.serl_per_insert(0x40000, 100, 0, 100, 1, None) == -1
    assert L.serl_per_insert(0x40000, 100, 0, 0, 101, None) == -1
    assert L.serl_per_insert(None, 100, 0, 0, 1, None) == -1
    assert L.serl_per_update(0x40000, 100, 0x50000, 0x60000, 129, 0.6, None) == -1
    assert L.serl_per_update(0x40000, 100, 0x50000, 0x60000, 86, 0.0, None) == -1
    assert L.serl_per_sample(0x40000, 100, 0, 86, 7, 1, 0.4, 0x50000, 0x60000, None) == -1
    assert L.serl_per_sample(0x40000, 100, 50, 86, 7, 1, 1.5, 0x50000, 0x60000, None) == -1
    assert L.serl_per_rebuild(None, 100, None) == -1


# ---- the weighted oracle ----------------------------------------------------------------------------------------------------

def td3_args(activation='tanh', use_caps=True, batch_size=16):
    return types.SimpleNamespace(device='cpu', individual_bs=100, hidden_size=32, num_layers=1, activation_actor=activation,
                                 state_dim=7, action_dim=3, lr=1e-3, gamma=0.98, tau=0.005, noise_sd=0.2962183114680794,
                                 noise_clip=0.5, policy_update_freq=3, use_caps=use_caps, batch_size=batch_size, seed=7)


def replay_rows(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn((n, 19), generator=g) * 0.3
    rows[:, 7:10] = torch.rand((n, 3), generator=g) * 2 - 1
    rows[:, 18] = (torch.rand(n, generator=g) < 0.1).float()
    return rows


def same_learner(a, b):
    for ma, mb in ((a.actor, b.actor), (a.actor_target, b.actor_target), (a.critic, b.critic), (a.critic_target, b.critic_target)):
        for pa, pb in zip(ma.parameters(), mb.parameters()):
            if not torch.equal(pa, pb):
                return False
    for oa, ob in ((a.actor_optim, b.actor_optim), (a.critic_optim, b.critic_optim)):
        for sa, sb in zip(oa.state.values(), ob.state.values()):
            if not all(torch.equal(sa[k], sb[k]) for k in ('exp_avg', 'exp_avg_sq', 'step')):
                return False
    return True


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('use_caps,champion,activation', [(True, False, 'tanh'), (False, False, 'elu'), (True, True, 'relu')])
def test_weighted_oracle_with_unit_weights_is_the_oracle_bit_for_bit(dtype, use_caps, champion, activation):
    from serl_b200.core.td3 import TD3
    torch.manual_seed(3)
    base = TD3(td3_args(activation, use_caps))
    a, b = (copy.deepcopy(base), copy.deepcopy(base)) if dtype == torch.float32 else (O.as_float64(base), O.as_float64(base))
    rows = replay_rows(64).to(dtype)
    g = torch.Generator().manual_seed(5)
    for it in range(1, 8):
        batch = rows[(it * 5) % 40:(it * 5) % 40 + 16]
        noise = ((torch.randn((16, 3), generator=g) * 0.3).clamp(-0.5, 0.5)).to(dtype)
        caps = torch.rand((16, 7), generator=g).to(dtype)
        pg_o, td_o = O.update_parameters(a, batch, it, noise, caps, champion)
        w = torch.ones(16, dtype=dtype) if it % 2 else None
        pg_p, td_p, delta = P.update_parameters(b, batch, it, noise, caps, champion, weights=w)
        assert torch.equal(td_o, td_p) and (pg_o is None) == (pg_p is None) and (pg_o is None or torch.equal(pg_o, pg_p))
        assert same_learner(a, b), it
        assert delta.shape == (16,) and torch.all(delta >= 0)


def test_torch_td3_weighted_path_is_the_weighted_oracle_bit_for_bit():
    """TD3.update_parameters on a prioritized batch (weights, rows) against the weighted oracle fed the same draws: the
    same parameters, moments, losses and TD errors; the TD errors are those of the critic before its update"""
    from serl_b200.core.td3 import TD3
    torch.manual_seed(4)
    ref = TD3(td3_args())
    ora = copy.deepcopy(ref)
    rows = replay_rows(64, seed=2)
    gw = torch.Generator().manual_seed(9)
    for it in range(1, 8):
        batch = rows[(it * 7) % 40:(it * 7) % 40 + 16]
        w = torch.rand((16, 1), generator=gw) + 0.1
        critic_before = copy.deepcopy(ref.critic)
        torch.manual_seed(100 + it)
        pg_r, td_r, delta_r = ref.update_parameters(O.split(batch) + (w, torch.arange(16)), it)
        torch.manual_seed(100 + it)
        state, action = batch[:, :7], batch[:, 7:10]
        noise = (torch.randn_like(action) * 0.2962183114680794).clamp(-0.5, 0.5)
        caps = torch.rand_like(state) if it % 3 == 0 else None
        pg_o, td_o, delta_o = P.update_parameters(ora, batch, it, noise, caps, weights=w)
        assert td_r == td_o.numpy() and torch.equal(delta_r, delta_o)
        assert (pg_r is None) == (pg_o is None) and (pg_r is None or pg_r == pg_o.numpy())
        assert same_learner(ref, ora), it
        with torch.no_grad():                        # delta is the pre-update critic's
            s, a, s2, r, d = O.split(batch)
            q1, q2 = critic_before(s, a)
            assert not torch.equal(q1, ref.critic(s, a)[0])
    # without weights the torch path returns what it always did
    out = ref.update_parameters(O.split(rows[:16]), 1)
    assert len(out) == 2


# ---- the public interface -----------------------------------------------------------------------------------------------------

def test_sweep_refuses_per_runs_by_name(tmp_path, monkeypatch):
    from serl_b200 import build
    from serl_b200.core import agent as agent_mod
    from serl_b200.parameters import Parameters
    from serl_b200.sweep import Sweep
    build.build()

    def no_agent(*a, **k):
        raise AssertionError('an Agent was built before the runs were checked')
    monkeypatch.setattr(agent_mod, 'Agent', no_agent)
    monkeypatch.chdir(tmp_path)
    runs = []
    for per in (False, True):
        p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=4, mut_type='normal', test_ea=False,
                                             fused_td3=True, per=per))
        p.state_dim, p.action_dim = 7, 3
        runs.append((p, None))
    with pytest.raises(ValueError, match=r'run 1 sets per \(prioritized experience replay\)'):
        Sweep(runs)


def test_train_example_accepts_per(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    spec = importlib.util.spec_from_file_location('train_example', os.path.join(ROOT, 'examples', 'train.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    from serl_b200.parameters import Parameters
    assert Parameters(mod.parser.parse_args(['-frames', '1000', '-per'])).per is True
    assert Parameters(mod.parser.parse_args(['-frames', '1000'])).per is False
