"""Checkpoint and resume on the H100 (serl_b200/checkpoint.py): a run saved after 2 generations and loaded into a fresh
Agent, built with the global generators scrambled, continues bit for bit like the uninterrupted run — statistics, genomes,
shared / per-actor / critical buffers, learner state and Adam counts, PER tree, counters, the next front's draws and the
four global generator states — in process, across processes (examples/train.py -checkpoint_every / -resume), in a Sweep,
and on 2 ranks."""
import os
import random
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from serl_b200 import checkpoint
from serl_b200.core import agent as agent_mod
from serl_b200.envs import config
from serl_b200.parameters import Parameters
from serl_b200.sweep import RNGState, Sweep

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make(env_name='PHlab_attitude_nominal', seed=7, pop=4, hidden=32, layers=3, activation='tanh', fused=True, per=False,
         indep=False, prefetch=True, mut='normal', distil=False, frames=10 ** 9, frac=0.02, **extra):
    p = Parameters(types.SimpleNamespace(env=env_name, seed=seed, pop_size=pop, mut_type=mut, fused_td3=fused, per=per,
                                         independent_refs=indep, prefetch_generation=prefetch, use_distil=distil, frames=frames))
    env = config.select_env(env_name)
    p.action_dim, p.state_dim = env.action_space.shape[0], env.observation_space.shape[0]
    p.hidden_size, p.num_layers, p.activation_actor = hidden, layers, activation
    p.learn_start, p.frac_frames_train = 200, frac            # gradient steps from the first generations on, a few per generation
    p.buffer_size = 30_000
    if not pop:                     # Parameters sets these only with a population
        p.num_evals, p.smooth_fitness = p.num_envs, False
    for k, v in extra.items():
        setattr(p, k, v)
    return p, env


def build(p, env):
    env.seed(p.seed)
    torch.manual_seed(p.seed)
    np.random.seed(p.seed)
    random.seed(p.seed)
    return agent_mod.Agent(p, env)


def scramble(k):
    random.seed(1000 + k)
    np.random.seed(2000 + k)
    torch.manual_seed(3000 + k)


def same(a, b):
    """bitwise equality of nested checkpoint values (NaN equal to NaN)"""
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and \
            bool(torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)))
    if isinstance(a, np.ndarray):
        return isinstance(b, np.ndarray) and a.shape == b.shape and a.tobytes() == b.tobytes()
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, (float, np.floating)) and np.isnan(a):
        return isinstance(b, (float, np.floating)) and np.isnan(b)
    return a == b


def diff(a, b, path=''):
    """the first path at which two checkpoint values differ (for the failure message)"""
    if isinstance(a, dict) and isinstance(b, dict):
        for k in a:
            if k not in b or not same(a[k], b[k]):
                return diff(a[k], b.get(k), path + '/' + str(k))
    if isinstance(a, (list, tuple)) and isinstance(b, (list, tuple)) and len(a) == len(b):
        for i, (x, y) in enumerate(zip(a, b)):
            if not same(x, y):
                return diff(x, y, path + '/%d' % i)
    return path


def assert_same_stats(x, y):
    assert len(x) == len(y)
    for s, t in zip(x, y):
        if s is None or t is None:
            assert s is None and t is None
            continue
        assert s.keys() == t.keys()
        for k in s:
            assert same(float(s[k]), float(t[k])), (k, s[k], t[k])


def snapshot(agent, rng=None):
    ck = checkpoint.capture(agent, rng)
    del ck['extra']
    return ck


CASES = {
    'fused': {},
    'torch_td3': dict(fused=False, frac=0.01),
    'per': dict(per=True),
    'independent_refs': dict(indep=True),
    'no_prefetch': dict(prefetch=False),
    'prefetch_speculative': dict(speculative_validations=2),
    'test_ea': dict(frac=0.0),
    'pop0': dict(pop=0),
    'proximal_distil': dict(mut='proximal', distil=True),
    'wide_256': dict(hidden=256),
    'symmetric': dict(env_name='PHlab_symmetric_nominal', fused=False, frac=0.01),
    'incremental': dict(env_name='PHlab_attitude_incremental', fused=False, frac=0.01),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_agent_resume_equals_uninterrupted(case, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    kw = CASES[case]
    full = build(*make(**kw))
    stats_full = [full.train() for _ in range(4)]
    want, want_rng = snapshot(full), RNGState.capture()
    if kw.get('frac', 0.02) > 0:
        assert full.rl_iteration > 0                 # the learner took gradient steps
    del full

    first = build(*make(**kw))
    stats = [first.train() for _ in range(2)]
    path = tmp_path / 'ck' / 'checkpoint.pt'
    first.save_checkpoint(path, extra={'stats': stats[-1]})
    del first
    scramble(1)
    resumed = agent_mod.Agent(*make(**kw))          # initial weights and buffers from scrambled generators
    scramble(2)
    extra = resumed.load_checkpoint(path)
    assert_same_stats([extra['stats']], [stats[-1]])
    stats += [resumed.train() for _ in range(2)]
    got, got_rng = snapshot(resumed), RNGState.capture()

    assert_same_stats(stats, stats_full)
    assert same(got, want), diff(got, want)
    for f in ('py', 'np', 'torch', 'cuda'):
        assert same(getattr(got_rng, f), getattr(want_rng, f)), f
    assert got['counters']['iterations'] == 4


def test_frames_extend_and_per_keeps_the_beta_schedule(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    a = build(*make(per=True, frames=50_000))
    a.train()
    a.save_checkpoint(tmp_path / 'ck.pt')
    b = build(*make(per=True, frames=200_000))
    assert b.replay_buffer.beta_frames == 200_000
    b.load_checkpoint(tmp_path / 'ck.pt')
    assert b.replay_buffer.beta_frames == 50_000 and b.args.num_frames == 200_000
    with pytest.raises(ValueError, match=r'Parameters\.hidden_size'):
        build(*make(per=True, hidden=64)).load_checkpoint(tmp_path / 'ck.pt')


def _train_py(cwd, *flags):
    cmd = [sys.executable, os.path.join(ROOT, 'examples', 'train.py'), '-pop_size', '4', '-hidden_size', '32', '-fused_td3',
           '-learn_start', '200', '-seed', '7', '-checkpoint_every', '1'] + [str(f) for f in flags]
    out = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    return out.stdout


def test_resume_across_processes(tmp_path):
    split, whole = tmp_path / 'split', tmp_path / 'whole'
    split.mkdir()
    whole.mkdir()
    _train_py(split, '-frames', 1)                                        # one generation
    n1 = checkpoint.read(split / 'tmp' / 'checkpoint.pt')['counters']['num_frames']
    frames = 2 * n1                                                       # two or more generations in all
    _train_py(split, '-frames', frames, '-resume', split / 'tmp' / 'checkpoint.pt')
    _train_py(whole, '-frames', frames)
    got, want = (checkpoint.read(d / 'tmp' / 'checkpoint.pt') for d in (split, whole))
    assert got['counters']['iterations'] >= 2 and got['rl']['critic_steps'] > 0
    for k in want:
        assert same(got[k], want[k]), (k, diff(got[k], want[k]))
    for name in ('evo_nets.pkl', 'elite_net.pkl', 'rl_net.pkl'):
        x, y = (torch.load(d / 'tmp' / name, weights_only=True) for d in (split, whole))
        assert same(x, y), name


def _sweep(frames_big=10 ** 9):
    runs = []
    for seed, (h, layers, act), frames in ((7, (72, 3, 'tanh'), frames_big), (8, (72, 3, 'tanh'), 1), (7, (256, 2, 'relu'), frames_big)):
        runs.append(make(seed=seed, hidden=h, layers=layers, activation=act, frames=frames))
    return Sweep(runs, mixed_shapes=True)


def test_sweep_resume_equals_uninterrupted(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    full = _sweep()
    stats_full = [full.train() for _ in range(4)]
    want = [snapshot(r.agent, r.rng) for r in full.runs]
    assert full.runs[1].finished and stats_full[1][1] is None           # run 1 finished after its first generation
    del full

    first = _sweep()
    stats = [first.train() for _ in range(2)]
    first.save_checkpoint(tmp_path / 'sweep')
    del first
    scramble(3)
    resumed = _sweep()
    scramble(4)
    outer = RNGState.capture()
    resumed.load_checkpoint(tmp_path / 'sweep')
    assert resumed.runs[1].finished and not resumed.runs[0].finished
    stats += [resumed.train() for _ in range(2)]
    for s, t in zip(stats, stats_full):
        assert_same_stats(s, t)
    for i, r in enumerate(resumed.runs):
        got = snapshot(r.agent, r.rng)
        assert same(got, want[i]), (i, diff(got, want[i]))
    now = RNGState.capture()                                             # the caller's generators are left alone
    for f in ('py', 'np', 'torch', 'cuda'):
        assert same(getattr(now, f), getattr(outer, f)), f


def _two_rank_resume(rank, world, port, folder, out):
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=rank, world_size=world,
                            device_id=torch.device('cuda', rank))
    os.makedirs(os.path.join(folder, 'rank%d' % rank), exist_ok=True)
    os.chdir(os.path.join(folder, 'rank%d' % rank))
    full = build(*make(pop=5))
    stats_full = [full.train() for _ in range(4)]
    want = snapshot(full)
    del full
    first = build(*make(pop=5))
    stats = [first.train() for _ in range(2)]
    path = os.path.join(folder, 'checkpoint.pt')
    first.save_checkpoint(path)
    del first
    scramble(5 + rank)
    resumed = agent_mod.Agent(*make(pop=5))
    resumed.load_checkpoint(path)
    stats += [resumed.train() for _ in range(2)]
    got = snapshot(resumed)
    ok_stats = all(same({k: float(v) for k, v in s.items()}, {k: float(v) for k, v in t.items()}) for s, t in zip(stats, stats_full))
    out[rank] = (ok_stats, same(got, want), diff(got, want), got['rl']['critic_steps'])
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_rank_resume_equals_uninterrupted(tmp_path):
    import torch.multiprocessing as mp
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_two_rank_resume, args=(2, 29900 + os.getpid() % 2000, str(tmp_path), out), nprocs=2, join=True)
    for rank in range(2):
        ok_stats, ok_state, where, steps = out[rank]
        assert ok_stats and steps > 0
        assert ok_state, where
