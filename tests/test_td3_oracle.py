"""K7 (the fused TD3 learner, csrc/td3.cu) without a GPU: the explicit-draw oracle (oracle/td3.py) against TD3.update_parameters
bit for bit, the C-ABI of include/serl_td3.h (binding, descriptor layout, constants, state size) and the argument checks
that reject an unsupported learner before any CUDA call."""
import copy
import ctypes
import os
import re
import subprocess
import types

import pytest
import torch

from oracle import td3 as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def td3_args(hidden=32, num_layers=1, activation='tanh', use_caps=True, device='cpu', batch_size=16):
    return types.SimpleNamespace(device=device, individual_bs=100, hidden_size=hidden, num_layers=num_layers,
                                 activation_actor=activation, state_dim=7, action_dim=3, lr=1e-3, gamma=0.98, tau=0.005,
                                 noise_sd=0.2962183114680794, noise_clip=0.5, policy_update_freq=3, use_caps=use_caps,
                                 batch_size=batch_size, seed=7)


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


@pytest.mark.parametrize('use_caps,champion,activation', [(True, False, 'tanh'), (False, False, 'elu'), (True, True, 'relu')])
def test_oracle_replays_td3_update_parameters_bit_for_bit(use_caps, champion, activation):
    """the same generator state fed to TD3 (which draws) and to the oracle (which is given the draws): identical parameters,
    Adam moments and losses over critic-only and actor iterations"""
    from serl_b200.core.td3 import TD3
    torch.manual_seed(3)
    args = td3_args(activation=activation, use_caps=use_caps)
    ref = TD3(args)
    ora = copy.deepcopy(ref)
    rows = replay_rows(64)
    for it in range(1, 8):
        batch = rows[(it * 5) % 40:(it * 5) % 40 + args.batch_size]
        torch.manual_seed(100 + it)
        pg_r, td_r = ref.update_parameters(O.split(batch), it, champion)
        torch.manual_seed(100 + it)
        state, action = batch[:, :7], batch[:, 7:10]
        noise = (torch.randn_like(action) * args.noise_sd).clamp(-args.noise_clip, args.noise_clip)
        caps = torch.rand_like(state) if (use_caps and it % 3 == 0) else None
        pg_o, td_o = O.update_parameters(ora, batch, it, noise, caps, champion)
        assert td_r == td_o.numpy()
        assert (pg_r is None) == (pg_o is None) and (pg_r is None or pg_r == pg_o.numpy())
        assert same_learner(ref, ora), it


def flat_state(agent):
    """the eight blocks of K7's state: each module's parameters, then each optimiser's exp_avg / exp_avg_sq (zero before
    the first step), in float64"""
    out = [torch.cat([p.detach().double().reshape(-1) for p in m.parameters()])
           for m in (agent.actor, agent.actor_target, agent.critic, agent.critic_target)]
    for opt in (agent.actor_optim, agent.critic_optim):
        for key in ('exp_avg', 'exp_avg_sq'):
            out.append(torch.cat([opt.state[p][key].double().reshape(-1) if p in opt.state else torch.zeros(p.numel(), dtype=torch.float64)
                                  for p in opt.param_groups[0]['params']]))
    return out


def test_float64_copy_starts_from_identical_values():
    from serl_b200.core.td3 import TD3
    torch.manual_seed(4)
    args = td3_args()
    ref = TD3(args)
    rows = replay_rows(64)
    for it in range(1, 5):                       # non-empty Adam state in both optimisers, unequal step counts
        O.update_parameters(ref, rows[it:it + args.batch_size], it, torch.zeros(args.batch_size, 3), torch.rand(args.batch_size, 7))
    d = O.as_float64(ref)
    assert all(p.dtype == torch.float64 for m in (d.actor, d.actor_target, d.critic, d.critic_target) for p in m.parameters())
    for a, b in zip(flat_state(ref), flat_state(d)):
        assert torch.equal(a, b)
    for oa, ob in ((ref.actor_optim, d.actor_optim), (ref.critic_optim, d.critic_optim)):
        assert ob.defaults['lr'] == oa.defaults['lr']
        for pa, pb in zip(oa.param_groups[0]['params'], ob.param_groups[0]['params']):
            assert ob.state[pb]['exp_avg'].dtype == torch.float64 and ob.state[pb]['step'] == oa.state[pa]['step']
    assert int(d.critic_optim.state[d.critic.q1[0].weight]['step']) == 4 and int(d.actor_optim.state[d.actor.net[0].weight]['step']) == 1
    # the copy is independent of the original, its Adam step counts included
    O.update_parameters(d, rows[:args.batch_size].double(), 5, torch.zeros(args.batch_size, 3, dtype=torch.float64))
    assert int(d.critic_optim.state[d.critic.q1[0].weight]['step']) == 5 and int(ref.critic_optim.state[ref.critic.q1[0].weight]['step']) == 4
    assert not torch.equal(ref.critic.q1[0].weight.double(), d.critic.q1[0].weight)


@pytest.mark.parametrize('reward_scale', [1.0, 30.0])
def test_float64_copy_tracks_the_float32_oracle_over_300_steps(reward_scale):
    """h = 72, L = 3, B = 86, CAPS: the fp32 oracle and its fp64 copy fed the same draws.  Measured (rewards x 30, the
    critic clipped at every step, in brackets): td loss within 3.2e-7 (2.5e-7) relative at every step, the four modules'
    parameters within 1.1e-5 (5.3e-6) of their displacement, no element further than 8.9e-3 (9.5e-3) lr.  Bounds: about
    twice those."""
    from serl_b200.core.td3 import TD3
    torch.manual_seed(11)
    args = td3_args(72, 3, batch_size=86)
    args.lr = 0.00018643512599969097
    t32 = TD3(args)
    t64 = O.as_float64(t32)
    p0 = torch.cat(flat_state(t32)[:4])
    gr = torch.Generator().manual_seed(5)
    rows = torch.randn((3000, 19), generator=gr) * 0.3
    rows[:, 7:10] = torch.rand((3000, 3), generator=gr) * 2 - 1
    rows[:, 17] = -torch.rand(3000, generator=gr) * reward_scale
    rows[:, 18] = (torch.rand(3000, generator=gr) < 0.05).float()
    g = torch.Generator().manual_seed(1)
    td_rel, clipped = 0.0, 0
    for it in range(1, 301):
        idx = torch.randperm(3000, generator=g)[:86]
        noise = (torch.randn(86, 3, generator=g) * args.noise_sd).clamp(-args.noise_clip, args.noise_clip)
        caps = torch.rand(86, 7, generator=g)
        norms = []
        _, td = O.update_parameters(t32, rows[idx], it, noise, caps, norms=norms)
        _, td6 = O.update_parameters(t64, rows[idx].double(), it, noise.double(), caps.double())
        td_rel = max(td_rel, abs(float(td) - float(td6)) / abs(float(td6)))
        clipped += norms[0] > 10
    p32, p64 = torch.cat(flat_state(t32)[:4]), torch.cat(flat_state(t64)[:4])
    err = float((p32 - p64).norm() / (p64 - p0).norm())
    worst = float((p32 - p64).abs().max() / args.lr)
    print('reward x %g: td rel %.2e, param err %.2e of the displacement, max %.2e lr, critic clipped on %d steps'
          % (reward_scale, td_rel, err, worst, clipped))
    assert clipped == (300 if reward_scale > 1 else 0)
    assert td_rel <= 6e-7 and err <= 2.5e-5 and worst <= 2e-2


def header_text(name):
    return re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', name)).read(), flags=re.S)


def test_binding_matches_the_td3_header():
    """_native.TD3_SIGNATURES against the prototypes of include/serl_td3.h (pointer / integer kinds and arity)"""
    from serl_b200 import _native
    protos = {n: [p.strip() for p in ps.split(',')]
              for _, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', header_text('serl_td3.h'))}
    assert sorted(protos) == sorted(_native.TD3_SIGNATURES) == ['serl_td3_state_floats', 'serl_td3_train']
    assert '#include "serl_td3.h"' in open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    for name, params in protos.items():
        restype, argtypes = _native.TD3_SIGNATURES[name]
        assert len(argtypes) == len(params)
        for decl, t in zip(params, argtypes):
            assert ('*' in decl) == (t is ctypes.c_void_p or issubclass(t, ctypes._Pointer)), (name, decl)
    assert _native.TD3_SIGNATURES['serl_td3_state_floats'][0] is ctypes.c_int64
    assert _native.TD3_SIGNATURES['serl_td3_train'][0] is ctypes.c_int


def test_ctypes_mirror_of_the_td3_descriptor_matches_the_header(tmp_path):
    """serl_b200/_native.py TD3Desc vs include/serl_td3.h: same size and field offsets (gcc offsetof), same constants"""
    from serl_b200 import _native
    fields = [f for f, _ in _native.TD3Desc._fields_]
    names = ['SERL_TD3_CRITIC_HIDDEN', 'SERL_TD3_MAX_BATCH', 'SERL_TD3_CHAMPION_TARGET', 'SERL_TD3_STATUS_INDEX']
    src = tmp_path / 'layout.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "serl_td3.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(serl_td3_desc));\n' +
                   ''.join('  printf("%%zu\\n", offsetof(serl_td3_desc, %s));\n' % f for f in fields) +
                   ''.join('  printf("%%lld\\n", (long long)%s);\n' % n for n in names) + '  return 0;\n}\n')
    exe = tmp_path / 'layout'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert out[0] == ctypes.sizeof(_native.TD3Desc)
    assert out[1:1 + len(fields)] == [getattr(_native.TD3Desc, f).offset for f in fields]
    assert out[1 + len(fields):] == [_native.TD3_CRITIC_HIDDEN, _native.TD3_MAX_BATCH, _native.TD3_CHAMPION_TARGET,
                                     _native.TD3_STATUS_INDEX]


def test_state_size_is_the_four_modules_and_their_adam_moments():
    from serl_b200 import build, rollout, td3_fused
    from serl_b200.core.genetic_agent import Actor
    from serl_b200.core.td3 import Critic
    build.build()
    for h, L, act in ((72, 3, 'tanh'), (32, 1, 'elu'), (128, 5, 'relu')):
        args = td3_args(h, L, act)
        pa = sum(p.numel() for p in Actor(args).parameters())
        pc = sum(p.numel() for p in Critic(args).parameters())
        assert td3_fused.state_floats(rollout.actor_shape(h, L, act)) == 4 * pa + 4 * pc
    assert td3_fused.state_floats(rollout.actor_shape(72)) * 4 == 437_840       # 438 KB at h = 72, L = 3


def test_unsupported_learner_is_rejected_before_any_cuda_call():
    """bad shapes, batch sizes and launch parameters fail with SERL_ERR_ARG; the device pointers are never dereferenced"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()

    def run(**kw):
        d = _native.TD3Desc()
        d.shape = rollout.actor_shape(72)
        d.d_state, d.d_replay, d.d_losses = 0x10000, 0x20000, 0x30000          # non-null, never read
        d.replay_cols, d.n_valid, d.batch, d.n_steps, d.policy_update_freq = 19, 1000, 86, 10, 3
        for k, v in kw.items():
            setattr(d, k, v)
        return L.serl_td3_train(ctypes.byref(d), None), L.serl_last_error().decode()

    for kw in (dict(shape=rollout.actor_shape(48)), dict(shape=rollout.actor_shape(72, 0)), dict(shape=_native.ActorShape(8, 3, 72, 3, 0)),
               dict(shape=_native.ActorShape(7, 3, 72, 3, 3)), dict(batch=129), dict(batch=0), dict(n_valid=85), dict(replay_cols=18),
               dict(policy_update_freq=0), dict(cluster_size=3), dict(cluster_size=16), dict(flags=2), dict(d_state=None)):
        rc, msg = run(**kw)
        assert rc == -1 and msg.startswith('serl_td3'), (kw, rc, msg)
    assert 'batch' in run(batch=129)[1] and 'shape' in run(shape=rollout.actor_shape(48))[1]
    assert run(n_steps=0)[0] == 0                         # nothing to do: no launch
    with pytest.raises(_native.NativeError):
        from serl_b200 import td3_fused
        td3_fused.state_floats(rollout.actor_shape(100))
