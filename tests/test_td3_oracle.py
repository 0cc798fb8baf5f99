"""K7 (the fused TD3 learner, csrc/td3.cu) without a GPU: the explicit-draw oracle (oracle/td3.py) against TD3.update_parameters
bit for bit, and the C-ABI of include/serl_td3.h and serl_td3_per.h: the binding, the descriptor layouts, the constants, the
state size, and the checks with which serl_td3_learn refuses a learner or a call before any CUDA call."""
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


def prototypes(name):
    return {n: (r.strip(), [p.strip() for p in ps.split(',')])
            for r, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', header_text(name))}


def test_binding_matches_the_learn_prototype():
    """_native.TD3_SIGNATURES against the prototypes of include/serl_td3.h (return, pointer and integer kinds, arity), the
    headers serl_b200.h includes, and a library that exports no other K7 entry point"""
    from serl_b200 import _native
    kinds = {'int': ctypes.c_int32, 'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64}
    protos = prototypes('serl_td3.h')
    assert sorted(protos) == sorted(_native.TD3_SIGNATURES) == ['serl_td3_learn', 'serl_td3_state_floats']
    for name, (ret, params) in protos.items():
        restype, argtypes = _native.TD3_SIGNATURES[name]
        assert kinds[ret] is restype, name
        assert len(argtypes) == len(params), name
        for decl, t in zip(params, argtypes):
            assert ('*' in decl) == (t is ctypes.c_void_p or issubclass(t, ctypes._Pointer)), (name, decl)
            if '*' not in decl:
                assert kinds[decl.split()[0]] is t, (name, decl)
    text = open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    assert all('#include "%s"' % h in text for h in ('serl_td3.h', 'serl_td3_per.h', 'serl_route.h'))
    from serl_b200 import build
    build.build()
    syms = subprocess.check_output(['nm', '-D', '--defined-only', _native.LIB_PATH], text=True).split()
    assert sorted(x for x in syms if x.startswith('serl_td3_')) == ['serl_td3_learn', 'serl_td3_state_floats']


def test_learn_takes_per_descriptors():
    """serl_td3_learn's parameters, declared and bound: the learners, their per descriptors, their count and the stream"""
    from serl_b200 import _native
    ret, params = prototypes('serl_td3.h')['serl_td3_learn']
    assert ret == 'int' and params == ['const serl_td3_desc* descs', 'const serl_td3_per_desc* pers', 'int n', 'void* stream']
    restype, argtypes = _native.TD3_SIGNATURES['serl_td3_learn']
    assert restype is ctypes.c_int and len(argtypes) == 4
    assert argtypes[0]._type_ is _native.TD3Desc and argtypes[1]._type_ is _native.TD3PerDesc
    assert argtypes[2] is ctypes.c_int32 and argtypes[3] is ctypes.c_void_p


def test_max_group_matches_the_header(tmp_path):
    from serl_b200 import _native
    src = tmp_path / 'c.c'
    src.write_text('#include "serl_b200.h"\n'
                   'int (*f)(const serl_td3_desc*, const serl_td3_per_desc*, int, void*) = serl_td3_learn;\n')
    out = subprocess.check_output(['gcc', '-E', '-dM', '-I', os.path.join(ROOT, 'include'), str(src)], text=True)
    assert '#define SERL_TD3_MAX_GROUP %d' % _native.TD3_MAX_GROUP in out
    assert _native.TD3_MAX_GROUP == 64


def test_k7_headers_compile_alone_in_any_order(tmp_path):
    """serl_b200.h, serl_td3.h and serl_td3_per.h each declare all of K7 on their own, whichever is included first"""
    src = tmp_path / 'c.c'
    for first in ('serl_b200.h', 'serl_td3.h', 'serl_td3_per.h', 'serl_route.h'):
        for second in ('', 'serl_b200.h', 'serl_td3.h', 'serl_td3_per.h'):
            src.write_text('#include "%s"\n' % first + ('#include "%s"\n' % second if second else '') +
                           'int (*f)(const serl_td3_desc*, const serl_td3_per_desc*, int, void*) = serl_td3_learn;\n'
                           'int64_t (*g)(int32_t) = serl_per_tree_doubles;\nint m = SERL_TD3_MAX_GROUP;\n')
            subprocess.check_call(['gcc', '-fsyntax-only', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), str(src)])



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
    p.d_tree, p.capacity, p.n_valid = tree, 2000, 1000                    # non-null, never read
    p.alpha, p.beta0, p.beta_frames = 0.6, 0.4, 1e5
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def learn(descs, pers=None, n=None):
    """serl_td3_learn on the given descriptors (and per descriptors, or NULL): (status, serl_last_error)"""
    from serl_b200 import _native
    a = (_native.TD3Desc * max(len(descs), 1))(*descs)
    b = None if pers is None else (_native.TD3PerDesc * max(len(pers), 1))(*pers)
    rc = _native.lib().serl_td3_learn(a, b, len(descs) if n is None else n, None)
    return rc, _native.lib().serl_last_error().decode()


def _group():
    """a prioritized narrow learner, a uniform narrow one and a prioritized wide one, all valid"""
    from serl_b200 import rollout
    shapes = [rollout.actor_shape(32, 1, 'tanh'), rollout.actor_shape(72, 3, 'elu'), rollout.actor_shape(256, 3, 'relu')]
    return shapes, [_desc(s, seed=k) for k, s in enumerate(shapes)], [_per(), _per(tree=None), _per()]


def _bad_shapes():
    from serl_b200 import _native, rollout
    return [rollout.actor_shape(48), rollout.actor_shape(100, 3), rollout.actor_shape(72, 0), rollout.actor_shape(400, 3),
            rollout.actor_shape(256, 9), rollout.actor_shape(72, 3, 'tanh', state_dim=6), _native.ActorShape(8, 3, 72, 3, 0),
            _native.ActorShape(7, 3, 72, 3, 3)]


def _bad_fields():
    return [dict(batch=129), dict(batch=0), dict(n_valid=85), dict(replay_cols=18), dict(policy_update_freq=0),
            dict(cluster_size=3), dict(cluster_size=16), dict(flags=2), dict(d_state=None), dict(d_replay=None),
            dict(d_losses=None), dict(n_steps=-1), dict(first_iteration=-1), dict(critic_adam_steps=-1),
            dict(actor_adam_steps=-1)]


def test_unsupported_learner_is_refused_alone():
    """bad shapes, batch sizes and launch parameters of one learner (n = 1) fail with SERL_ERR_ARG; the device pointers are
    never dereferenced"""
    from serl_b200 import build, _native, rollout, td3_fused
    build.build()
    before = _native.lib().serl_launch_count()
    for shape in _bad_shapes():
        rc, msg = learn([_desc(shape)])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 0: unsupported actor shape'), (shape.hidden, msg)
        with pytest.raises(_native.NativeError):
            td3_fused.state_floats(shape)
    for kw in _bad_fields():
        rc, msg = learn([_desc(**kw)])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 0: '), (kw, rc, msg)
    assert 'batch' in learn([_desc(batch=129)])[1]
    assert _native.lib().serl_launch_count() == before
    assert learn([_desc(n_steps=0)])[0] == 0                  # nothing to do: no launch
    with pytest.raises(_native.NativeError):
        td3_fused.state_floats(rollout.actor_shape(100))


def test_shapes_outside_the_wide_domain_are_refused():
    from serl_b200 import build, _native, rollout, td3_fused
    build.build()
    bad = [rollout.actor_shape(321, 3), rollout.actor_shape(256, 9), rollout.actor_shape(320, 9), rollout.actor_shape(256, 0),
           _native.ActorShape(8, 3, 256, 3, 0), _native.ActorShape(7, 4, 256, 3, 0), _native.ActorShape(7, 3, 256, 3, 3)]
    for shape in bad:
        rc, msg = learn([_desc(shape)])
        assert rc == -1 and 'shape' in msg, (shape.hidden, shape.num_layers, rc, msg)
        with pytest.raises(_native.NativeError):
            td3_fused.state_floats(shape)
    for kw in _bad_fields():
        rc, msg = learn([_desc(rollout.actor_shape(256, 3), **kw)])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 0: '), (kw, rc, msg)
    for h, nl in ((129, 1), (256, 3), (320, 8)):
        assert learn([_desc(rollout.actor_shape(h, nl), n_steps=0)])[0] == 0          # accepted; nothing to do, no launch


def test_refusals_keep_their_messages():
    from serl_b200 import build
    build.build()
    assert learn([_desc(batch=129)]) == (-1, 'serl_td3_learn: learner 0: batch must be 1..128')
    assert learn([_desc(cluster_size=3)]) == (-1, 'serl_td3_learn: learner 0: cluster_size must be 0, 1, 2, 4 or 8')
    assert learn([_desc()], [_per(alpha=0.0)]) == (-1, 'serl_td3_learn: learner 0: alpha must be in (0, 1]')
    assert learn([_desc(), _desc(cluster_size=4)]) == (-1, "serl_td3_learn: learner 1: cluster_size differs from learner 0's")


def test_call_is_refused_before_any_cuda_call():
    """the call's own checks, and every check of a learner made for each learner of a group, naming it"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    before = L.serl_launch_count()
    ok = [_desc(seed=s) for s in range(3)]
    assert L.serl_td3_learn(None, None, 2, None) == -1
    assert L.serl_last_error().decode() == 'serl_td3_learn: null descriptors'
    assert learn(ok, None, 0) == (-1, 'serl_td3_learn: n must be 1..SERL_TD3_MAX_GROUP (64)')
    assert learn([_desc()] * (_native.TD3_MAX_GROUP + 1)) == (-1, 'serl_td3_learn: n must be 1..SERL_TD3_MAX_GROUP (64)')
    rc, msg = learn(ok[:1] + [_desc(cluster_size=4)])
    assert rc == -1 and 'learner 1' in msg and 'cluster_size' in msg
    for kw in _bad_fields() + [dict(shape=s) for s in _bad_shapes()]:
        rc, msg = learn(ok[:1] + [_desc(**kw)] + ok[1:])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 1:'), (kw, rc, msg)
    rc, msg = learn([_desc(rollout.actor_shape(100))] * 2)
    assert rc == -1 and 'learner 0' in msg and 'shape' in msg
    # the same shape everywhere, cluster_size 0 and 8 agreeing, and nothing to do: no launch
    assert learn([_desc(n_steps=0, cluster_size=c) for c in (0, 8, 0)])[0] == 0
    assert L.serl_launch_count() == before


def test_learner_is_refused_at_every_place_of_a_mixed_group():
    """narrow and wide, prioritized and uniform learners: a bad learner anywhere is named, with or without per descriptors,
    and nothing is launched"""
    from serl_b200 import build, _native
    build.build()
    before = _native.lib().serl_launch_count()
    shapes, ok, pers = _group()
    for kw in _bad_fields() + [dict(shape=s) for s in _bad_shapes()]:
        for i in range(3):                  # learners 0 and 2 are prioritized, learner 1 uniform
            descs = list(ok)
            descs[i] = _desc(**dict(dict(shape=shapes[i]), **kw))
            for p in (pers, None):
                rc, msg = learn(descs, p)
                assert rc == -1 and msg.startswith('serl_td3_learn: learner %d: ' % i), (kw, i, rc, msg)
    rc, msg = learn(ok[:2] + [_desc(shapes[2], cluster_size=4)], pers)
    assert (rc, msg) == (-1, "serl_td3_learn: learner 2: cluster_size differs from learner 0's")
    assert _native.lib().serl_launch_count() == before


def test_mixed_learners_without_steps_make_no_launch():
    from serl_b200 import build, _native
    build.build()
    before = _native.lib().serl_launch_count()
    shapes, _, _ = _group()
    # different shapes, both hidden classes, cluster_size 0 and 8 agreeing, and nothing to do
    assert learn([_desc(s, n_steps=0, cluster_size=c) for s, c in zip(shapes, (0, 8, 0))])[0] == 0
    assert _native.lib().serl_launch_count() == before


def test_bad_per_learner_is_refused_alone():
    """every check of prioritized replay for one learner with a tree, naming the field"""
    from serl_b200 import build, _native
    build.build()
    before = _native.lib().serl_launch_count()
    for kw, word in _per_cases():
        rc, msg = learn([_desc()], [_per(**kw)])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 0: ') and word in msg, (kw, rc, msg)
    for kw in (dict(batch=129), dict(cluster_size=3), dict(d_state=None)):
        rc, msg = learn([_desc(**kw)], [_per()])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 0: '), (kw, msg)
    assert _native.lib().serl_launch_count() == before
    assert learn([_desc(n_steps=0)], [_per()])[0] == 0                  # nothing to do: no launch


def _per_cases():
    return ((dict(alpha=0.0), 'alpha'), (dict(alpha=1.5), 'alpha'), (dict(alpha=float('nan')), 'alpha'),
            (dict(beta0=-0.1), 'beta0'), (dict(beta0=1.1), 'beta0'), (dict(beta_frames=0.0), 'beta_frames'),
            (dict(beta_frames=float('nan')), 'beta_frames'), (dict(capacity=999, n_valid=1000), 'n_valid'),
            (dict(n_valid=999), 'n_valid'), (dict(capacity=0), 'capacity'), (dict(capacity=(1 << 30) + 1), 'capacity'))


def test_bad_per_learner_is_refused_in_a_group():
    """every check of a learner, for a prioritized and a uniform one, and every check of prioritized replay for a learner
    with a tree in a group; a learner without a tree does not read the rest of its per descriptor"""
    from serl_b200 import build, _native
    build.build()
    before = _native.lib().serl_launch_count()
    shapes, ok, pers = _group()
    for kw in _bad_fields():
        for j in (0, 1):                  # learner 0 is prioritized, learner 1 uniform
            descs = list(ok)
            descs[j] = _desc(shapes[j], **kw)
            rc, msg = learn(descs, pers)
            assert rc == -1 and msg.startswith('serl_td3_learn: learner %d:' % j), (kw, j, rc, msg)
    for kw, word in _per_cases():
        rc, msg = learn(ok, pers[:2] + [_per(**kw)])
        assert rc == -1 and msg.startswith('serl_td3_learn: learner 2: ') and word in msg, (kw, rc, msg)
        # ...which a learner without a tree ignores
        assert learn([_desc(s, n_steps=0) for s in shapes], pers[:2] + [_per(tree=None, **kw)])[0] == 0, kw
    assert _native.lib().serl_launch_count() == before


def test_prioritized_and_uniform_learners_without_steps_make_no_launch():
    """prioritized and uniform, narrow and wide learners (cluster_size 0 and 8 agreeing) with nothing to do are accepted
    and launch nothing, with per descriptors, without, and one by one"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    before = L.serl_launch_count()
    shapes = [rollout.actor_shape(72), rollout.actor_shape(256), rollout.actor_shape(72, 2), rollout.actor_shape(320, 8),
              rollout.actor_shape(129, 1), rollout.actor_shape(32, 1, 'elu')]
    descs = [_desc(s, n_steps=0, cluster_size=c) for s, c in zip(shapes, (0, 8, 0, 8, 0, 8))]
    per_descs = [_per(), _per(tree=None), _per(tree=None), _per(), _per(), _per(tree=None)]
    assert learn(descs, per_descs)[0] == 0
    assert learn(descs)[0] == 0
    for d, p in zip(descs, per_descs):
        assert learn([d], [p])[0] == 0 and learn([d])[0] == 0
    assert L.serl_launch_count() == before
