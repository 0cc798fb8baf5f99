"""K7 (csrc/td3.cu) for actors wider than 128, without a GPU: the state size of the wide shapes, the header's bounds of
the wide domain against _native, and the argument checks that reject a shape outside it before any CUDA call."""
import ctypes
import os
import subprocess
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_ARG = -1                  # SERL_ERR_ARG (include/serl_b200.h)


def td3_args(hidden, num_layers, activation='tanh'):
    return types.SimpleNamespace(device='cpu', individual_bs=100, hidden_size=hidden, num_layers=num_layers,
                                 activation_actor=activation, state_dim=7, action_dim=3, lr=1e-3, gamma=0.98, tau=0.005,
                                 noise_sd=0.2, noise_clip=0.5, policy_update_freq=3, use_caps=True, batch_size=86, seed=7)


@pytest.mark.parametrize('hidden', [129, 256, 320])
@pytest.mark.parametrize('num_layers', [1, 3, 8])
def test_wide_state_size_is_the_four_modules_and_their_adam_moments(hidden, num_layers):
    from serl_b200 import build, rollout, td3_fused
    from serl_b200.core.genetic_agent import Actor
    from serl_b200.core.td3 import Critic
    build.build()
    args = td3_args(hidden, num_layers)
    pa = sum(p.numel() for p in Actor(args).parameters())
    pc = sum(p.numel() for p in Critic(args).parameters())
    assert td3_fused.state_floats(rollout.actor_shape(hidden, num_layers)) == 4 * pa + 4 * pc


def test_wide_bounds_match_the_header(tmp_path):
    from serl_b200 import _native
    names = ['SERL_TD3_MAX_HIDDEN', 'SERL_TD3_MAX_WIDE_LAYERS', 'SERL_TD3_MAX_BATCH', 'SERL_TD3_CRITIC_HIDDEN']
    src = tmp_path / 'bounds.c'
    src.write_text('#include <stdio.h>\n#include "serl_td3.h"\nint main(void) {\n' +
                   ''.join('  printf("%%lld\\n", (long long)%s);\n' % n for n in names) + '  return 0;\n}\n')
    exe = tmp_path / 'bounds'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(exe), str(src)])
    out = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert out == [_native.TD3_MAX_HIDDEN, _native.TD3_MAX_WIDE_LAYERS, _native.TD3_MAX_BATCH, _native.TD3_CRITIC_HIDDEN]
    assert (_native.TD3_MAX_HIDDEN, _native.TD3_MAX_WIDE_LAYERS) == (320, 8)


def test_shapes_outside_the_wide_domain_are_rejected_before_any_cuda_call():
    """the descriptor's device pointers are never dereferenced: every case fails with SERL_ERR_ARG in the argument checks"""
    from serl_b200 import build, _native, rollout, td3_fused
    build.build()
    L = _native.lib()

    def run(**kw):
        d = _native.TD3Desc()
        d.shape = rollout.actor_shape(256, 3)
        d.d_state, d.d_replay, d.d_losses = 0x10000, 0x20000, 0x30000          # non-null, never read
        d.replay_cols, d.n_valid, d.batch, d.n_steps, d.policy_update_freq = 19, 1000, 86, 10, 3
        for k, v in kw.items():
            setattr(d, k, v)
        return L.serl_td3_train(ctypes.byref(d), None), L.serl_last_error().decode()

    bad_shapes = [rollout.actor_shape(321, 3), rollout.actor_shape(256, 9), rollout.actor_shape(320, 9),
                  rollout.actor_shape(256, 0), rollout.actor_shape(48, 3), rollout.actor_shape(100, 3),
                  _native.ActorShape(8, 3, 256, 3, 0), _native.ActorShape(7, 4, 256, 3, 0), _native.ActorShape(7, 3, 256, 3, 3)]
    for shape in bad_shapes:
        rc, msg = run(shape=shape)
        assert rc == ERR_ARG and 'shape' in msg, (shape.hidden, shape.num_layers, rc, msg)
        with pytest.raises(_native.NativeError):
            td3_fused.state_floats(shape)
    for kw in (dict(batch=129), dict(batch=0), dict(n_valid=85), dict(replay_cols=18), dict(policy_update_freq=0),
               dict(cluster_size=3), dict(cluster_size=16), dict(flags=2), dict(d_state=None), dict(d_replay=None),
               dict(d_losses=None), dict(n_steps=-1), dict(first_iteration=-1)):
        rc, msg = run(**kw)
        assert rc == ERR_ARG and msg.startswith('serl_td3'), (kw, rc, msg)
    for h, nl in ((129, 1), (256, 3), (320, 8)):
        assert run(shape=rollout.actor_shape(h, nl), n_steps=0)[0] == 0          # accepted; nothing to do, no launch
