"""K7 (csrc/td3.cu) for actors wider than 128, without a GPU: the state size of the wide shapes and the header's bounds of
the wide domain against _native.  serl_td3_learn's refusal of shapes outside it is in test_td3_oracle.py."""
import ctypes
import os
import subprocess
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
