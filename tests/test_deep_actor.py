"""Deep width lists and the routing of uniform actors without a GPU: the binding of include/serl_route.h, parameter counts,
which kernel flies a shape (serl_actor_tc_widths) and the K1-TC envelope checks that come before any CUDA call."""
import ctypes
import os
import re

import pytest
import torch

from oracle import actor as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_binding_matches_the_route_header():
    """_native.ROUTE_SIGNATURES against the prototype of include/serl_route.h, which serl_b200.h includes"""
    from serl_b200 import _native
    text = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'serl_route.h')).read(), flags=re.S)
    protos = {n: (r.strip(), [p.strip() for p in ps.split(',')])
              for r, n, ps in re.findall(r'([A-Za-z_][\w ]*\**)\s*\b(serl_[a-z0-9_]+)\s*\(([^)]*)\)\s*;', text)}
    assert sorted(protos) == sorted(_native.ROUTE_SIGNATURES) == ['serl_actor_tc_widths']
    assert '#include "serl_route.h"' in open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    restype, argtypes = _native.ROUTE_SIGNATURES['serl_actor_tc_widths']
    ret, params = protos['serl_actor_tc_widths']
    assert ret == 'int32_t' and restype is ctypes.c_int32
    assert len(params) == len(argtypes) == 3
    assert issubclass(argtypes[0], ctypes._Pointer) and argtypes[1] is ctypes.c_void_p and argtypes[2] is ctypes.c_int32
    from serl_b200 import build
    build.build()
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), 'serl_actor_tc_widths')


@pytest.mark.parametrize('h', [8, 32, 72, 100, 101, 128, 160, 256, 320])
def test_uniform_list_has_the_uniform_actors_parameter_count(h):
    from serl_b200 import rollout
    for L in range(1, 9):
        n = rollout.num_params(rollout.actor_shape(h, L))
        assert rollout.num_params_wide([h] * (L + 1)) == n == A.num_params_wide([h] * (L + 1)) == A.num_params(7, 3, h, L), (h, L)


def test_k1_keeps_the_shapes_it_holds_and_hands_the_rest_to_k1_tc():
    from serl_b200 import rollout
    for h in (32, 50, 64, 72, 96, 100, 128):            # 100: the widest the one-thread-per-env kernel holds at L = 3
        assert rollout.tc_widths(rollout.actor_shape(h, 3)) is None, h
    for h in (101, 108, 160, 256):
        assert rollout.tc_widths(rollout.actor_shape(h, 3)) == [h] * 4, h
    assert rollout.tc_widths(rollout.actor_shape(256, 1)) == [256, 256]
    assert rollout.tc_widths(rollout.actor_shape(141, 1)) is None and rollout.tc_widths(rollout.actor_shape(142, 1)) == [142, 142]
    assert rollout.tc_widths(rollout.actor_shape(200, 8, 'elu')) == [200] * 9
    assert rollout.tc_widths(rollout.actor_shape(256, 0)) is None          # L = 0 keeps K1's rules
    bad = rollout.actor_shape(256, 3)
    bad.state_dim = 9
    assert rollout.tc_widths(bad) is None                                  # K1 reports the shape


def test_query_needs_room_for_the_widths():
    from serl_b200 import _native, rollout
    out = (ctypes.c_int32 * 4)()
    assert _native.lib().serl_actor_tc_widths(rollout.actor_shape(256, 3), out, 3) == -1
    assert _native.lib().serl_actor_tc_widths(rollout.actor_shape(256, 3), out, 4) == 4 and list(out) == [256] * 4


def _run(widths):
    """serl_rollout_run with fake device pointers (never dereferenced: every rejection comes first)"""
    from serl_b200 import _native, build, rollout
    build.build()
    L = _native.lib()
    warr = (ctypes.c_int32 * len(widths))(*widths)
    d = _native.RolloutDesc()
    fake = iter(range(0x10000, 0x100000, 0x1000))
    for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_fitness', 'd_trace', 'd_status'):
        setattr(d, f, next(fake))
    d.pop, d.shape, d.n_envs, d.horizon = 4, rollout.actor_shape(72), 8, 100
    d.widths, d.n_widths = ctypes.cast(warr, ctypes.c_void_p), len(widths)
    return L.serl_rollout_run(ctypes.byref(d), None), L.serl_last_error().decode()


@pytest.mark.parametrize('widths,what', [([64] * 10, '2 to 9 widths'), ([64], '2 to 9 widths'), ([256, 400, 256], 'w_i <= 320'),
                                         ([256, 256, 4], 'w_i <= 320'), ([1100, 64, 64], 'w0 <= 1024'),
                                         ([96, 320, 320, 64], 'shared memory')])
def test_rollout_run_rejects_deep_lists_outside_the_envelope_before_any_cuda_call(widths, what):
    rc, msg = _run(widths)
    assert rc == -3 and what in msg, (rc, msg)


@pytest.mark.skipif(torch.cuda.is_available(), reason='the fake pointers must not reach a device')
@pytest.mark.parametrize('widths', [[256] * 4, [108] * 4, [96, 200, 64, 320], [1024, 256, 256], [64] * 9] +
                         [[h] * (L + 1) for h in (101, 200, 256) for L in (1, 3, 8)])
def test_the_envelope_lists_pass_every_check(widths):
    """Without a GPU, a list that passes the checks stops at the first CUDA call (SERL_ERR_CUDA), not at SERL_ERR_UNSUPPORTED"""
    rc, msg = _run(widths)
    assert rc == -2, (rc, msg)
