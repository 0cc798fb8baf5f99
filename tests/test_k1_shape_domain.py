"""Which kernel flies a uniform actor, pinned at every boundary of K1's shape domain without a GPU: serl_actor_tc_widths
(rollout.tc_widths) and the shapes serl_rollout_run and serl_actor_forward refuse before any CUDA call.

K1's warp kernel keeps the plant tables (51,152 B) next to one genome slot (the genome and the exchange buffers of 4 warps)
in 227 KB of shared memory; h = 128 alone also has an instantiation that reads the tables from global memory.  A genome that
fits neither goes to the one-thread-per-env kernel (the genome and 2 x h x 128 floats), else to K1-TC as [h] * (L + 1)."""
import ctypes

import pytest
import torch

# hidden size -> (deepest L on the warp kernel, deepest L K1 keeps at all: the one-thread-per-env kernel takes h = 32 further)
K1_WARP = {32: (39, 44), 64: (9, 9), 72: (7, 7), 96: (4, 4), 128: (3, 3)}
# the one-thread-per-env kernel alone: hidden size -> deepest L
K1_SIMPLE = {2: 5757, 3: 3183, 8: 636, 31: 47, 33: 41, 50: 16, 100: 3, 101: 2, 127: 1, 129: 1, 141: 1}


def widths(h, L):
    from serl_b200 import rollout
    return rollout.tc_widths(rollout.actor_shape(h, L))


@pytest.mark.parametrize('h', sorted(K1_WARP))
def test_k1_keeps_every_depth_up_to_its_limit_at_a_warp_size(h):
    deepest = K1_WARP[h][1]
    for L in range(deepest + 1):
        assert widths(h, L) is None, (h, L)
    assert widths(h, deepest + 1) == [h] * (deepest + 2)
    assert widths(h, 2 * deepest + 8) == [h] * (2 * deepest + 9)


def test_shapes_trained_on_k7_past_the_warp_kernel_go_to_k1_tc():
    """(96, 5) and (72, 8): the genome fits next to the exchange buffers but not next to the plant tables as well"""
    assert widths(96, 5) == [96] * 6 and widths(96, 6) == [96] * 7
    assert widths(72, 8) == [72] * 9 and widths(72, 10) == [72] * 11
    assert widths(64, 10) == [64] * 11 and widths(64, 13) == [64] * 14          # K1-TC refuses more than 9 widths
    assert widths(128, 4) == [128] * 5


@pytest.mark.parametrize('h', sorted(K1_SIMPLE))
def test_k1_keeps_every_depth_the_one_thread_per_env_kernel_holds(h):
    d = K1_SIMPLE[h]
    assert widths(h, 0) is None and widths(h, d) is None
    assert widths(h, d + 1) == [h] * (d + 2)


def test_l0_and_the_widest_one_layer_actor():
    for h in (2, 3, 32, 72, 128, 141, 142, 200, 255, 256):
        assert widths(h, 0) is None, h               # L = 0 stays with K1, which flies it or reports why it cannot
    assert widths(141, 1) is None and widths(142, 1) == [142, 142]


def _lib():
    from serl_b200 import _native, build
    build.build()
    return _native.lib()


def _rollout_run(h, L):
    """serl_rollout_run of a uniform actor with fake device pointers (never dereferenced when the call is refused first)"""
    from serl_b200 import _native, rollout
    d = _native.RolloutDesc()
    fake = iter(range(0x10000, 0x100000, 0x1000))
    for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_fitness', 'd_status'):
        setattr(d, f, next(fake))
    d.pop, d.shape, d.n_envs, d.horizon = 4, rollout.actor_shape(h, L), 8, 100
    lib = _lib()
    before = lib.serl_launch_count()
    rc = lib.serl_rollout_run(ctypes.byref(d), None)
    assert lib.serl_launch_count() == before
    return rc, lib.serl_last_error().decode()


def _actor_forward(h, L):
    from serl_b200 import rollout
    lib = _lib()
    rc = lib.serl_actor_forward(0x10000, rollout.actor_shape(h, L), 0x20000, 5, 0x30000, None)
    return rc, lib.serl_last_error().decode()


@pytest.mark.parametrize('h,L', [(96, 5), (72, 8), (64, 10), (32, 45), (128, 4), (256, 0), (142, 1)])
def test_rollout_run_refuses_what_no_k1_kernel_holds_before_any_cuda_call(h, L):
    """without widths, serl_rollout_run flies the shape on K1 or refuses it; tc_widths says where it goes instead"""
    rc, msg = _rollout_run(h, L)
    assert rc == -3 and 'shared memory' in msg, (h, L, rc, msg)


@pytest.mark.parametrize('h,L', [(96, 6), (64, 13), (32, 51), (128, 4), (256, 0), (100, 4)])
def test_actor_forward_refuses_what_neither_forward_kernel_holds_before_any_cuda_call(h, L):
    rc, msg = _actor_forward(h, L)
    assert rc == -3 and 'shared memory' in msg, (h, L, rc, msg)


@pytest.mark.skipif(torch.cuda.is_available(), reason='the fake pointers must not reach a device')
@pytest.mark.parametrize('h,L', [(96, 4), (72, 7), (64, 9), (32, 39), (32, 44), (128, 3), (141, 1), (2, 5757)])
def test_the_deepest_shapes_k1_keeps_pass_every_check(h, L):
    """Without a GPU, a shape that passes the checks stops at the first CUDA call (SERL_ERR_CUDA), not at SERL_ERR_UNSUPPORTED"""
    assert _rollout_run(h, L)[0] == -2, (h, L)


@pytest.mark.skipif(torch.cuda.is_available(), reason='the fake pointers must not reach a device')
@pytest.mark.parametrize('h,L', [(96, 5), (64, 12), (32, 50), (72, 10), (128, 3), (100, 3)])
def test_the_deepest_shapes_actor_forward_holds_pass_every_check(h, L):
    assert _actor_forward(h, L)[0] == -2, (h, L)
