"""Symmetric control (the reference's PHlab_symmetric_<mode>) without a GPU: the oracle's restatement on the reference's own
binary, the env mirror's name grammar and spaces, the 2 -> 1 actor's parameter count, the replay layout of 8 columns, the
symmetric reference parameters, the launch checks of SERL_ROLLOUT_SYMMETRIC, and the refusals of the paths that do not fly it."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import actor as A, build as OB, refsig

from symmetric_oracle import SymmetricCitationEnv, KernelOrderActor, run_episode  # noqa: E402  (tests/ on sys.path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def genome(hidden, activation, seed, scale=1.0):
    torch.manual_seed(seed)
    g = A.flatten(A.Actor(state_dim=2, action_dim=1, hidden=hidden, num_layers=3, activation=activation))
    return (g * np.float32(scale)).astype(np.float32)


# ---- the oracle: the reference binary and the C restatement agree bit for bit under symmetric control -------------------
@pytest.mark.refbin
@pytest.mark.skipif(not OB.have_ref(), reason='needs the reference plant binaries under oracle/_ref')
@pytest.mark.parametrize('policy,mode', [('tanh', 'nominal'), ('elu', 'se'), ('relu', 'be'), ('saturating', 'nominal'), ('saturating', 'se')])
def test_symmetric_env_on_the_reference_binary_equals_the_c_restatement(policy, mode):
    """300-step closed loops of random 2 -> 1 actors (and an open loop of full elevator commands past the input limits) on
    both plant back-ends: every step's state, command, reward and observation is identical"""
    lv, st = refsig.make_ref_params(1, seed_base=41)
    actions = None
    if policy == 'saturating':
        rs = np.random.RandomState(5)
        actions = np.repeat(np.sign(rs.randn(10, 1)), 30, axis=0).astype(np.float32)        # +-10 deg held for 0.3 s
        actor = None
    else:
        actor = KernelOrderActor(genome(72, policy, 3, scale=3.0), 72, activation=policy)
    out = {}
    for backend in ('ref', 'port'):
        env = SymmetricCitationEnv(mode, backend)
        out[backend] = run_episode(env, actor, lv[0], st[0], horizon=300, actions=actions)
    a, b = out['ref'], out['port']
    assert a['steps'] == b['steps'] and a['ret'] == b['ret']
    assert np.array_equal(a['rows'].view(np.uint32), b['rows'].view(np.uint32))
    assert np.array_equal(a['u'], b['u'])
    if policy == 'saturating':
        assert np.abs(a['u']).max() == np.deg2rad(10)


def test_symmetric_oracle_observes_theta_error_and_q():
    from serl_b200 import refsig as R
    env = SymmetricCitationEnv('nominal', 'port')
    lv, st = R.make_ref_params(1, seed_base=2, symmetric=True)
    acts = np.tile(np.float32([0.3]), (40, 1))
    r = run_episode(env, None, lv[0], st[0], horizon=40, actions=acts)
    assert r['rows'].shape == (40, 8)
    assert r['rows'][0, 0] == 0.0                                                  # reset(): error 0
    assert np.all(r['rows'][:, 7] == 0.0) and np.all(r['rows'][:, 6] == 0.0)
    assert np.array_equal(r['rows'][1:, 0:2], r['rows'][:-1, 3:5])                 # obs_{k+1} = next_obs_k
    assert np.all(r['rows'][:, 5] <= 0.0) and np.all(r['rows'][:, 5] >= -1.0)      # one clipped term over error.shape[0] = 1


# ---- env mirror: name grammar and spaces ---------------------------------------------------------------------------------
@pytest.mark.parametrize('name,mode', [('PHlab_symmetric_nominal', 'nominal'), ('PHlab_symmetric_be', 'be'), ('phlab_symmetric_se', 'se'),
                                       ('PHlab_longsymmetric_ice', 'ice')])
def test_any_configuration_containing_symmetric_flies_the_elevator_alone(name, mode):
    from serl_b200 import rollout
    from serl_b200.envs import config
    env = config.select_env(name)
    assert env.symmetric and not env.incremental and env.mode == mode and env.mode_code == rollout.mode_code(mode)
    assert env.n_actions == 1 and env.obs_idx == [1] and env.n_obs == 2 and env.observation_space.shape == (2,)
    assert np.array_equal(env.action_space.high, np.deg2rad(10) * np.ones(1)) and env.action_space.shape == (1,)
    assert np.array_equal(env.error_scaler, 6 / np.pi * np.array([1.])) and env.theta_trim == 0.22


@pytest.mark.parametrize('name,match', [('PHlab_symmetric_incremental', 'symmetric control with incremental'),
                                        ('PHlab_symmetric_gust-incremental', 'symmetric control with incremental'),
                                        ('PHlab_fullstate_nominal', 'full-state'), ('PHlab_full_nominal', 'full-state')])
def test_symmetric_incremental_and_full_state_are_refused(name, match):
    from serl_b200.envs import config
    with pytest.raises(ValueError, match=match):
        config.select_env(name)


def test_the_mirror_draws_the_theta_reference_alone():
    from serl_b200.envs import config
    env = config.select_env('PHlab_symmetric_nominal')
    np.random.seed(3)
    lv, st = env.draw_reference()
    np.random.seed(3)
    grid = np.linspace(-30, 30, 10)
    want = grid[np.random.randint(0, 10, size=6)]
    want[0] = 0.0
    assert np.array_equal(lv[0], want) and np.array_equal(st[0], 4.0 * np.arange(6)) and not lv[1].any() and not st[1].any()


def test_symmetric_reference_parameters():
    from serl_b200 import refsig as R
    assert R.widths(20, symmetric=True) == (4.0, 2.0, 0.0)
    assert R.widths(80, symmetric=True) == (16.0, 11.0, 0.0)
    assert R.widths(20) == (4.0, 3.0, 0.04)                                       # the attitude mode's are unchanged
    lv, st = R.make_ref_params(3, symmetric=True)
    assert not lv[:, 1].any() and not st[:, 1].any()
    assert np.array_equal(st[:, 0], np.tile(4.0 * np.arange(6), (3, 1)))          # no timing jitter


def test_parameter_count_of_the_two_input_one_output_actor():
    from serl_b200 import evo, rollout
    for h in (32, 64, 72, 96, 128, 256):
        sh = rollout.actor_shape(h, 3, 'tanh', state_dim=2, action_dim=1)
        assert rollout.is_symmetric(sh)
        P = rollout.num_params(sh)
        assert P == len(A.flatten(A.Actor(state_dim=2, action_dim=1, hidden=h, num_layers=3))) == 3 * h * h + 13 * h + 1
        table, Pt = evo.param_table(2, 1, h, 3)
        assert Pt == P and table[0] == (0, h, 2)
    for widths in ([400, 300], [256] * 4, [128, 256, 64]):
        assert rollout.num_params_wide(widths, 2, 1) == len(A.flatten(A.WideActor(widths, state_dim=2, action_dim=1)))


# ---- replay layout ---------------------------------------------------------------------------------------------------------
def test_replay_layout_of_symmetric_control(tmp_path):
    from serl_b200 import _native, rollout
    from serl_b200.core.replay_memory import DeviceReplayMemory, PopulationBuffers, ActorBuffer
    assert rollout.replay_dims(2, 1) == (2, 1, 2, 1, 1, 1) and rollout.replay_cols(2, 1) == 8 and rollout.transition_cols(2, 1) == 7
    assert rollout.replay_cols(7) == 20 and rollout.replay_cols(10) == 26
    src = tmp_path / 'cols.c'
    src.write_text('#include <stdio.h>\n#include "serl_b200.h"\nint main(void) { printf("%d %d %d %d %d %d\\n", SERL_REPLAY_COLS_SA(2, 1), '
                   'SERL_REPLAY_COLS_SA(7, 3), SERL_REPLAY_COLS_OF(7), SERL_REPLAY_COLS_OF(10), SERL_REPLAY_COLS, SERL_ROLLOUT_SYMMETRIC); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(tmp_path / 'cols'), str(src)])
    assert subprocess.check_output([str(tmp_path / 'cols')], text=True).split() == ['8', '20', '20', '26', '20', str(_native.ROLLOUT_SYMMETRIC)]
    rows = torch.arange(6 * 8, dtype=torch.float32).reshape(6, 8)
    mem = DeviceReplayMemory(4, 'cpu', state_dim=2, action_dim=1)
    mem.add_rows(rows)
    assert len(mem) == 4 and mem.data.shape == (4, 7)
    s, a, s2, r, d = mem.sample(3)
    assert (s.shape, a.shape, s2.shape, r.shape, d.shape) == ((3, 2), (3, 1), (3, 2), (3, 1), (3, 1))
    assert torch.equal(a[:, 0] - s[:, 0], torch.full((3,), 2.0)) and torch.equal(s2[:, 0] - s[:, 0], torch.full((3,), 3.0))
    assert torch.equal(r[:, 0] - s[:, 0], torch.full((3,), 5.0)) and torch.equal(d[:, 0] - s[:, 0], torch.full((3,), 6.0))
    pb = PopulationBuffers(2, 8, 'cpu', state_dim=2, action_dim=1)
    pb.append(torch.tensor([1]), rows[None], torch.ones((1, 6), dtype=torch.bool))
    assert torch.equal(pb.rows_of(1), rows[:, :7])
    latest = ActorBuffer(pb, 1).get_latest(2)
    assert len(latest) == 2 and latest[-1].state.shape == (1, 2) and latest[-1].action.shape == (1, 1)


# ---- launch checks (no CUDA call) --------------------------------------------------------------------------------------------
def test_rollout_run_checks_the_symmetric_flag_before_any_cuda_call():
    from serl_b200 import _native, build
    build.build()
    L = _native.lib()
    warr = (ctypes.c_int32 * 2)(128, 128)
    SYM = _native.ROLLOUT_SYMMETRIC

    def run(state_dim=2, action_dim=1, flags=SYM, **kw):
        d = _native.RolloutDesc()
        fake = iter(range(0x10000, 0x100000, 0x1000))      # non-null, never read
        for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_fitness', 'd_replay', 'd_status'):
            setattr(d, f, next(fake))
        d.pop, d.shape, d.n_envs, d.horizon, d.replay_env, d.flags = 4, _native.ActorShape(state_dim, action_dim, 72, 3, 0), 8, 100, 0, flags
        d.t_max, d.smooth_width = 20.0, 2.0
        for k, v in kw.items():
            setattr(d, k, v)
        return L.serl_rollout_run(ctypes.byref(d), None), L.serl_last_error().decode()

    cases = [dict(state_dim=7, action_dim=3), dict(action_dim=3), dict(state_dim=7), dict(flags=0),
             dict(flags=SYM | _native.ROLLOUT_INCREMENTAL), dict(d_track=0x9000), dict(d_track=0x9000, d_cost=0xa000),
             dict(flags=SYM | _native.ROLLOUT_GUST), dict(d_sensor_noise=0xb000),
             dict(d_track=0x9000, widths=ctypes.cast(warr, ctypes.c_void_p), n_widths=2),
             dict(flags=SYM | _native.ROLLOUT_GUST, widths=ctypes.cast(warr, ctypes.c_void_p), n_widths=2)]
    for kw in cases:
        rc, msg = run(**kw)
        assert rc == -1 and ('symmetric' in msg.lower() or (kw.get('flags', 0) & _native.ROLLOUT_INCREMENTAL and 'incremental' in msg.lower())), (kw, rc, msg)
    assert 'SERL_ROLLOUT_SYMMETRIC' in run(flags=0)[1]          # a 2 -> 1 shape without the flag is told which flag it needs


def test_symmetric_actors_k1_cannot_hold_are_routed_to_k1_tc():
    """serl_actor_tc_widths counts the 2 -> 1 genome: K1 keeps the shapes whose genome fits its kernels, the others get the
    width list [h] * (L + 1) of the same genome for K1-TC, whose parameter count is the uniform actor's"""
    from serl_b200 import build, rollout
    build.build()
    sym = lambda h, L: rollout.actor_shape(h, L, 'tanh', state_dim=2, action_dim=1)
    keeps = {}
    for h in (32, 64, 72, 96, 128):
        L = 1
        while rollout.tc_widths(sym(h, L + 1)) is None:
            L += 1
        keeps[h] = L
    assert keeps == {32: 44, 64: 10, 72: 7, 96: 4, 128: 3}, keeps       # the limits include/serl_route.h states
    for h, L in ((101, 3), (143, 1)):
        assert rollout.tc_widths(sym(h, L)) is None and rollout.tc_widths(sym(h + 1, L)) == [h + 1] * (L + 1), (h, L)
    for h, L in ((72, 8), (96, 5), (128, 4), (256, 3), (256, 1), (320, 8)):
        w = rollout.tc_widths(sym(h, L))
        assert w == [h] * (L + 1), (h, L, w)
        assert rollout.num_params_wide(w, 2, 1) == rollout.num_params(sym(h, L))


# ---- refusals of the paths that fly attitude control only ---------------------------------------------------------------
def test_k7_sweep_suite_and_operator_study_refuse_symmetric_control():
    from serl_b200 import evaluation, operators, rollout, sweep, td3_fused
    args = types.SimpleNamespace(state_dim=2, action_dim=1, fused_td3=True, hidden_size=72, num_layers=3, activation_actor='tanh')
    with pytest.raises(ValueError, match='symmetric control'):
        td3_fused.FusedTD3(args)
    with pytest.raises(ValueError, match='symmetric control'):
        sweep.Sweep([(args, None)])
    with pytest.raises(ValueError, match='symmetric control'):
        evaluation.evaluate_population(np.zeros((1, 1)), rollout.actor_shape(72, 3, 'tanh', state_dim=2, action_dim=1), ['nominal'], [])
    with pytest.raises(ValueError, match='symmetric control'):
        operators.OperatorRunner(args)
    with pytest.raises(ValueError, match='symmetric control'):
        evaluation.condition_env('PHlab_symmetric_nominal')


def test_agent_refuses_widths_that_do_not_match_the_env():
    from serl_b200.core import agent
    from serl_b200.envs import config
    env = config.select_env('PHlab_symmetric_nominal')
    with pytest.raises(ValueError, match='action_dim'):
        agent.Agent(types.SimpleNamespace(state_dim=2, action_dim=3), env)
    with pytest.raises(ValueError, match='symmetric control has 2'):
        agent.Agent(types.SimpleNamespace(state_dim=7, action_dim=1), env)
    with pytest.raises(ValueError, match='action_dim'):
        agent.Agent(types.SimpleNamespace(state_dim=7, action_dim=1), config.select_env('PHlab_attitude_nominal'))


# ---- drop-in: the reference's unmodified base/train.py with -env PHlab_symmetric_nominal ---------------------------------
TRAIN = '/root/reference/base/train.py'


@pytest.mark.skipif(not os.path.exists(TRAIN), reason='needs the reference tree (build container only)')
@pytest.mark.skipif(torch.cuda.is_available(), reason='CPU leg')
def test_unmodified_reference_train_py_with_symmetric_control_reaches_the_gpu_boundary(tmp_path):
    run = ("import sys; sys.path.insert(0, %r); import serl_b200.dropin as d; d.install(); import runpy; "
           "sys.argv = ['train.py'] + %r; runpy.run_path(%r, run_name='__main__')")
    args = ['-frames', '6000', '-pop_size', '6', '-mut_type', 'normal', '-test_ea', '-env', 'PHlab_symmetric_nominal']
    p = subprocess.run([sys.executable, '-c', run % (ROOT, args, TRAIN)], cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert p.returncode != 0
    assert 'needs a CUDA device' in p.stderr and 'NativeError' in p.stderr, p.stderr[-2000:]
    # Agent() got past its checks that parameters.state_dim / action_dim (2 / 1, the env's widths) match the env
    assert 'agent.Agent(parameters, env)' in p.stderr and 'ValueError' not in p.stderr
