"""Incremental control (the reference's PHlab_attitude_incremental) without a GPU: the oracle's restatement on the reference's
own nominal binary, the env mirror's name grammar and spaces, the 10-input actor's parameter count, the replay layout of
state_dim 10, the launch checks of SERL_ROLLOUT_INCREMENTAL, and the refusals of the paths that do not fly it."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import actor as A, build as OB, refsig

from incremental_oracle import IncrementalCitationEnv, KernelOrderActor, run_episode  # noqa: E402  (tests/ on sys.path)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def genome(hidden, activation, seed, scale=1.0):
    torch.manual_seed(seed)
    g = A.flatten(A.Actor(state_dim=10, hidden=hidden, num_layers=3, activation=activation))
    return (g * np.float32(scale)).astype(np.float32)


# ---- the oracle: the reference binary and the C restatement agree bit for bit under incremental control -----------------
@pytest.mark.refbin
@pytest.mark.skipif(not OB.have_ref(), reason='needs the reference plant binaries under oracle/_ref')
@pytest.mark.parametrize('policy', ['tanh', 'elu', 'relu', 'saturating'])
def test_incremental_env_on_the_reference_binary_equals_the_c_restatement(policy):
    """300-step closed loops of random 10-input actors (and an open loop of full-rate commands that drives u far past the
    plant's input limits) on both plant back-ends: every step's state, deflection, reward and observation is identical."""
    lv, st = refsig.make_ref_params(1, seed_base=41)
    actions = None
    if policy == 'saturating':
        rs = np.random.RandomState(5)
        actions = np.repeat(np.sign(rs.randn(10, 3)), 30, axis=0).astype(np.float32)      # +-25 deg/s held for 0.3 s
        actor = None
    else:
        actor = KernelOrderActor(genome(72, policy, 3, scale=3.0), 72, activation=policy)
    out = {}
    for backend in ('ref', 'port'):
        env = IncrementalCitationEnv(backend)
        out[backend] = run_episode(env, actor, lv[0], st[0], horizon=300, actions=actions)
    a, b = out['ref'], out['port']
    assert a['steps'] == b['steps'] and a['ret'] == b['ret']
    assert np.array_equal(a['rows'].view(np.uint32), b['rows'].view(np.uint32))
    assert np.array_equal(a['u'], b['u'])
    if policy == 'saturating':
        assert np.abs(a['u']).max() > np.deg2rad(25) * 0.01 * 100      # well beyond any actuator's deflection limit


def test_incremental_oracle_integrates_rates_in_the_reference_order():
    """u_k = u_{k-1} + rate_k * 0.01 with rate = low + 0.5 (a + 1) (high - low), a float32 action; obs[7:] = u; no clip"""
    env = IncrementalCitationEnv('port')
    lv, st = refsig.make_ref_params(1, seed_base=2)
    acts = np.tile(np.float32([1.0, -0.5, 0.25]), (40, 1))
    r = run_episode(env, None, lv[0], st[0], horizon=40, actions=acts)
    b = np.deg2rad(25)
    u = np.zeros(3)
    for k in range(r['steps']):
        rate = -b + (0.5 * (acts[k] + np.float32(1.0))).astype(np.float32) * (b - (-b))
        u = u + rate * 0.01
        assert np.array_equal(r['u'][k], u)
        assert np.array_equal(r['rows'][k, 13 + 7:13 + 10], u.astype(np.float32))           # next_obs[7:10]
    assert np.array_equal(r['rows'][0, 7:10], np.zeros(3, dtype=np.float32))                 # reset(): last_u = 0
    assert r['rows'].shape[1] == 26


# ---- env mirror: name grammar and spaces ---------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['PHlab_attitude_incremental', 'PHlab_attitude_h2000-v90-incremental', 'PHlab_attitude_gust-incremental',
                                  'phlab_attitude_noise-incremental'])
def test_any_mode_containing_incremental_flies_the_nominal_plant_with_incremental_control(name):
    from serl_b200 import rollout
    from serl_b200.envs import config
    env = config.select_env(name)
    assert env.incremental and env.mode == 'nominal' and not env.sensor_noise
    assert env.mode_code == rollout.mode_code('nominal') and not rollout.mode_gust(env.mode_code)
    assert env.bound == np.deg2rad(25) and np.array_equal(env.action_space.high, np.deg2rad(25) * np.ones(3))
    assert env.n_obs == 10 and env.observation_space.shape == (10,)


@pytest.mark.parametrize('name,mode,noise', [('PHlab_attitude_be', 'be', False), ('PHlab_attitude_gust', 'gust', True),
                                             ('PHlab_attitude_nominal', 'nominal', False)])
def test_absolute_modes_are_unchanged(name, mode, noise):
    from serl_b200.envs import config
    env = config.select_env(name)
    assert not env.incremental and env.mode == mode and env.sensor_noise == noise
    assert env.bound == np.deg2rad(10) and env.n_obs == 7 and env.observation_space.shape == (7,)


def test_parameter_count_and_table_of_the_ten_input_actor():
    from serl_b200 import evo, rollout
    for h in (32, 64, 72, 96, 128, 256):
        sh = rollout.actor_shape(h, 3, 'tanh', state_dim=10)
        assert rollout.num_params(sh) == 3 * h * h + 23 * h + 3
        table, P = evo.param_table(10, 3, h, 3)
        assert P == rollout.num_params(sh) and table[0] == (0, h, 10) and table[1] == (10 * h, h, 0)
        assert P == len(A.flatten(A.Actor(state_dim=10, hidden=h, num_layers=3)))


# ---- replay layout ---------------------------------------------------------------------------------------------------------
def test_replay_layout_has_one_rule_that_the_header_and_every_buffer_follow(tmp_path):
    from serl_b200 import _native, rollout
    from serl_b200.core.replay_memory import DeviceReplayMemory, PopulationBuffers, ActorBuffer
    assert rollout.replay_cols(7) == _native.REPLAY_COLS == 20 and rollout.replay_cols(10) == 26
    assert rollout.transition_cols(10) == 25 and rollout.TRANSITION_COLS == rollout.REPLAY_COST == 19
    src = tmp_path / 'cols.c'
    src.write_text('#include <stdio.h>\n#include "serl_b200.h"\nint main(void) { printf("%d %d %d %d\\n", SERL_REPLAY_COLS_OF(7), '
                   'SERL_REPLAY_COLS_OF(10), SERL_REPLAY_COLS, SERL_ROLLOUT_INCREMENTAL); return 0; }\n')
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), '-o', str(tmp_path / 'cols'), str(src)])
    assert subprocess.check_output([str(tmp_path / 'cols')], text=True).split() == ['20', '26', '20', str(_native.ROLLOUT_INCREMENTAL)]
    rows = torch.arange(6 * 26, dtype=torch.float32).reshape(6, 26)
    mem = DeviceReplayMemory(4, 'cpu', state_dim=10)
    mem.add_rows(rows)
    assert len(mem) == 4 and mem.data.shape == (4, 25)
    s, a, s2, r, d = mem.sample(3)
    assert (s.shape, a.shape, s2.shape, r.shape, d.shape) == ((3, 10), (3, 3), (3, 10), (3, 1), (3, 1))
    assert torch.equal(s2[:, 0] - s[:, 0], torch.full((3,), 13.0)) and torch.equal(r[:, 0] - s[:, 0], torch.full((3,), 23.0))
    pb = PopulationBuffers(2, 8, 'cpu', state_dim=10)
    pb.append(torch.tensor([1]), rows[None], torch.ones((1, 6), dtype=torch.bool))
    assert torch.equal(pb.rows_of(1), rows[:, :25])
    latest = ActorBuffer(pb, 1).get_latest(2)
    assert len(latest) == 2 and latest[-1].state.shape == (1, 10) and float(latest[-1].done) == rows[5, 24]


# ---- launch checks (no CUDA call) --------------------------------------------------------------------------------------------
def test_rollout_run_checks_the_incremental_flag_before_any_cuda_call():
    from serl_b200 import _native, build
    build.build()
    L = _native.lib()
    warr = (ctypes.c_int32 * 2)(128, 128)

    def run(state_dim=10, flags=_native.ROLLOUT_INCREMENTAL, **kw):
        d = _native.RolloutDesc()
        fake = iter(range(0x10000, 0x100000, 0x1000))      # non-null, never read
        for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_fitness', 'd_replay', 'd_status'):
            setattr(d, f, next(fake))
        d.pop, d.shape, d.n_envs, d.horizon, d.replay_env, d.flags = 4, _native.ActorShape(state_dim, 3, 72, 3, 0), 8, 100, 0, flags
        for k, v in kw.items():
            setattr(d, k, v)
        return L.serl_rollout_run(ctypes.byref(d), None), L.serl_last_error().decode()

    cases = [dict(state_dim=7), dict(flags=0), dict(d_track=0x9000), dict(d_track=0x9000, d_cost=0xa000),
             dict(flags=_native.ROLLOUT_INCREMENTAL | _native.ROLLOUT_GUST), dict(d_sensor_noise=0xb000),
             dict(state_dim=7, widths=ctypes.cast(warr, ctypes.c_void_p), n_widths=2),
             dict(d_track=0x9000, widths=ctypes.cast(warr, ctypes.c_void_p), n_widths=2)]
    for kw in cases:
        rc, msg = run(**kw)
        assert rc == -1 and 'incremental' in msg.lower(), (kw, rc, msg)
    assert 'SERL_ROLLOUT_INCREMENTAL' in run(flags=0)[1]        # a 10-input shape without the flag is told which flag it needs


def test_k1_fit_rule_counts_the_ten_input_genome():
    """serl_actor_tc_widths: K1 keeps the 10-input actor where its genome fits, else routes it to K1-TC's widths; the limits
    the header states for state_dim 10, and the parameter count of the 10-input width list"""
    from serl_b200 import build, rollout
    build.build()
    keeps = {}
    for h in (32, 64, 72, 96, 128):
        L = 1
        while rollout.tc_widths(rollout.actor_shape(h, L + 1, 'tanh', state_dim=10)) is None:
            L += 1
        keeps[h] = L
    assert keeps == {32: 44, 64: 9, 72: 7, 96: 4, 128: 3}, keeps
    assert rollout.tc_widths(rollout.actor_shape(101, 3, 'tanh', state_dim=10)) == [101] * 4
    for widths in ([101] * 4, [400, 300], [128, 256, 64]):
        assert rollout.num_params_wide(widths, 10) == len(A.flatten(A.WideActor(widths, state_dim=10)))
    assert rollout.num_params_wide([101] * 4, 10) == rollout.num_params(rollout.actor_shape(101, 3, 'tanh', state_dim=10))
    assert rollout.tc_widths(rollout.actor_shape(100, 3, 'tanh', state_dim=10)) is None


# ---- refusals of the paths that fly absolute control only ---------------------------------------------------------------
def test_k7_sweep_suite_and_operator_study_refuse_incremental_control():
    from serl_b200 import evaluation, operators, rollout, sweep, td3_fused
    args = types.SimpleNamespace(state_dim=10, action_dim=3, fused_td3=True, hidden_size=72, num_layers=3, activation_actor='tanh')
    with pytest.raises(ValueError, match='incremental control'):
        td3_fused.FusedTD3(args)
    with pytest.raises(ValueError, match='incremental control'):
        sweep.Sweep([(args, None)])
    with pytest.raises(ValueError, match='incremental control'):
        evaluation.evaluate_population(np.zeros((1, 1)), rollout.actor_shape(72, 3, 'tanh', state_dim=10), ['nominal'], [])
    with pytest.raises(ValueError, match='incremental control'):
        operators.OperatorRunner(args)
    with pytest.raises(ValueError, match='incremental control'):       # examples/evaluate.py -env incremental, any of its modes
        evaluation.condition_env('incremental')
    with pytest.raises(ValueError, match='incremental control'):
        operators.OperatorRunner(types.SimpleNamespace(state_dim=7, hidden_size=72, num_layers=3, activation_actor='tanh'), 'incremental',
                                  device=torch.device('cpu'))


def test_agent_refuses_a_state_dim_that_does_not_match_the_env():
    from serl_b200.core import agent
    from serl_b200.envs import config
    env = config.select_env('PHlab_attitude_incremental')
    with pytest.raises(ValueError, match='incremental control'):
        agent.Agent(types.SimpleNamespace(state_dim=7), env)
    with pytest.raises(ValueError, match='incremental control'):
        agent.Agent(types.SimpleNamespace(state_dim=10), config.select_env('PHlab_attitude_nominal'))


# ---- drop-in: the reference's unmodified base/train.py with -env PHlab_attitude_incremental -----------------------------
TRAIN = '/root/reference/base/train.py'


@pytest.mark.skipif(not os.path.exists(TRAIN), reason='needs the reference tree (build container only)')
@pytest.mark.skipif(torch.cuda.is_available(), reason='CPU leg')
def test_unmodified_reference_train_py_with_incremental_control_reaches_the_gpu_boundary(tmp_path):
    run = ("import sys; sys.path.insert(0, %r); import serl_b200.dropin as d; d.install(); import runpy; "
           "sys.argv = ['train.py'] + %r; runpy.run_path(%r, run_name='__main__')")
    args = ['-frames', '6000', '-pop_size', '6', '-mut_type', 'normal', '-test_ea', '-env', 'PHlab_attitude_incremental']
    p = subprocess.run([sys.executable, '-c', run % (ROOT, args, TRAIN)], cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert p.returncode != 0
    assert 'needs a CUDA device' in p.stderr and 'NativeError' in p.stderr, p.stderr[-2000:]
    # Agent() got past its check that parameters.state_dim (the env's observation width, 10) matches the env
    assert 'agent.Agent(parameters, env)' in p.stderr and 'ValueError' not in p.stderr
