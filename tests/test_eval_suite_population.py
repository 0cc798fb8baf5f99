"""Host side of the population evaluation suite (serl_b200/evaluation.py, examples/evaluate.py): the reference signals of
base/evaluation_utils.py gen_refs, the vectorised sensor-noise draws, nMAE from the kernel's tracking-error sums, the
checkpoint loaders and the -save_stats files.  No GPU."""
import os
import sys
import tomllib

import numpy as np
import pytest
import torch
import yaml

from serl_b200 import evaluation, signals
from serl_b200.core.genetic_agent import Actor
from serl_b200.core.utils import calc_nMAE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def restated_gen_refs(t_max, amp_times, ampl_max, num_trails):
    """base/evaluation_utils.py:23-55 step by step: per trial a 6-level choice, level 0 forced to zero, then the block times
    of the PREVIOUS trial (the base times for the first) each moved by one uniform(-0.05, 0.05)"""
    refs = []
    prev = [float(t) for t in amp_times]
    for _ in range(num_trails):
        choices = np.linspace(-ampl_max, ampl_max, 6)
        amps = np.random.choice(choices, size=6, replace=True)
        amps[0] = 0.0
        moved = [prev[0]]
        for t in prev[1:]:
            moved.append(t + np.random.uniform(-0.05, 0.05))
        prev = moved
        refs.append((np.array(moved), amps.copy(), t_max // 10))
    return refs


@pytest.mark.parametrize('seed', [0, 7, 123])
@pytest.mark.parametrize('num_trails', [1, 2, 5])
def test_gen_refs_matches_the_reference_draw_for_draw(seed, num_trails):
    t_max = 80
    times = np.linspace(0., t_max, 6)
    np.random.seed(seed)
    want = restated_gen_refs(t_max, times, 12.0, num_trails)
    state_want = np.random.get_state()[1].copy()
    np.random.seed(seed)
    got = evaluation.gen_refs(t_max, times, 12.0, num_trails)
    assert np.array_equal(np.random.get_state()[1], state_want)
    assert len(got) == num_trails
    for g, (st, lv, sw) in zip(got, want):
        assert np.array_equal(g.starts, st) and np.array_equal(g.levels, lv) and g.smooth_width == sw == 8
    if num_trails > 1:      # the jitter accumulates: trial 1's times are trial 0's moved again
        assert np.abs(got[1].starts[1:] - got[0].starts[1:]).max() <= 0.05
        assert not np.array_equal(got[1].starts, got[0].starts)


def test_eval_refs_appends_the_base_reference_last():
    np.random.seed(7)
    refs = evaluation.eval_refs(2)
    np.random.seed(7)
    th = evaluation.gen_refs(80, np.linspace(0, 80, 6), 12.0, 2)
    ph = evaluation.gen_refs(80, np.linspace(0, 80, 6), 10.0, 2)
    assert len(refs) == 3
    for i in range(2):
        assert np.array_equal(refs[i][0].levels, th[i].levels) and np.array_equal(refs[i][1].starts, ph[i].starts)
    assert list(refs[2][0].levels) == [0, 12, 3, -4, -8, 2] and list(refs[2][1].levels) == [2, -2, 2, 10, 2, -6]
    assert np.array_equal(refs[2][0].starts, np.linspace(0, 80, 6)) and refs[2][1].smooth_width == 8


def loop_noise_draws(n_traj, horizon):
    """the per-native-call draws of envs/noise/citation.py:72-82 (randn(3), randn(1), randn(1), randn(2)), one call at a time"""
    z = np.empty((n_traj, horizon + 1, 7), dtype=np.float32)
    for i in range(n_traj):
        for c in range(horizon + 1):
            z[i, c, 0:3] = np.random.randn(3)
            z[i, c, 3] = np.random.randn(1)[0]
            z[i, c, 4] = np.random.randn(1)[0]
            z[i, c, 5:7] = np.random.randn(2)
    return z


@pytest.mark.parametrize('n_traj,horizon,warm', [(1, 0, False), (3, 4, False), (2, 5, True), (5, 12, True), (1, 2, True)])
def test_vectorised_noise_draws_equal_the_per_call_loop(n_traj, horizon, warm):
    """legacy randn keeps its cached second gaussian across calls: one call of n draws continues the stream as n calls of
    one draw would.  Odd totals and a warm cache (an odd number of draws before) included."""
    np.random.seed(11)
    if warm:
        np.random.randn(1)
    want = loop_noise_draws(n_traj, horizon)
    after_want = np.random.get_state()
    np.random.seed(11)
    if warm:
        np.random.randn(1)
    got = evaluation.sensor_noise_draws(n_traj, horizon)
    after = np.random.get_state()
    assert got.dtype == np.float32 and got.shape == (n_traj, horizon + 1, 7)
    assert np.array_equal(got, want)
    assert np.array_equal(after[1], after_want[1]) and after[2:] == after_want[2:]       # incl. the gauss cache


def test_nmae_from_track_equals_calc_nmae():
    rs = np.random.RandomState(3)
    for n, scale, bias in [(8001, 0.05, 0.0), (1234, 0.01, 0.2), (3, 1e-4, 0.0)]:
        e = rs.randn(n, 3) * scale + bias
        track = np.array([np.abs(e[:, 0]).sum(), np.abs(e[:, 1]).sum(), np.abs(e[:, 2]).sum(), e[:, 2].sum()])
        got = evaluation.nmae_from_track(track[None], np.array([n]))[0]
        assert got == pytest.approx(calc_nMAE(e), rel=1e-12)


class Args:
    state_dim, action_dim, hidden_size, num_layers, activation_actor = 7, 3, 16, 2, 'tanh'


def write_run(run_dir, genomes, args, rl=None):
    """a run directory as training leaves it: files/config.yaml (wandb layout) and the checkpoints of Agent.save_agent"""
    files = os.path.join(run_dir, 'files')
    os.makedirs(files, exist_ok=True)
    cfg = {k: {'desc': None, 'value': getattr(args, k)} for k in ('hidden_size', 'num_layers', 'activation_actor')}
    with open(os.path.join(files, 'config.yaml'), 'w') as f:
        yaml.safe_dump(cfg, f)

    def state(g):
        a = Actor(args)
        a.bind(torch.as_tensor(np.asarray(g, dtype=np.float32)).clone())
        return {k: v.detach().clone() for k, v in a.state_dict().items()}
    torch.save({f'actor_{i}': state(g) for i, g in enumerate(genomes)}, os.path.join(files, 'evo_nets.pkl'))
    if rl is not None:
        torch.save(state(rl), os.path.join(files, 'rl_net.pkl'))


def test_loaders_read_a_saved_checkpoint(tmp_path):
    torch.manual_seed(0)
    P = sum(p.numel() for p in Actor(Args).parameters())
    g = torch.randn(4, P).numpy().astype(np.float32)
    rl = torch.randn(P).numpy().astype(np.float32)
    write_run(str(tmp_path), g, Args, rl)

    class Fresh:
        state_dim, action_dim = 7, 3
        hidden_size, num_layers, activation_actor = 72, 3, 'elu'           # replaced by config.yaml
        def update_from_dict(self, d):
            self.__dict__.update(d)
    args = evaluation.run_config(str(tmp_path), Fresh())
    assert (args.hidden_size, args.num_layers, args.activation_actor) == (16, 2, 'tanh')
    pop = evaluation.load_pop(str(tmp_path), args)
    assert pop.dtype == np.float32 and np.array_equal(pop, g)
    assert np.array_equal(evaluation.load_rl_agent(str(tmp_path), args), rl[None])


def test_stats_files_round_trip(tmp_path):
    sm, nm = [-18.007365454720173, -43.4378341918449], [9.89261565667466, 11.937120033579463]
    evaluation.write_final_performance(str(tmp_path), 'be', sm, nm)
    rows = np.loadtxt(os.path.join(tmp_path, 'figures', 'be', 'final_performance.csv'), delimiter=',')
    assert np.array_equal(rows, np.array([sm, nm]).T)
    champ = evaluation.Stats(6.581009081951172, 1.7417491912166163, -2.810896612027241, 0.5116869271083809)
    avg = evaluation.Stats(15.193464394940273, 7.7828326612143925, -59.97064836909332, 66.14170593751305)
    evaluation.append_stats_toml(str(tmp_path), 'nominal', 8, champ, avg)
    evaluation.append_stats_toml(str(tmp_path), 'high-q', 3, avg, champ)
    with open(os.path.join(tmp_path, 'stats.toml'), 'rb') as f:
        t = tomllib.load(f)
    assert t['nominal']['champion_idx'] == 8 and t['high-q']['champion_idx'] == 3
    assert t['nominal']['champion'] == champ._asdict() and t['nominal']['average'] == avg._asdict()
    assert t['high-q']['champion'] == avg._asdict()
    # the reference's logged files parse the same way (layout of logs/wandb/*/stats.toml)
    text = open(os.path.join(tmp_path, 'stats.toml')).read()
    assert text.startswith('[nominal]\nchampion_idx = 8\n\n[nominal.champion]\nnmae = 6.581009081951172\n')


def test_rl_stats_and_trajectory_files_round_trip(tmp_path):
    s1 = evaluation.Stats(7.432706455646595, 1.6067772053365974, -344.2960229984458, 48.79411793655151)
    s2 = evaluation.Stats(11.529252356850398, 2.2470341631458277, -138.7459762272979, 71.47751582326993)
    evaluation.append_rl_stats_toml(str(tmp_path), 'nominal', s1)
    evaluation.append_rl_stats_toml(str(tmp_path), 'low-q', s2)
    with open(os.path.join(tmp_path, 'stats.toml'), 'rb') as f:
        t = tomllib.load(f)
    assert t == {'nominal': s1._asdict(), 'low-q': s2._asdict()}
    text = open(os.path.join(tmp_path, 'stats.toml')).read()
    assert text.startswith('\n\n[nominal]\nnmae = 7.432706455646595\n')         # the layout of a TD3 run's stats.toml
    data = np.random.RandomState(0).randn(5, 19)
    evaluation.write_trajectory(str(tmp_path), 'be', data)
    path = os.path.join(tmp_path, 'figures', 'be', 'nominal_trajectory.csv')
    assert ',' not in open(path).read() and np.array_equal(np.loadtxt(path), data)


def test_cli_takes_the_reference_flags():
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import evaluate as cli
    finally:
        sys.path.pop(0)
    cla = cli.parser.parse_args(['-agent_name', 'runs/x', '-env', 'all', '-eval_pop', '-num_trails', '2', '-seed', '3',
                                 '-save_stats', '-save_trajectory', '-verbose'])
    assert cla.eval_pop and cla.save_stats and cla.save_trajectory and cla.verbose and cla.num_trails == 2 and cla.seed == 3
    assert cli.conditions(cla.env) == list(evaluation.CONDITIONS)
    cla = cli.parser.parse_args(['-agent_name', 'r', '-env', 'PHlab_attitude_be', '-eval_actor', '-index', '4'])
    assert cla.eval_actor and cla.index == 4 and cli.conditions(cla.env) == ['be'] and cla.seed == 7 and cla.num_trails == 1
    cla = cli.parser.parse_args(['-agent_name', 'r', '-env', 'nominal,ice,cg-shift', '-eval_rl'])
    assert cla.eval_rl and cli.conditions(cla.env) == ['nominal', 'ice', 'cg-shift']
    for c in evaluation.CONDITIONS:          # every condition names an env the kernels fly
        assert evaluation.condition_env(c).t_max == 80
