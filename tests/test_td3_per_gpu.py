"""K7 with prioritized replay (serl_td3_learn with a priority tree) and the device priority tree (csrc/per.cu) on the GPU.

Every K7 case runs with its draws recorded (rows, weights, TD errors, noise, CAPS uniforms) and replays them on the CPU
through the weighted fp32 oracle and its float64 copy (tests/td3_per_oracle.py), under the error budget of
tests/test_td3_reference_gpu.py.  The tree is checked after launches: every leaf a step re-prioritised equals
(delta + 1e-5)^0.6 of the recorded delta, and every internal node is its children's sum and min, bitwise.  The draws
follow P(i) = p_i / sum p (chi-square, with rows repeated inside a batch), K7 draws the rows the standalone sampler
draws, and the result is bitwise the same at every cluster size and launch split."""
import os
import types

import numpy as np
import pytest
import torch

import td3_per_oracle as P
from oracle import td3 as O
from test_td3_reference_gpu import Reference, fused, synthetic_rows, td3_args

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def per_buffer(rows, seed=7, skew=True, capacity=None):
    """a DevicePrioritizedReplayMemory holding rows [n, 19] (device), its priorities made uneven by a few update_priorities
    calls when `skew`"""
    from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory
    n = rows.shape[0]
    buf = DevicePrioritizedReplayMemory(capacity or n, DEV, seed=seed, beta_frames=1000)
    buf.add_rows(torch.cat([rows, torch.zeros((n, 1), device=rows.device)], 1))
    if skew:
        g = torch.Generator().manual_seed(seed)
        for _ in range(6):
            idx = torch.randint(0, n, (128,), generator=g)
            buf.update_priorities(idx, torch.rand(128, generator=g) ** 3 * 4)
    return buf


def tree_host(buf):
    return buf.tree.view(-1, 2).cpu().numpy()


def check_internal_nodes(t):
    L = t.shape[0] // 2
    v = np.arange(1, L)
    assert np.array_equal(t[v, 0], t[2 * v, 0] + t[2 * v + 1, 0])
    assert np.array_equal(t[v, 1], np.fmin(t[2 * v, 1], t[2 * v + 1, 1]))


class PerReference(Reference):
    def replay(self, rows_cpu, launch, first_iteration, champion=False):
        idx, noise, caps, w = launch.indices.cpu().long(), launch.noise.cpu(), launch.caps.cpu(), launch.weights.cpu()
        use_caps = self.t32.caps_dict is not None
        l32, l64, self.delta64 = [], [], []
        for k in range(idx.shape[0]):
            it = first_iteration + k
            rows = rows_cpu[idx[k]]
            pg, td, _ = P.update_parameters(self.t32, rows, it, noise[k], caps[k] if use_caps else None, champion, weights=w[k])
            pg6, td6, d6 = P.update_parameters(self.t64, rows.double(), it, noise[k].double(), caps[k].double() if use_caps else None,
                                               champion, weights=w[k].double())
            l32.append((float(td), float('nan') if pg is None else float(pg)))
            l64.append((float(td6), float('nan') if pg6 is None else float(pg6)))
            self.delta64.append(d6.numpy())
        return np.array(l32), np.array(l64), None


def run_per(f, buf, n, first, label, champion=False):
    ref = PerReference(f)
    r = f.run(buf.data, len(buf), n, first, champion, record=True, per=buf)
    r.check()
    l32, l64, _ = ref.replay(buf.data[:len(buf), :19].cpu(), r, first, champion)
    ref.check(f, r, l32, l64, label)
    return r, ref


def check_delta_and_leaves(r, ref, buf):
    """the recorded delta against the float64 oracle's, and every re-prioritised leaf = (delta + 1e-5)^0.6 of its last draw"""
    td = r.td.cpu().double().numpy()
    d64 = np.stack(ref.delta64)
    assert np.abs(td - d64).max() <= 1e-5 * max(1.0, np.abs(d64).max()), np.abs(td - d64).max()
    last = {}
    for k, row in enumerate(r.indices.cpu().numpy()):
        for j, i in enumerate(row):
            last[int(i)] = td[k, j]
    t = tree_host(buf)
    L = t.shape[0] // 2
    rows = np.array(sorted(last))
    want = (np.array([last[i] for i in rows]) + 1e-5) ** 0.6
    np.testing.assert_allclose(t[L + rows, 0], want, rtol=1e-15)
    assert np.array_equal(t[L + rows, 0], t[L + rows, 1])
    check_internal_nodes(t)


@pytest.mark.parametrize('hidden,num_layers', [(32, 2), (64, 1), (64, 2), (96, 1), (96, 4), (128, 5)])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
def test_one_per_step_matches_float64(hidden, num_layers, activation):
    f = fused(td3_args(hidden, num_layers, activation))
    buf = per_buffer(synthetic_rows(3000, seed=hidden + num_layers).to(DEV))
    r, ref = run_per(f, buf, 1, 3, 'PER h%d L%d %s' % (hidden, num_layers, activation))
    w = r.weights.cpu().numpy()
    assert w.max() <= 1.0 and w.min() < 0.9                  # the priorities are uneven: so are the weights
    check_delta_and_leaves(r, ref, buf)


def test_wide_actor_and_20_steps_match_float64():
    """a wide (tiled) actor, and 20 steps in which each step samples the tree the previous one re-prioritised"""
    f = fused(td3_args(256, 2, 'elu'))
    buf = per_buffer(synthetic_rows(2000, seed=3).to(DEV))
    r, ref = run_per(f, buf, 1, 1, 'PER wide')
    check_delta_and_leaves(r, ref, buf)
    f = fused(td3_args())
    buf = per_buffer(synthetic_rows(500, seed=4).to(DEV))
    r, ref = run_per(f, buf, 20, 1, 'PER 20 steps')
    check_delta_and_leaves(r, ref, buf)
    assert any(len(np.unique(b)) < b.size for b in r.indices.cpu().numpy())     # rows repeat inside a batch


def test_k7_draws_what_the_sampler_draws_and_weights_like_the_reference():
    """K7's first step draws the standalone sampler's rows and weights (same tree, iteration and seed), and the weights are
    the reference buffer's formula on the tree's priorities with beta of the learner's critic step"""
    from serl_b200 import _native
    f = fused(td3_args())
    buf = per_buffer(synthetic_rows(3000, seed=5).to(DEV), seed=f.seed)
    f.critic_steps = 41                                        # the 42nd sample: beta = 0.4 + 42 * 0.6 / 1000
    pri = buf.leaves().cpu().numpy()
    rows = torch.empty(86, dtype=torch.int32, device=DEV)
    w = torch.empty((86, 1), dtype=torch.float32, device=DEV)
    beta = buf.beta_by_frame(42)
    _native.call('serl_per_sample', buf.tree, buf.capacity, len(buf), 86, f.seed, 100, beta, rows, w, device=DEV)
    r = f.run(buf.data, len(buf), 1, 100, record=True, per=buf)
    assert torch.equal(r.indices[0], rows) and torch.equal(r.weights[0], w[:, 0])
    N, P_ = len(pri), pri / pri.sum()
    want = (N * P_[rows.cpu().numpy()]) ** -beta / (N * P_.min()) ** -beta
    np.testing.assert_allclose(r.weights[0].cpu().double().numpy(), want, rtol=1e-6)


def test_draws_follow_the_priorities():
    """2000 batches of 86 from 40 rows with priorities 1..40^2: chi-square against P(i) = p_i / sum p, every row drawn, and
    batches holding repeats as often as independent draws do"""
    from scipy import stats
    from serl_b200 import _native
    from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory
    n, B, T = 40, 86, 2000
    buf = DevicePrioritizedReplayMemory(n, DEV, seed=3)
    buf.add_rows(torch.zeros((n, 20), device=DEV))
    pri = (np.arange(1, n + 1, dtype=np.float64)) ** 2
    L = buf.tree.numel() // 4
    buf.tree.view(-1, 2)[L:L + n] = torch.as_tensor(np.stack([pri, pri], 1), device=DEV)
    _native.call('serl_per_rebuild', buf.tree, n, device=DEV)
    check_internal_nodes(tree_host(buf))
    rows = torch.empty((T, B), dtype=torch.int32, device=DEV)
    w = torch.empty((T, B), dtype=torch.float32, device=DEV)
    for it in range(T):
        _native.call('serl_per_sample', buf.tree, n, n, B, 3, it + 1, 0.5, rows[it], w[it], device=DEV)
    idx = rows.cpu().numpy()
    counts = np.bincount(idx.reshape(-1), minlength=n)
    p = stats.chisquare(counts, T * B * pri / pri.sum()).pvalue
    assert p > 1e-4, p
    assert counts.min() > 0
    # the position of a draw in its batch does not matter: the first and last halves of the batch, separately
    for half in (idx[:, :B // 2], idx[:, B // 2:]):
        c = np.bincount(half.reshape(-1), minlength=n)
        assert stats.chisquare(c, half.size * pri / pri.sum()).pvalue > 1e-4
    np.testing.assert_allclose(w.cpu().double().numpy(), (pri[idx] / pri.min()) ** -0.5, rtol=1e-6)


def test_cluster_sizes_and_launch_splits_are_bitwise_identical():
    args = td3_args()
    torch.manual_seed(5)
    from serl_b200.td3_fused import FusedTD3
    f = FusedTD3(args)
    s0 = f.state.clone()
    rows = synthetic_rows(3000, seed=3).to(DEV)

    def go(plan, cs):
        buf = per_buffer(rows)
        f.state.copy_(s0)
        f.critic_steps = f.actor_steps = 0
        first, losses = 1, []
        for n in plan:
            losses.append(f.run(buf.data, len(buf), n, first, False, cluster_size=cs, per=buf).losses)
            first += n
        torch.cuda.synchronize()
        return f.state.clone(), torch.cat(losses), buf.tree.clone()

    ref_state, ref_loss, ref_tree = go([30], 1)
    assert torch.isfinite(ref_loss[:, 0]).all()
    check_internal_nodes(ref_tree.view(-1, 2).cpu().numpy())
    for cs, plan in ((2, [30]), (4, [30]), (8, [30]), (8, [11, 19]), (2, [1, 29])):
        s, l, t = go(plan, cs)
        assert torch.equal(s, ref_state) and torch.equal(t, ref_tree), (cs, plan)
        assert torch.equal(l.nan_to_num(7.0), ref_loss.nan_to_num(7.0)), (cs, plan)


def test_torch_path_reprioritises_like_k7():
    """the torch path's update_priorities fed K7's recorded rows and TD errors leaves K7's tree, bit for bit; its sample is
    K7's draw at the same iteration"""
    f = fused(td3_args())
    rows = synthetic_rows(1000, seed=6).to(DEV)
    k7, host = per_buffer(rows, seed=f.seed), per_buffer(rows, seed=f.seed)
    assert torch.equal(k7.tree, host.tree)
    host.frame = 1
    batch = host.sample(86)
    r = f.run(k7.data, len(k7), 1, 1, record=True, per=k7)
    assert torch.equal(batch[6], r.indices[0]) and torch.equal(batch[5][:, 0], r.weights[0])
    assert torch.equal(batch[0], k7.data[r.indices[0].long(), :7])
    host.update_priorities(r.indices[0], r.td[0])
    assert torch.equal(k7.tree, host.tree)


def _agent(tmp_path, fused_td3):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.parameters import Parameters
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        args = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=4, mut_type='normal', test_ea=False,
                                                fused_td3=fused_td3, per=True, frames=20000))
    finally:
        os.chdir(cwd)
    args.save_foldername = str(tmp_path) + '/'
    args.state_dim, args.action_dim, args.hidden_size = 7, 3, 32
    args.learn_start, args.frac_frames_train = 300, 0.2
    torch.manual_seed(7)
    return agent_mod.Agent(args, config.select_env('PHlab_attitude_nominal'))


@pytest.mark.parametrize('fused_td3', [True, False])
def test_agent_trains_with_per(tmp_path, fused_td3):
    from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory
    ag = _agent(tmp_path, fused_td3)
    assert isinstance(ag.replay_buffer, DevicePrioritizedReplayMemory) and ag.replay_buffer.beta_frames == 20000
    before = torch.cat([p.detach().reshape(-1) for p in ag.rl_agent.actor.parameters()]).clone()
    for _ in range(3):
        stats = ag.train()
    assert np.isfinite(stats['TD_loss']) and np.isfinite(stats['PG_obj']) and ag.rl_iteration > 0
    assert not torch.equal(before, torch.cat([p.detach().reshape(-1) for p in ag.rl_agent.actor.parameters()]))
    pri = ag.replay_buffer.leaves().cpu().numpy()
    assert len(pri) == len(ag.replay_buffer) and np.all(pri > 0)
    assert len(np.unique(pri)) > 100                           # the trained rows were re-prioritised
    check_internal_nodes(tree_host(ag.replay_buffer))
