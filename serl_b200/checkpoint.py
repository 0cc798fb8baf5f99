"""Checkpoint and resume a training run, bit for bit.

`save(agent, path)` writes everything the next `Agent.train()` reads; `load(agent, path)` puts it back into an Agent freshly
built from the same Parameters and env (every buffer and module already has its shape and device).  Loading and then
calling train() k times gives the bits the uninterrupted run's next k train() calls give: statistics, genomes, replay
contents, per-actor and critical buffers, learner state, counters and the global generators.

A checkpoint is one file, `torch.save` of a dict of CPU tensors and plain values, read back with `weights_only=True`:

  * the population genomes and the `PopulationBuffers` (rows, ring positions, counts, generator) behind the per-actor and
    critical buffers; SSNE's selection bookkeeping, device generators and the elites of its last plan (the speculative
    validations of the next front read them);
  * the shared replay buffer (its written rows, ring position, length, generator; with `per` the fp64 priority tree,
    `frame` and `beta_frames`) and the RL actor's own two buffers;
  * the learner: FusedTD3's flat state (restored in place: the modules' parameters are views into it), Adam step counts
    and seed, or the torch TD3's four modules and two Adam optimisers;
  * the Agent's counters and the champion's index and state histories (a final save_agent writes the same files);
  * the global stdlib `random`, legacy `np.random`, torch CPU and torch default CUDA generator states (sweep.RNGState);
  * the prefetched front's host-side inputs.  `train()` queues the next generation's front before it returns, and that
    front has already drawn its references and exploration noise from np.random.  The checkpoint keeps those draws (and
    the np.random state the exploration noise was drawn from) and `load` re-launches the front from them: flights are
    deterministic, so the re-launched front gives the bits of the one in flight at the save.

`load` refuses, before it writes anything, a file of another format or version, one without the completion marker, one
written by a different torch.distributed world size, and one whose Parameters differ from the agent's in anything that
fixes the state's shape or meaning (IDENTITY).  `frames` alone may differ, so that a run can be extended; a prioritized
buffer keeps the checkpoint's `beta_frames`, i.e. the beta schedule of the run as first started.

Writes are atomic: a temporary file in the same directory, flushed and fsynced, then `os.replace`.  With a world larger
than 1 every rank holds the same replicated state: rank 0 writes and every rank loads the same file.
"""
import json
import os
import tempfile

import numpy as np
import torch

from . import engine, evo
from .core import agent as agent_mod

FORMAT = 'serl_b200.checkpoint'
VERSION = 1

# the Parameters that fix the shape or meaning of a run's state: a checkpoint loads only into an Agent that agrees on all
IDENTITY = ('pop_size', 'hidden_size', 'num_layers', 'activation_actor', 'state_dim', 'action_dim', 'buffer_size',
            'individual_bs', 'batch_size', 'per', 'fused_td3', 'num_envs', 'independent_references', 'env_name', 'use_caps',
            'seed', 'mut_type')


def identity(args):
    """the IDENTITY fields of a Parameters as plain values"""
    num_envs = getattr(args, 'num_envs', getattr(args, 'num_evals', None))
    out = {}
    for f in IDENTITY:
        v = num_envs if f == 'num_envs' else getattr(args, f, None)
        if f in ('per', 'fused_td3', 'independent_references', 'use_caps'):
            v = bool(v)
        elif isinstance(v, (bool, np.bool_)):
            v = bool(v)
        elif isinstance(v, (int, np.integer)):
            v = int(v)
        elif isinstance(v, str) and f == 'activation_actor':
            v = v.lower()
        out[f] = v
    return out


# ------------------------------------------------------------------------------------------------ file format
def write(obj, path, json_doc=False):
    """torch.save `obj` (json_doc: json.dump it) to `path` atomically: a temporary file in the same directory, flushed and
    fsynced, then renamed over `path`.  If anything fails before the rename, `path` is left as it was and the temporary
    file is removed."""
    path = os.path.abspath(path)
    folder = os.path.dirname(path)
    os.makedirs(folder, exist_ok=True)
    fd, tmp = tempfile.mkstemp(prefix='.' + os.path.basename(path) + '.', suffix='.tmp', dir=folder)
    try:
        with os.fdopen(fd, 'w' if json_doc else 'wb') as f:
            if json_doc:
                json.dump(obj, f, indent=1)
            else:
                torch.save(obj, f)
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise
    try:                                   # make the rename itself durable
        dfd = os.open(folder, os.O_RDONLY)
    except OSError:
        return
    try:
        os.fsync(dfd)
    except OSError:
        pass
    finally:
        os.close(dfd)


def read_json(path):
    """a sweep's manifest (`write(..., json_doc=True)`); ValueError for another format or version"""
    with open(path) as f:
        obj = json.load(f)
    if not isinstance(obj, dict) or obj.get('format') != FORMAT or obj.get('version') != VERSION:
        raise ValueError('checkpoint manifest %s: not a version %d serl_b200 checkpoint manifest' % (path, VERSION))
    return obj


def read(path):
    """the checkpoint dict at `path`; ValueError for another format, an unknown version or a missing completion marker"""
    ck = torch.load(path, map_location='cpu', weights_only=True)
    if not isinstance(ck, dict) or ck.get('format') != FORMAT:
        raise ValueError('checkpoint %s: not a serl_b200 checkpoint' % path)
    if ck.get('version') != VERSION:
        raise ValueError('checkpoint %s: format version %r, this build reads version %d' % (path, ck.get('version'), VERSION))
    if ck.get('complete') is not True:
        raise ValueError('checkpoint %s: no completion marker (the file was not written to the end)' % path)
    return ck


def check(ck, args, world=None):
    """ValueError naming the first field in which the checkpoint cannot continue the run of `args` on `world` ranks"""
    world = engine.world_info()[0] if world is None else int(world)
    if ck['world'] != world:
        raise ValueError('checkpoint: written by a torch.distributed world of %d, this run has %d (world size)'
                         % (ck['world'], world))
    mine = identity(args)
    for f in IDENTITY:
        if ck['params'].get(f) != mine[f]:
            raise ValueError('checkpoint: Parameters.%s is %r in the checkpoint and %r here; only frames may change at a resume'
                             % (f, ck['params'].get(f), mine[f]))


# ------------------------------------------------------------------------------------------------ plain values
def _plain(x):
    """x with numpy arrays as tensors, numpy scalars as Python scalars and device tensors on the CPU (torch.load's
    weights_only reader takes nothing else)"""
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().clone()
    if isinstance(x, np.ndarray):
        return torch.from_numpy(np.array(x))
    if isinstance(x, np.generic):
        return x.item()
    if isinstance(x, dict):
        return {k: _plain(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_plain(v) for v in x)
    return x


def _np_state_out(s):
    name, keys, pos, has_gauss, cached = s
    return [name, torch.from_numpy(np.asarray(keys, dtype=np.int64)), int(pos), int(has_gauss), float(cached)]


def _np_state_in(s):
    name, keys, pos, has_gauss, cached = s
    return (name, keys.numpy().astype(np.uint32), int(pos), int(has_gauss), float(cached))


def _rng_out(s):
    ver, state, gauss_next = s.py           # the SSNE planner hands the stdlib state back with a numpy float cached
    py = (int(ver), tuple(int(x) for x in state), None if gauss_next is None else float(gauss_next))
    return {'py': py, 'np': _np_state_out(s.np), 'torch': s.torch.clone(), 'cuda': None if s.cuda is None else s.cuda.clone()}


def _rng_in(d, s):
    s.py = (d['py'][0], tuple(d['py'][1]), d['py'][2])
    s.np = _np_state_in(d['np'])
    s.torch, s.cuda = d['torch'], d['cuda']
    return s


def _gen_out(g):
    return None if g is None else g.get_state()


def _gen_in(g, state, device, seed):
    """the generator `g` (or, if None, a new one on `device` seeded `seed`, as its owner creates it) set to `state`"""
    if state is None:
        return None
    if g is None:
        g = torch.Generator(device=device)
        g.manual_seed(seed)
    g.set_state(state)
    return g


# ------------------------------------------------------------------------------------------------ pieces of the state
def _replay_out(buf):
    n = len(buf)
    d = {'count': int(buf._count), 'position': int(buf.position), 'gen': _gen_out(buf.gen),
         'rows': None if buf.data is None else buf.data[:n].cpu()}       # rows past len are never read
    if hasattr(buf, 'tree'):
        d.update(tree=None if buf.tree is None else buf.tree.cpu(), frame=int(buf.frame), beta_frames=float(buf.beta_frames))
    return d


def _replay_in(buf, d):
    if d['rows'] is None:
        buf.data, buf.gen = None, None
        if hasattr(buf, 'tree'):
            buf.tree = None
    else:
        buf._alloc()
        buf.data.zero_()
        buf.data[:d['rows'].shape[0]].copy_(d['rows'])
        buf.gen.set_state(d['gen'])
        if hasattr(buf, 'tree'):
            buf.tree.copy_(d['tree'])
    buf._count, buf.position = d['count'], d['position']
    if hasattr(buf, 'tree'):
        buf.frame, buf.beta_frames = d['frame'], d['beta_frames']


def _pbuf_out(b):
    return {'data': None if b.data is None else b.data.cpu(), 'pos': b.pos.cpu(), 'count': b.count.cpu(), 'gen': _gen_out(b.gen)}


def _pbuf_in(b, d):
    if d['data'] is None:
        b.data, b.gen = None, None
    else:
        b._alloc()
        b.data.copy_(d['data'])
        b.gen.set_state(d['gen'])
    b.pos.copy_(d['pos'])
    b.count.copy_(d['count'])


def _learner_out(rl):
    d = {'buffer': _replay_out(rl.buffer), 'critical_buffer': _replay_out(rl.critical_buffer)}
    if hasattr(rl, 'state'):                      # FusedTD3
        d.update(kind='fused', state=rl.state.cpu(), critic_steps=int(rl.critic_steps), actor_steps=int(rl.actor_steps),
                 seed=int(rl.seed))
    else:
        d.update(kind='torch', **{k: _plain(getattr(rl, k).state_dict())
                                  for k in ('actor', 'actor_target', 'critic', 'critic_target', 'actor_optim', 'critic_optim')})
    return d


def _learner_in(rl, d):
    if d['kind'] == 'fused':
        rl.state.copy_(d['state'])                # in place: the four modules' parameters are views into it
        rl.critic_steps, rl.actor_steps, rl.seed = d['critic_steps'], d['actor_steps'], d['seed']
        rl._bump_versions()
    else:
        for k in ('actor', 'actor_target', 'critic', 'critic_target', 'actor_optim', 'critic_optim'):
            getattr(rl, k).load_state_dict(d[k])
    _replay_in(rl.buffer, d['buffer'])
    _replay_in(rl.critical_buffer, d['critical_buffer'])


def _ssne_out(s):
    plan = s.last_plan
    return {'rl_policy': s.rl_policy, 'selection_stats': dict(s.selection_stats), 'current_gen': int(s.current_gen),
            'gen': _gen_out(s._gen), 'mut_gen': _gen_out(getattr(s, '_mut_gen', None)),
            'last_plan': None if plan is None else {'elitist_index': [int(i) for i in plan.elitist_index],
                                                    'new_elitists': [int(i) for i in plan.new_elitists]}}


def _ssne_in(s, d, device, seed):
    s.rl_policy, s.selection_stats, s.current_gen = d['rl_policy'], dict(d['selection_stats']), d['current_gen']
    s._gen = _gen_in(s._gen, d['gen'], device, seed + 2)
    if s.mutate is not None:
        s._mut_gen = _gen_in(s._mut_gen, d['mut_gen'], device, seed + 1)
    s.last_plan = None
    if d['last_plan'] is not None:            # what the next front reads of it: the ranked elites and their clones
        s.last_plan = evo.EvoPlan()
        s.last_plan.elitist_index, s.last_plan.new_elitists = d['last_plan']['elitist_index'], d['last_plan']['new_elitists']


def front_inputs(fr):
    """the host-side inputs of a queued front: every flight's reference draws, the np.random state the exploration noise was
    drawn from, the population's draws"""
    pairs = lambda f: [(lv, st) for lv, st in zip(f.levels, f.starts)]
    d = {'explore': pairs(fr.f_explore), 'noise_state': fr.f_explore.noise_state}
    if fr.f_rlval is not None:
        d['rlval'] = pairs(fr.f_rlval)
    if fr.val_draws is not None:
        d['val_draws'] = list(fr.val_draws)
    if fr.draws is not None:
        d['pop_draws'] = {'levels': fr.draws.levels, 'starts': fr.draws.starts}
    return d


def _front_out(d):
    out = _plain({k: v for k, v in d.items() if k != 'noise_state'})
    out['noise_state'] = _np_state_out(d['noise_state'])
    return out


def _front_in(d):
    draws = lambda lst: [(lv.numpy(), st.numpy()) for lv, st in lst]
    out = {'explore': draws(d['explore']), 'noise_state': _np_state_in(d['noise_state'])}
    if 'rlval' in d:
        out['rlval'] = draws(d['rlval'])
    if 'val_draws' in d:
        out['val_draws'] = draws(d['val_draws'])
    if 'pop_draws' in d:
        p = agent_mod._PopDraws()
        p.levels, p.starts = d['pop_draws']['levels'].numpy(), d['pop_draws']['starts'].numpy()
        out['pop_draws'] = p
    return out


# ------------------------------------------------------------------------------------------------ Agent
def capture(agent, rng=None, extra=None):
    """the checkpoint dict of `agent` between two train() calls, with the generator states `rng` (sweep.RNGState; None:
    the global generators now)"""
    from .sweep import RNGState
    if agent._front is not None or agent._gen is not None:
        raise RuntimeError('checkpoint: the agent is inside a generation; save between two train() calls')
    torch.cuda.synchronize(agent.device)          # the prefetched front and the last generation's work are done
    rng = RNGState.capture() if rng is None else rng
    a = agent.args
    pop = agent.pop
    fr = agent._prefetched
    ck = {'format': FORMAT, 'version': VERSION, 'world': engine.world_info()[0], 'params': identity(a),
          'frames': int(a.num_frames),
          'counters': {k: int(getattr(agent, k)) for k in ('num_episodes', 'num_frames', 'iterations', 'rl_iteration',
                                                           'spec_tries', 'spec_hits')},
          'champion': None if agent.champion is None else int(agent.champion.index),
          'champion_history': _plain(agent.champion_history), 'rl_history': _plain(agent.rl_history),
          'population': None, 'ssne': None,
          'replay': _replay_out(agent.replay_buffer), 'rl': _learner_out(agent.rl_agent),
          # a front whose inputs changed since its launch is flown again by the next train(): nothing of it to keep
          'front': _front_out(front_inputs(fr)) if fr is not None and fr.signature == agent._signature() else None,
          'rng': _rng_out(rng), 'extra': _plain(extra)}
    if len(pop):
        ck['population'] = {'genomes': pop.genomes.cpu(), 'buffers': _pbuf_out(pop.buffers),
                            'critical_buffers': _pbuf_out(pop.critical_buffers)}
        ck['ssne'] = _ssne_out(agent.evolver)
    ck['complete'] = True
    return ck


def save(agent, path, rng=None, extra=None):
    """write `agent`'s checkpoint to `path` (rank 0 of a torch.distributed world; the other ranks wait for it)"""
    world, rank = engine.world_info()
    if rank == 0:
        write(capture(agent, rng, extra), path)
    else:
        torch.cuda.synchronize(agent.device)
    if world > 1:
        torch.distributed.barrier()


def apply(agent, ck, rng=None):
    """put the checkpoint dict `ck` (already checked) into `agent`; the generator states go to the globals, or into the
    sweep.RNGState `rng`.  Returns the checkpoint's `extra`."""
    from .sweep import RNGState
    torch.cuda.synchronize(agent.device)          # nothing of the fresh agent may still be in flight
    agent._prefetched = agent._front = agent._gen = None
    seed = int(getattr(agent.args, 'seed', 7))
    if ck['population'] is not None:
        p = ck['population']
        agent.pop.genomes.copy_(p['genomes'])
        _pbuf_in(agent.pop.buffers, p['buffers'])
        _pbuf_in(agent.pop.critical_buffers, p['critical_buffers'])
        _ssne_in(agent.evolver, ck['ssne'], agent.pop.genomes.device, seed)
    _replay_in(agent.replay_buffer, ck['replay'])
    _learner_in(agent.rl_agent, ck['rl'])
    for k, v in ck['counters'].items():
        setattr(agent, k, v)
    agent.champion = agent.pop[ck['champion']] if ck['champion'] is not None else None
    agent.champion_actor = agent.champion.actor if agent.champion is not None else None
    hist = lambda h: None if h is None else h.numpy()
    agent.champion_history, agent.rl_history = hist(ck['champion_history']), hist(ck['rl_history'])
    if ck['front'] is not None:
        # the front the saved run had queued, re-launched from its draws (nothing is drawn from the global generators)
        agent._prefetched = agent._launch_front(_front_in(ck['front']))
    if rng is None:
        _rng_in(ck['rng'], RNGState()).restore()
    else:
        _rng_in(ck['rng'], rng)
    return ck['extra']


def load(agent, path, rng=None):
    """continue the run saved at `path` in `agent` (built fresh from the same Parameters and env); refusals come before
    anything is written.  Returns the `extra` the checkpoint was saved with."""
    ck = read(path)
    check(ck, agent.args)
    return apply(agent, ck, rng)
