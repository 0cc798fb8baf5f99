"""Checkpoint format on the CPU (serl_b200/checkpoint.py): a synthetic state round-trips, every refusal fires before the
agent is touched, an interrupted write leaves the previous checkpoint loadable, and the example drivers' -checkpoint_every /
-resume flags parse without changing Parameters.save_periodic."""
import copy
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch

from serl_b200 import checkpoint
from serl_b200.parameters import Parameters

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def args(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                  # Parameters makes ./tmp/
    p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=4, mut_type='normal', fused_td3=True))
    p.state_dim, p.action_dim = 7, 3
    return p


def synthetic(args, **over):
    ck = {'format': checkpoint.FORMAT, 'version': checkpoint.VERSION, 'world': 1, 'params': checkpoint.identity(args),
          'frames': int(args.num_frames), 'counters': {'num_frames': 12345, 'iterations': 3},
          'genomes': torch.randn(4, 9), 'gen': torch.Generator().get_state(), 'rows': torch.arange(12, dtype=torch.float64),
          'tree': torch.tensor([1.0, float('inf'), float('nan')], dtype=torch.float64), 'champion': None,
          'py': (3, tuple(range(625)), None), 'extra': {'stats': {'elite_index': 2, 'TD_loss': float('nan')}}}
    ck.update(over)
    ck['complete'] = True
    return ck


def same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and \
            bool(torch.equal(a.view(torch.uint8), b.view(torch.uint8)))
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, float) and np.isnan(a):
        return isinstance(b, float) and np.isnan(b)
    return a == b


class Untouchable:
    """an Agent stand-in that only has `args`: load must refuse before it reads or writes anything else"""

    def __init__(self, args):
        object.__setattr__(self, 'args', args)

    def __getattr__(self, name):
        raise AssertionError('load read agent.%s before refusing' % name)

    def __setattr__(self, name, value):
        raise AssertionError('load wrote agent.%s before refusing' % name)


def test_synthetic_state_round_trips(args, tmp_path):
    ck = synthetic(args)
    path = tmp_path / 'ck.pt'
    checkpoint.write(ck, path)
    assert same(checkpoint.read(path), ck)
    assert not [f for f in os.listdir(tmp_path) if f.endswith('.tmp')]


def test_plain_values_load_with_weights_only(tmp_path):
    state = np.random.RandomState(3).get_state()
    obj = checkpoint._plain({'a': np.arange(5.0), 'b': np.float64(2.5), 'c': [np.int64(4)], 'd': (np.zeros((2, 6)),)})
    obj['np'] = checkpoint._np_state_out(state)
    torch.save(obj, tmp_path / 'x.pt')
    back = torch.load(tmp_path / 'x.pt', weights_only=True)
    assert back['b'] == 2.5 and back['c'] == [4] and torch.equal(back['a'], torch.arange(5.0, dtype=torch.float64))
    s = checkpoint._np_state_in(back['np'])
    assert s[0] == state[0] and np.array_equal(s[1], state[1]) and s[1].dtype == np.uint32 and s[2:] == state[2:]
    rs = np.random.RandomState()
    rs.set_state(s)
    assert np.array_equal(rs.randn(7), np.random.RandomState(3).randn(7))


def test_frames_alone_may_differ(args):
    ck = synthetic(args)
    longer = copy.copy(args)
    longer.num_frames = 3 * args.num_frames
    checkpoint.check(ck, longer, world=1)


CHANGES = {'pop_size': 5, 'hidden_size': 96, 'num_layers': 2, 'activation_actor': 'relu', 'state_dim': 10, 'action_dim': 1,
           'buffer_size': 1000, 'individual_bs': 500, 'batch_size': 64, 'per': True, 'fused_td3': False, 'num_envs': 5,
           'independent_references': True, 'env_name': 'PHlab_attitude_be', 'use_caps': False, 'seed': 8, 'mut_type': 'proximal'}


def test_every_identity_field_has_a_case():
    assert set(CHANGES) == set(checkpoint.IDENTITY)


@pytest.mark.parametrize('field', sorted(CHANGES))
def test_parameters_mismatch_refused_before_anything_is_written(args, tmp_path, field):
    path = tmp_path / 'ck.pt'
    checkpoint.write(synthetic(args), path)
    other = copy.copy(args)
    setattr(other, field, CHANGES[field])
    with pytest.raises(ValueError, match=r'Parameters\.%s\b' % field):
        checkpoint.load(Untouchable(other), path)


@pytest.mark.parametrize('change, message', [({'version': checkpoint.VERSION + 1}, 'version'),
                                             ({'format': 'something else'}, 'not a serl_b200 checkpoint'),
                                             ({'world': 2}, 'world size')])
def test_file_refused_before_anything_is_written(args, tmp_path, change, message):
    path = tmp_path / 'ck.pt'
    checkpoint.write(synthetic(args, **change), path)
    with pytest.raises(ValueError, match=message):
        checkpoint.load(Untouchable(args), path)


def test_missing_completion_marker_refused(args, tmp_path):
    ck = synthetic(args)
    del ck['complete']
    path = tmp_path / 'ck.pt'
    torch.save(ck, path)
    with pytest.raises(ValueError, match='completion marker'):
        checkpoint.load(Untouchable(args), path)


def test_interrupted_write_leaves_the_previous_checkpoint(args, tmp_path, monkeypatch):
    folder = tmp_path / 'run'
    path = folder / 'checkpoint.pt'
    first = synthetic(args, counters={'num_frames': 1})
    checkpoint.write(first, path)

    def boom(src, dst):
        raise OSError('interrupted')
    monkeypatch.setattr(checkpoint.os, 'replace', boom)
    with pytest.raises(OSError, match='interrupted'):
        checkpoint.write(synthetic(args, counters={'num_frames': 2}), path)
    monkeypatch.undo()
    assert os.listdir(folder) == ['checkpoint.pt']                      # no temporary file left behind
    assert same(checkpoint.read(path), first)


def test_manifest_round_trips_and_refuses_other_versions(tmp_path):
    m = {'format': checkpoint.FORMAT, 'version': checkpoint.VERSION, 'runs': 2, 'params': [{'seed': 7}, {'seed': 8}]}
    checkpoint.write(m, tmp_path / 'manifest.json', json_doc=True)
    assert checkpoint.read_json(tmp_path / 'manifest.json') == m
    checkpoint.write(dict(m, version=checkpoint.VERSION + 1), tmp_path / 'manifest.json', json_doc=True)
    with pytest.raises(ValueError, match='manifest'):
        checkpoint.read_json(tmp_path / 'manifest.json')


def _example(name):
    """the example module, loaded under a private name; sweep.py adds its flags to train.py's parser, so the `train`
    module it imports is dropped again and leaves no parser with those flags behind for later imports"""
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    had_train = sys.modules.get('train')
    try:
        spec = importlib.util.spec_from_file_location('example_' + name, os.path.join(ROOT, 'examples', name + '.py'))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        sys.path.remove(os.path.join(ROOT, 'examples'))
        if had_train is None:
            sys.modules.pop('train', None)
        else:
            sys.modules['train'] = had_train


@pytest.mark.parametrize('name', ['train', 'sweep'])
def test_example_flags_parse(name, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    parser = _example(name).parser
    cla = parser.parse_args(['-frames', '1000'])
    assert cla.checkpoint_every == 0 and cla.resume is None
    cla = parser.parse_args(['-frames', '1000', '-checkpoint_every', '5', '-resume', 'tmp/checkpoint.pt'])
    assert cla.checkpoint_every == 5 and cla.resume == 'tmp/checkpoint.pt'
    # the new flags are not the reference's -save_periodic, whose mere presence sets Parameters.save_periodic
    assert not hasattr(cla, 'save_periodic')
    assert Parameters(cla).save_periodic is False


def test_save_periodic_keeps_the_reference_hasattr_quirk(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    assert Parameters(types.SimpleNamespace(save_periodic=False)).save_periodic is True
    assert Parameters(types.SimpleNamespace()).save_periodic is False
