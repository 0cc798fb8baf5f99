"""Run the REFERENCE's proximal mutation (base/core/mod_neuro_evo.py SSNE.proximal_mutate) and distillation step
(base/core/genetic_agent.py GeneticAgent.update_parameters) on the inputs tests/test_evo_prox.py rebuilds from seeds, and
record what they computed: run once where the reference tree exists, output tests/golden/evo_ref_kat.npz.

  prox_mag                   the mutation magnitude of the reference's parameters for mut_type = proximal
  prox_G_ref / distil_G_ref  the mutated / trained genomes [3, P] at the columns SAMPLE_COLS (a seeded sample)
  prox_moved / distil_moved  max |genome after - genome before| over ALL columns
  distil_mse                 the three MSE values update_parameters returns
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
REF = '/root/reference/base'
OUT = os.path.join(ROOT, 'tests', 'golden', 'evo_ref_kat.npz')


def reference_modules():
    saved = {k: sys.modules.pop(k) for k in list(sys.modules) if k == 'core' or k.startswith('core.') or k == 'parameters'}
    sys.path.insert(0, REF)
    try:
        from core import mod_neuro_evo as ne, genetic_agent as ga
        from parameters import Parameters
        return ne, ga, Parameters
    finally:
        sys.path.remove(REF)
        for k in [k for k in sys.modules if k == 'core' or k.startswith('core.') or k == 'parameters']:
            del sys.modules[k]
        sys.modules.update(saved)


def main():
    import test_evo_prox as T
    import torch.distributions as dist
    os.chdir(tempfile.mkdtemp())          # the reference's Parameters may write files next to it
    ne, ga, RefP = reference_modules()
    args = RefP(types.SimpleNamespace(pop_size=4, mut_type='proximal', env='x', frames=1, seed=1, disable_cuda=True))
    args.state_dim, args.action_dim, args.device = 7, 3, torch.device('cpu')
    assert (args.hidden_size, args.num_layers, args.activation_actor) == (72, 3, 'tanh')
    flat = lambda g: torch.cat([p.data.reshape(-1) for p in g.actor.parameters()])
    out = {'prox_mag': np.array(args.mutation_mag)}

    # proximal mutation of three actors, each with its own batch of states
    torch.manual_seed(0)
    genes = [ga.GeneticAgent(args) for _ in range(3)]
    G = torch.stack([flat(g) for g in genes])
    states = torch.randn(3, 32, 7) * 0.1
    G_in, states_in, deltas_in = T.proximal_inputs(args.mutation_mag)
    assert torch.equal(G, G_in) and torch.equal(states, states_in)          # the test rebuilds the same inputs
    ssne = ne.SSNE(args, None, None)

    class FakeBuf:
        def __init__(self, st):
            self.st = st

        def __len__(self):
            return 32

        def sample(self, n):
            return (self.st, None, None, None, None)
    for k, g in enumerate(genes):
        g.buffer = FakeBuf(states[k])
        tot = g.actor.count_parameters()
        torch.manual_seed(100 + k)
        assert torch.equal(dist.Normal(torch.zeros(tot), torch.ones(tot) * args.mutation_mag).sample(), deltas_in[k])
        torch.manual_seed(100 + k)
        ssne.proximal_mutate(g, mag=args.mutation_mag)
    G_ref = torch.stack([flat(g) for g in genes])
    out['prox_G_ref'] = G_ref[:, T.SAMPLE_COLS].numpy()
    out['prox_moved'] = np.array((G_ref - G).abs().max().item())

    # one Q-filtered behaviour-cloning Adam step for three children
    torch.manual_seed(0)
    kids = [ga.GeneticAgent(args) for _ in range(3)]
    p1s = [ga.GeneticAgent(args) for _ in range(3)]
    p2s = [ga.GeneticAgent(args) for _ in range(3)]
    lin = torch.nn.Linear(10, 2)
    states = torch.randn(3, 40, 7) * 0.2
    G0_in, G1_in, G2_in, lin_in, states_in = T.distillation_inputs()
    assert torch.equal(torch.stack([flat(k) for k in kids]), G0_in) and torch.equal(torch.stack([flat(p) for p in p2s]), G2_in)
    assert torch.equal(states, states_in) and torch.equal(lin.weight, lin_in.weight)
    G0 = torch.stack([flat(k) for k in kids])

    def critic(s, a):
        q = lin(torch.cat((s, a), 1))
        return q[:, :1], q[:, 1:]
    mse = [kids[c].update_parameters((states[c], None, None, None, None), p1s[c].actor, p2s[c].actor, critic) for c in range(3)]
    G_ref = torch.stack([flat(k) for k in kids])
    out['distil_G_ref'] = G_ref[:, T.SAMPLE_COLS].numpy()
    out['distil_moved'] = np.array((G_ref - G0).abs().max().item())
    out['distil_mse'] = np.array(mse, dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
