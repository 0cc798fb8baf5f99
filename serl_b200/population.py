"""Device-resident population: one [pop, P] fp32 genome matrix owned by the engine (SURVEY.md 8(b) "Ownership").

`PopulationList` is the `Agent.pop` the reference code indexes / iterates (agent.py:21-24): a plain list of GeneticAgent
whose actors are views into the matrix.  Construction order matches the reference (Actor(args) pop times after
torch.manual_seed, base/train.py:89, agent.py:23-24), so the initial genomes are the ones the reference would draw.
"""
import torch

from .core import genetic_agent, replay_memory
from . import rollout


class PopulationList(list):
    def __init__(self, args, device=None):
        super().__init__()
        self.args = args
        self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.shape = rollout.actor_shape(args.hidden_size, args.num_layers, args.activation_actor, args.state_dim, args.action_dim)
        self.shape_tuple = (args.state_dim, args.action_dim, args.hidden_size, args.num_layers)
        P = rollout.num_params(self.shape)
        agents = [genetic_agent.GeneticAgent(args) for _ in range(args.pop_size)]     # CPU init, reference RNG order
        self.genomes = torch.empty((args.pop_size, P), dtype=torch.float32, device=self.device)
        for i, a in enumerate(agents):
            self.genomes[i].copy_(a.actor.flat())
            a.actor.bind(self.genomes[i])
            a.index = i
        # GeneticAgent.buffer / .critical_buffer of every actor: two device tensors, allocated on first use
        self.buffers = replay_memory.PopulationBuffers(args.pop_size, args.individual_bs, self.device, args.state_dim, args.action_dim)
        self.critical_buffers = replay_memory.PopulationBuffers(args.pop_size, args.individual_bs, self.device, args.state_dim,
                                                                args.action_dim)
        for i, a in enumerate(agents):
            a.buffer = replay_memory.ActorBuffer(self.buffers, i)
            a.critical_buffer = replay_memory.ActorBuffer(self.critical_buffers, i)
        self.extend(agents)

    def isEmpty(self):            # the reference calls this on its (list) population (agent.py:326)
        return len(self) == 0
