"""Bootstrapped DQN on the device-resident uint8 pixel env -- the torchrl_b200 counterpart of the reference's
bootstrapped_dqn.json setup (same flags, same JSON schema; the reference ships no working launcher for it).

    python examples/bootstrapped_dqn_atari_vec.py --config config/bootstrapped_dqn_synth_atari.json --vec_env_nums 512

The replay ring is frame-de-duplicated (one frame of obs and one of next_obs per transition), and every transition
carries its Bernoulli mask over the heads.  `batch_size` counts transitions; rows of all envs are sampled together,
so it must be a multiple of --vec_env_nums.
"""
import torch

from _common import Run, main  # noqa: F401  (also puts the repository root on sys.path)
import torchrl_b200.networks as networks
import torchrl_b200.policies as policies
from torchrl_b200.algo import BootstrappedDQN
from torchrl_b200.collector import PixelVecCollector
from torchrl_b200.replay_buffers import MemoryEfficientReplayBuffer


def experiment(run):
    cfg = run.params
    algo = dict(cfg["bootstrapped_dqn"])
    head_num = algo["head_num"]
    qf = networks.BootstrappedNet(input_shape=tuple(run.env.observation_space.shape), output_shape=run.act_dim,
                                  base_type=networks.CNNBase, activation_func=torch.nn.ReLU, head_num=head_num,
                                  **cfg["net"])
    pf = policies.BootstrappedDQNDiscretePolicy(qf=qf, head_num=head_num, action_shape=run.act_dim, **cfg["policy"])
    ring = MemoryEfficientReplayBuffer(**run.buffer_kwargs())
    collector = PixelVecCollector(**run.collector_kwargs(pf, ring))
    BootstrappedDQN(qf=qf, pf=pf, **algo, **run.agent_kwargs(ring, collector)).train()


if __name__ == "__main__":
    main(experiment)
