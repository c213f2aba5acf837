"""Discrete TRPO on the device-resident uint8 pixel env -- the torchrl_b200 counterpart of the reference's
trpo_continuous_vec.py with the CategoricalDisPolicy over the Atari CNN of ppo_discrete_atari_vec.py (same flags,
same JSON schema: a "trpo" section in place of "ppo").

    python examples/trpo_atari_vec.py --config config/trpo_synth_atari.json --vec_env_nums 8

One natural-gradient step per epoch on the whole rollout keeps the policy's CNN graph over all of its rows: the
rollout size (replay_buffer size = epoch_frames) bounds that memory (scripts/trpo_atari_bench.py reports the peak).
`batch_size` counts transitions of the value sweeps; it must be a multiple of --vec_env_nums.
"""
import torch

from _common import Run, main  # noqa: F401  (also puts the repository root on sys.path)
import torchrl_b200.networks as networks
import torchrl_b200.policies as policies
from torchrl_b200.algo import TRPO
from torchrl_b200.collector import VecOnPolicyCollector
from torchrl_b200.replay_buffers import OnPolicyReplayBuffer


def experiment(run):
    cfg = run.params
    net = dict(cfg["net"], base_type=networks.CNNBase, activation_func=torch.nn.Tanh)
    shape = tuple(run.env.observation_space.shape)
    pf = policies.CategoricalDisPolicy(input_shape=shape, output_shape=run.act_dim, **net, **cfg["policy"])
    vf = networks.Net(input_shape=shape, output_shape=1, **net)
    buf = OnPolicyReplayBuffer(**run.buffer_kwargs())
    collector = VecOnPolicyCollector(vf, **run.collector_kwargs(pf, buf))
    TRPO(pf=pf, vf=vf, **cfg["trpo"], **run.agent_kwargs(buf, collector)).train()


if __name__ == "__main__":
    main(experiment)
