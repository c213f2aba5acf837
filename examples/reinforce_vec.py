"""REINFORCE on the device -- the torchrl_b200 launcher for the reference's Reinforce agent and its reinforce.json
schema (a "reinforce" section; collector settings either in a "collector" section or, as in the reference's
reinforce.json, inside "general_setting").

    python examples/reinforce_vec.py --config config/reinforce_cartpole.json --vec_env_nums 8
    python examples/reinforce_vec.py --config config/reinforce_synth_atari.json --vec_env_nums 8
    python examples/reinforce_vec.py --config config/reinforce_synth_halfcheetah.json --vec_env_nums 4096

The policy follows the env: an MLP for state vectors, the Atari CNN for uint8 frames; a CategoricalDisPolicy for a
Discrete action space, a GuassianContPolicyBasicBias for a Box.  `batch_size` counts transitions; rows of all envs are
taken together, so it must be a multiple of --vec_env_nums.
"""
import os.path as osp

import torch

from _common import Run, main  # noqa: F401  (also puts the repository root on sys.path)
import torchrl_b200.networks as networks
import torchrl_b200.policies as policies
from torchrl_b200.algo import Reinforce
from torchrl_b200.collector import VecOnPolicyCollector
from torchrl_b200.replay_buffers import OnPolicyReplayBuffer

_COLLECTOR_KEYS = ("epoch_frames", "max_episode_frames", "eval_episodes")


def experiment(run):
    cfg = run.params
    general = dict(cfg["general_setting"])
    col_kw = dict(cfg.get("collector", {}))
    for k in _COLLECTOR_KEYS:
        if k in general:
            col_kw[k] = general.pop(k)
    shape = tuple(run.env.observation_space.shape)
    pixel = len(shape) == 3
    net = dict(cfg["net"], base_type=networks.CNNBase if pixel else networks.MLPBase, activation_func=torch.nn.Tanh)
    if hasattr(run.env.action_space, "n"):
        pf = policies.CategoricalDisPolicy(input_shape=shape if pixel else shape[0], output_shape=run.act_dim, **net,
                                           **cfg["policy"])
    else:
        pf = policies.GuassianContPolicyBasicBias(input_shape=shape[0], output_shape=run.act_dim, **net, **cfg["policy"])
    buf_cfg = cfg["replay_buffer"]
    buf = OnPolicyReplayBuffer(env_nums=run.n_envs, max_replay_buffer_size=int(buf_cfg["size"]),
                               time_limit_filter=buf_cfg.get("time_limit_filter", False))
    collector = VecOnPolicyCollector(networks.ZeroNet(), env=run.env, eval_env=run.eval_env, pf=pf, replay_buffer=buf,
                                     device=run.device, train_render=False, discount=general.get("discount", 0.99),
                                     **col_kw)
    general.update(env=run.env, replay_buffer=buf, logger=run.logger, device=run.device, collector=collector,
                   save_dir=osp.join(run.logger.work_dir, "model"))
    Reinforce(pf=pf, **cfg["reinforce"], **general).train()


if __name__ == "__main__":
    main(experiment)
