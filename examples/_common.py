"""Shared wiring of the example launchers: device, env pair, seeding, run directory / logger and the keyword
dictionaries the agents take (the JSON schema and command-line flags are the reference's, SURVEY.md Appendix B)."""
import os
import os.path as osp
import random
import sys

import numpy as np
import torch

sys.path.append(osp.join(osp.dirname(osp.abspath(__file__)), ".."))
from torchrl_b200.env import get_vec_env  # noqa: E402
from torchrl_b200.utils import Logger, get_args, get_params  # noqa: E402


class Run:
    """Everything an example needs before it builds its networks."""

    def __init__(self, args, params):
        if not args.cuda:
            raise SystemExit("torchrl_b200 needs a CUDA device (there is no CPU path)")
        self.args, self.params = args, params
        self.device = torch.device("cuda:{}".format(args.device))
        self.n_envs = args.vec_env_nums
        make = lambda: get_vec_env(params["env_name"], params["env"], self.n_envs, device=self.device)  # noqa: E731
        self.env, self.eval_env = make(), make()
        self.seed_everything(args.seed)
        name = args.id if args.id is not None else osp.splitext(osp.basename(args.config))[0]
        self.logger = Logger(name, params["env_name"], args.seed, params, args.log_dir, args.overwrite)
        self.obs_dim = self.env.observation_space.shape[0]
        space = self.env.action_space
        self.act_dim = space.n if hasattr(space, "n") else space.shape[0]     # discrete: the number of actions

    def seed_everything(self, seed):
        self.env.seed(seed)
        torch.manual_seed(seed)
        np.random.seed(seed)
        random.seed(seed)
        torch.cuda.manual_seed_all(seed)

    def buffer_kwargs(self):
        cfg = self.params["replay_buffer"]
        return dict(env_nums=self.n_envs, max_replay_buffer_size=int(cfg["size"]),
                    time_limit_filter=cfg["time_limit_filter"])

    def collector_kwargs(self, pf, replay_buffer):
        return dict(env=self.env, eval_env=self.eval_env, pf=pf, replay_buffer=replay_buffer, device=self.device,
                    train_render=False, **self.params["collector"])

    def agent_kwargs(self, replay_buffer, collector):
        general = dict(self.params["general_setting"])
        general.update(env=self.env, replay_buffer=replay_buffer, logger=self.logger, device=self.device,
                       collector=collector, save_dir=osp.join(self.logger.work_dir, "model"))
        return general


def main(experiment):
    args = get_args()
    experiment(Run(args, get_params(args.config)))
