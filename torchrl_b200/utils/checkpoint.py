"""Full training-state checkpoint and RESUME (SURVEY.md 8(f).2; the reference only writes model_*.pth and
the obs normaliser, /root/reference/torchrl/algo/rl_algo.py:83-94, and has no way back in).

`save_checkpoint(agent, path)` captures everything the next epoch depends on: network weights, Adam
moments and step counts, target networks, algorithm scalars (e.g. SAC's log-alpha), the collector's
carried observation / per-env step counters / episode returns, the device env's state, the observation
normaliser, the replay ring (optional for on-policy agents), every RNG stream (NumPy global, torch CPU,
torch CUDA, the device Philox (seed, counter) pairs) and the host counters.

`load_checkpoint(agent, path)` copies it back IN PLACE (storage addresses do not change, so captured CUDA
graphs stay valid) into an agent that was constructed with the same configuration.
"""
import numpy as np
import torch

FORMAT = 1
_AGENT_SCALARS = ("current_epoch", "training_update_num", "best_eval", "pretrain_frames", "total_frames")
_COLLECTOR_SCALARS = ("_host_step", "_host_steps")
_ENV_SCALARS = ("_host_elapsed", "_host_mirror_ok", "training")
_BUFFER_SCALARS = ("_top", "_size")
_POLICY_SCALARS = ("count", "epsilon")                 # epsilon-greedy schedule position
_POLICY_TENSORS = ("head",)                            # Bootstrapped DQN: the per-env heads
_OPT_TENSORS = ("exp_avg", "exp_avg_sq", "step_counts", "lr_host", "lr")


def _tensors(obj, skip=()):
    return {k: v.detach().to("cpu", copy=True) for k, v in vars(obj).items()
            if torch.is_tensor(v) and k not in skip}


def _scalars(obj, names):
    return {k: getattr(obj, k) for k in names if hasattr(obj, k)}


def _rng_holders(agent):
    """(name, _DeviceRng) of every device Philox stream the run consumes.  Policies create theirs lazily on
    the first sampling launch, so a freshly built agent is asked to create it now."""
    out = []
    for name in ("pf", "target_pf"):
        m = getattr(agent, name, None)
        if m is None:
            continue
        if hasattr(m, "_rng_state"):
            out.append((name + "._rng", m._rng_state(agent.device)))
        elif getattr(m, "_rng", None) is not None:
            out.append((name + "._rng", m._rng.ensure(agent.device)))
    if getattr(agent, "_rng", None) is not None:
        out.append(("agent._rng", agent._rng.ensure(agent.device)))
    return out


def save_checkpoint(agent, path, include_replay=None):
    col, rb = agent.collector, agent.replay_buffer
    env = col.env
    if include_replay is None:
        include_replay = not getattr(col, "on_policy", False)    # an on-policy ring is refilled every epoch
    state = {"format": FORMAT, "algo": type(agent).__name__}
    state["networks"] = [n.state_dict() for n in agent.networks]
    state["opt"] = {k: getattr(agent.opt, k).detach().to("cpu", copy=True) for k in _OPT_TENSORS}
    state["agent_tensors"] = _tensors(agent)
    state["agent_scalars"] = _scalars(agent, _AGENT_SCALARS)
    state["episode_rewards"] = list(agent.episode_rewards)
    state["training_episode_rewards"] = list(agent.training_episode_rewards)
    state["policy_scalars"] = _scalars(agent.pf, _POLICY_SCALARS)
    state["policy_tensors"] = {k: v.detach().to("cpu", copy=True) for k, v in _scalars(agent.pf, _POLICY_TENSORS).items()
                               if torch.is_tensor(v)}
    state["collector_tensors"] = _tensors(col)
    state["collector_scalars"] = _scalars(col, _COLLECTOR_SCALARS)
    state["env_tensors"] = _tensors(env)
    state["env_scalars"] = _scalars(env, _ENV_SCALARS)
    nrm = getattr(env, "_obs_normalizer", None)
    state["normalizer"] = _tensors(nrm) if nrm is not None else None
    storage = tuple("_" + k for k in getattr(rb, "_keys", ())) + ("_advs", "_estimate_returns", "_old_logp")
    state["buffer_tensors"] = _tensors(rb, skip=() if include_replay else storage)
    state["buffer_scalars"] = _scalars(rb, _BUFFER_SCALARS)
    state["rng"] = {
        "numpy": np.random.get_state(),
        "torch_cpu": torch.get_rng_state(),
        "torch_cuda": torch.cuda.get_rng_state(agent.device),
        "philox": {name: (r.seed, None if r.counter is None else int(r.counter.item()))
                   for name, r in _rng_holders(agent)},
    }
    torch.save(state, path)
    return path


def _restore(obj, saved, what, device=None):
    """Copy saved tensors into the live object's tensors IN PLACE.  A saved tensor whose destination does not exist
    yet (state the object allocates lazily: replay keys, priorities, ...) is materialised with the saved shape on
    `device`; a destination of another kind is an error -- nothing is dropped silently."""
    for k, v in saved.items():
        dst = getattr(obj, k, None)
        if dst is None and device is not None:
            setattr(obj, k, v.to(device, copy=True))
            continue
        if not torch.is_tensor(dst):
            raise ValueError("checkpoint/%s.%s is a tensor but the agent holds %r there" % (what, k, type(dst)))
        if tuple(dst.shape) != tuple(v.shape):
            raise ValueError("checkpoint/%s.%s has shape %s, the agent expects %s -- different configuration"
                             % (what, k, tuple(v.shape), tuple(dst.shape)))
        dst.copy_(v)


def load_checkpoint(agent, path):
    state = torch.load(path, map_location="cpu", weights_only=False)
    if state.get("format") != FORMAT:
        raise ValueError("unknown checkpoint format %r" % (state.get("format"),))
    if state["algo"] != type(agent).__name__:
        raise ValueError("checkpoint was written by %s, not %s" % (state["algo"], type(agent).__name__))
    col, rb = agent.collector, agent.replay_buffer
    env = col.env
    with torch.no_grad():
        for net, sd in zip(agent.networks, state["networks"]):
            net.load_state_dict(sd)                    # in-place copies: flat-buffer views stay intact
        for k, v in state["opt"].items():
            getattr(agent.opt, k).copy_(v)
        agent.opt.grad.zero_()
        dev = agent.device
        _restore(agent, state["agent_tensors"], "agent", dev)
        _restore(col, state["collector_tensors"], "collector", dev)
        _restore(env, state["env_tensors"], "env", dev)
        if state["normalizer"] is not None:
            _restore(env._obs_normalizer, state["normalizer"], "normalizer", dev)
        if hasattr(rb, "_ensure_prio"):
            rb._ensure_prio()                          # prioritised ring: priorities exist before they are restored
        _restore(rb, state["buffer_tensors"], "buffer", dev)
        _restore(agent.pf, state.get("policy_tensors", {}), "policy", dev)
    for f in (getattr(agent, "opt", None), getattr(agent, "_target_flat", None)):
        if f is not None and hasattr(f, "refresh_split"):
            f.refresh_split()                          # TF32 planes follow the restored weights
    for obj, key in ((agent, "agent_scalars"), (col, "collector_scalars"), (env, "env_scalars"),
                     (rb, "buffer_scalars"), (agent.pf, "policy_scalars")):
        for k, v in state[key].items():
            setattr(obj, k, v)
    agent.episode_rewards.clear()
    agent.episode_rewards.extend(state["episode_rewards"])
    agent.training_episode_rewards.clear()
    agent.training_episode_rewards.extend(state["training_episode_rewards"])
    rng = state["rng"]
    np.random.set_state(rng["numpy"])
    torch.set_rng_state(rng["torch_cpu"])
    torch.cuda.set_rng_state(rng["torch_cuda"], agent.device)
    for name, r in _rng_holders(agent):
        seed, ctr = rng["philox"].get(name, (None, None))
        if seed is None:
            continue
        r.ensure(agent.device)
        r.seed = seed
        r.counter.fill_(ctr)
    return state["agent_scalars"].get("current_epoch", 0)
