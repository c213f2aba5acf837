"""Host cost of eager ops.py wrapper calls: the Python-side checks, the ctypes call and the launch, per call.

    python scripts/host_cost.py [--calls 2000] [--repeats 7]
Tiny operands, so the GPU drains each kernel faster than the host enqueues the next and the timed loop (no
synchronisation inside it) measures the host.  Prints one JSON line: median and minimum microseconds per call of
each wrapper over the repeats, with the GPU's name.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torchrl_b200 import ops  # noqa: E402


def wrappers(dev):
    F64, U8, I32 = torch.float64, torch.uint8, torch.int32
    z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
    T, N, o, a, B = 8, 64, 17, 6, 64
    r, v, last = z(T, N), z(T, N), z(N)
    term, tl = z(T, N, dtype=U8), z(T, N, dtype=U8)
    advs, rets = z(T, N), z(T, N)
    mean, log_std, acts, old_logp, adv = z(B, a), z(a), z(B, a), z(B), z(B)
    scratch = ops.LossScratch(B, a, dev)
    g_mean, g_ls, info = z(B, a), z(a), z(16)
    fin = dict(cur_ob_in=z(N, o), next_norm=z(N, o), state=z(N, o), act=z(N, a), value=z(N), v_next=z(N),
               reward=z(N), done=z(N, dtype=U8), tl=z(N, dtype=U8), elapsed=z(N, dtype=I32), episode=z(N, dtype=I32),
               seeds=z(N, dtype=I32), step_count=z(N, dtype=I32), ep_return=z(N, dtype=F64),
               epoch_reward=z(N, dtype=F64), ret_log=z(T, N), n_done=z(1, dtype=I32), any_reset=z(2, dtype=I32),
               norm_mean=z(o, dtype=F64), norm_var=z(o, dtype=F64), cur_ob_out=z(N, o), b_obs=z(T, N, o),
               b_next_obs=z(T, N, o), b_acts=z(T, N, a), b_values=z(T, N, 1), b_rewards=z(T, N, 1),
               b_terminals=z(T, N, 1, dtype=U8), b_time_limits=z(T, N, 1, dtype=U8), t_ptr=z(1, dtype=I32),
               max_episode_frames=1000, discount=0.99, init_scale=0.1, clip=10.0, terminal_includes_surpass=False,
               raw_obs_after_reset=True)
    x, w, bias, out = z(64, 256), torch.randn(256, 256, device=dev), z(256), z(64, 256)
    planes = ops.split_tf32(w)
    return {
        "gae_scan": lambda: ops.gae_scan(r, v, term, tl, last, 0.99, 0.95, True, advs, rets),
        "ppo_actor_loss": lambda: ops.ppo_actor_loss(mean, log_std, acts, old_logp, adv, None, 0.2, 0.005, True,
                                                     scratch, g_mean, g_ls, info),
        "collect_finalize": lambda: ops.collect_finalize(**fin),
        "gemm3_pair": lambda: ops.gemm3_pair(x, w, out=out, planes=planes, bias=bias, act=1),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("host_cost.py needs a CUDA device")
    dev = torch.device("cuda")
    result = {"gpu": torch.cuda.get_device_name(dev), "calls": args.calls}
    for name, fn in wrappers(dev).items():
        for _ in range(50):
            fn()
        torch.cuda.synchronize()
        us = []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            for _ in range(args.calls):
                fn()
            us.append((time.perf_counter() - t0) / args.calls * 1e6)
            torch.cuda.synchronize()
        us.sort()
        result[name] = {"us_median": round(us[len(us) // 2], 2), "us_min": round(us[0], 2)}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
