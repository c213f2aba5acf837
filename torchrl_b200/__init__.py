"""torchrl_b200 -- H100-native (sm_90a) implementation of the RchalYang/torchrl hot path.

The package mirrors the reference's agent / collector / replay-buffer / env Python API
(reference: /root/reference/torchrl) with all rollout data resident on the GPU and every
op between the policy/value MLPs executed by hand-written CUDA kernels reached through
the C ABI in include/torchrl_b200.h.  No CPU fallback: ops raise if the library is absent.
"""
__version__ = "0.1.0"
