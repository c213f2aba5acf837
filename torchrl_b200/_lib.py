"""ctypes binding of libtorchrl_b200.so (the C ABI declared in include/torchrl_b200.h).

There is NO fallback: if the shared object is missing or a symbol is absent the import
of any op raises.  ``load()`` only dlopens the library -- it needs libcudart's static
copy inside the .so but no GPU, so the symbol/ABI checks run on CPU boxes too.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtorchrl_b200.so")

c_f32p = ctypes.c_void_p
c_u8p = ctypes.c_void_p
c_i32p = ctypes.c_void_p
c_i64p = ctypes.c_void_p
c_f64p = ctypes.c_void_p
vp = ctypes.c_void_p
i64 = ctypes.c_int64
i32 = ctypes.c_int
f32 = ctypes.c_float
f64 = ctypes.c_double
u64 = ctypes.c_uint64
u32 = ctypes.c_uint32

# name -> argtypes   (restype is int unless listed in _RESTYPES)
SIGNATURES = {
    "trl_last_error": [],
    "trl_abi_version": [],
    "trl_device_info": [vp, vp, vp],
    "trl_gae_scan": [vp, vp, vp, vp, vp, vp, vp, i64, i64, f32, f32, i32, i32, vp],
    "trl_discount_return": [vp, vp, vp, vp, vp, vp, vp, i64, i64, f32, i32, i32, vp],
    "trl_synth_env_smem_bytes": [i32, i32],
    "trl_synth_env_num_ctas": [i64],
    "trl_synth_env_step": [vp] * 20 + [i64, i32, i32, f32, f32, f32, f32, f32, i32, i32, i32, vp],
    "trl_synth_env_reset": [vp, vp, vp, vp, vp, i64, i32, f64, vp],
    "trl_synth_env_seed": [vp, vp, i64, u32, u32, u32, vp],
    "trl_obs_norm_moments": [vp, i64, i32, vp, vp],
    "trl_obs_norm_merge": [vp, f64, i32, vp, vp, vp, vp],
    "trl_obs_norm_filt": [vp, vp, vp, i64, i32, f64, vp, vp],
    "trl_tanh_gaussian_sample": [vp, vp, i32, vp, f32, u64, vp, i64, i32, i32, vp, vp, vp, vp, vp, vp],
    "trl_tanh_gaussian_sample_bwd": [vp, vp, vp, i32, vp, vp, i64, i32, i32, vp, vp, vp],
    "trl_collect_finalize": [vp] * 29 + [i64, i32, i32, i32, f32, f64, f64, i32, i32, vp],
    "trl_step_advance": [vp, i32, vp, vp, vp],
    "trl_row_gather": [i32, vp, vp, vp, vp, vp, i32, vp],
    "trl_ring_write": [i32, vp, vp, vp, vp, vp],
    "trl_ring_write_advance": [i32, vp, vp, vp, vp, i32, vp, vp, vp],
    "trl_vec_stats": [vp, i64, vp, vp],
    "trl_vec_moments": [vp, i64, vp, vp],
    "trl_vec_stats_from_moments": [vp, i32, f64, vp, vp],
    "trl_row_group_moments": [vp, vp, i32, i32, i64, vp, vp],
    "trl_group_stats_from_moments": [vp, i32, i32, f64, vp, vp],
    "trl_ppo_actor_scratch_doubles": [i64, i32],
    "trl_ppo_actor_loss": [vp, vp, i32, vp, vp, vp, vp, vp, i64, i32, i32, f32, f32, f32, f32, vp, vp, vp, vp, vp, vp, vp],
    "trl_ppo_critic_loss": [vp, vp, vp, i64, i32, f32, vp, vp, vp, vp, vp],
    "trl_gaussian_log_prob": [vp, vp, i32, vp, i64, i32, i32, vp, vp],
    "trl_categorical_sample": [vp, vp, u64, vp, i64, i32, vp, vp, vp, vp],
    "trl_categorical_log_prob": [vp, vp, i64, i32, vp, vp],
    "trl_ppo_categorical_actor_scratch_doubles": [i64],
    "trl_ppo_categorical_actor_loss": [vp, vp, vp, vp, vp, vp, i64, i32, f32, f32, vp, vp, vp, vp, vp, vp],
    "trl_vmpo_select": [vp, vp, i32, i32, i64, vp, vp, vp],
    "trl_vmpo_categorical_scratch_doubles": [i64],
    "trl_vmpo_categorical_loss": [vp, vp, vp, vp, vp, vp, vp, i64, i32, f32, f32, i32, vp, vp, vp, vp, vp, vp],
    "trl_categorical_fisher_vp": [vp, vp, i64, i32, f32, vp, vp],
    "trl_tangent_bias_act": [vp, vp, vp, i64, i32, i64, i32, vp],
    "trl_categorical_surrogate": [vp, vp, vp, vp, i64, i32, vp, vp, vp, vp],
    "trl_grad_sumsq_blocks": [i32],
    "trl_grad_sumsq": [vp, vp, i32, u32, vp, vp, f64, f64, vp, vp, vp],
    "trl_adam_step": [vp, vp, vp, vp, vp, i32, u32, vp, vp, vp, vp, f32, f32, f32, i32, vp, vp, vp],
    "trl_polyak_update": [vp, vp, i64, f32, vp, vp, vp],
    "trl_bias_act_bwd_scratch_floats": [i64, i32],
    "trl_bias_act_fwd": [vp, vp, i64, i32, i32, vp],
    "trl_split_tf32": [vp, i64, vp, vp, vp],
    "trl_bias_act_bwd": [vp, vp, vp, vp, i64, i32, i32, vp, vp, vp],
    "trl_per_sample": [vp, i32, vp, i32, f32, vp, vp, vp],
    "trl_per_scratch_doubles": [i32],
    "trl_per_sample_rows": [vp, i32, vp, vp, vp, i32, f32, vp, vp, vp, vp],
    "trl_per_update": [vp, vp, vp, i32, i32, f32, f32, vp, vp],
    "trl_per_insert": [vp, vp, vp, vp],
    "trl_gemm_tf32x3_nt": [vp, vp, vp, i64, i64, i32, vp, vp, i32, vp],
    "trl_gemm_tf32x3_tn": [vp, vp, vp, i64, i64, i32, vp, vp],
    "trl_transpose_f32": [vp, vp, i64, i32, vp],
    "trl_frame_ring_write": [vp, vp, vp, vp, vp, vp, vp, vp, i64, i32, i64, i32, i32, vp],
    "trl_frame_hist_advance": [vp, vp, i32, vp],
    "trl_frame_stack_gather": [vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, i64, i32, i64, i32, f32, vp, vp, vp],
    "trl_comm_flag_bytes": [],
    "trl_comm_ipc_handle_bytes": [],
    "trl_comm_alloc": [i64, vp],
    "trl_comm_free": [vp],
    "trl_comm_ipc_get": [vp, vp],
    "trl_comm_ipc_open": [vp, vp],
    "trl_comm_ipc_close": [vp],
    "trl_comm_scratch_doubles": [i32],
    "trl_allreduce_grad": [vp, vp, i32, i32, vp, i64, vp, i32, u32, vp, vp, f64, f64, vp, vp, vp, i32, vp],
    "trl_allreduce_f64": [vp, vp, i32, i32, vp, i32, i32, vp, vp],
    "trl_comm_ll_recv_bytes": [i32, i32],
    "trl_allreduce_f64_ll": [vp, vp, i32, i32, vp, i32, i32, i32, vp, vp],
    "trl_gemm3_pair": [vp, vp, vp, vp, i64, i64, i32, vp, i32, vp],
    "trl_gemm3_pair_tn": [vp, vp, vp, i64, i64, i32, vp, vp],
    "trl_gemm3_pair_tn_cluster": [vp, vp, vp, i64, i64, i32, vp, vp, vp],
    "trl_gemm3_pair_dgrad_act_wgrad": [vp, vp, vp, vp, vp, i64, i32, i32, vp, vp],
    "trl_skinny_k_fwd": [vp, vp, vp, vp, i64, i32, i32, i32, vp],
    "trl_skinny_tn_scratch_floats": [i64, i32, i32],
    "trl_skinny_tn": [vp, vp, vp, vp, i64, i32, i32, i32, vp, vp],
    "trl_skinny_n_fwd": [vp, vp, vp, vp, i64, i32, i32, vp],
    "trl_skinny_n_dgrad": [vp, vp, vp, i64, i32, i32, vp],
    "trl_skinny_act_wgrad": [vp, vp, vp, vp, vp, i64, i32, i32, i32, vp, vp],
    "trl_skinny_dgrad_act_scratch_floats": [i64, i32],
    "trl_skinny_n_dgrad_act": [vp, vp, vp, vp, vp, i64, i32, i32, i32, vp, vp],
    "trl_skinny_tn_partial": [vp, vp, i64, i32, i32, i32, vp, vp],
    "trl_skinny_act_wgrad_partial": [vp, vp, vp, i64, i32, i32, i32, vp, vp],
    "trl_skinny_n_dgrad_act_partial": [vp, vp, vp, vp, i64, i32, i32, i32, vp, vp],
    "trl_skinny_reduce_jobs": [i32, vp, vp, vp, vp, vp, vp, vp, vp, vp],
    "trl_skinny_n_dgrad_act_wgrad_partial": [vp, vp, vp, vp, i64, i32, i32, i32, vp, vp, vp],
    "trl_skinny_n_dgrad_act_wgrad": [vp, vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, vp, vp, vp],
    "trl_synth_atari_step": [vp, vp, vp, vp, vp, vp, vp, i64, i32, vp],
    "trl_synth_atari_reset": [vp, vp, vp, vp, vp, vp, vp, i32, i32, i64, vp],
    "trl_u8_to_f32": [vp, vp, i64, f32, vp],
    "trl_cartpole_num_ctas": [i64],
    "trl_cartpole_step": [vp] * 16 + [i64, f32, i32, i32, i32, vp],
    "trl_pendulum_num_ctas": [i64],
    "trl_pendulum_step": [vp] * 17 + [i64, f32, i32, i32, i32, vp],
    "trl_pendulum_reset": [vp] * 13 + [i64, f64, i32, vp],
    "trl_offpolicy_scratch_doubles": [i64],
    "trl_td_target": [vp, vp, vp, vp, vp, vp, f32, f32, i64, vp, vp, vp, vp, vp],
    "trl_td3_smooth_action": [vp, vp, f32, f32, u64, vp, i64, vp, vp],
    "trl_sac_alpha_step": [vp, f32, vp, vp, f32, f32, f32, f32, i64, vp, vp, vp, vp],
    "trl_sac_policy_loss": [vp, vp, vp, vp, f32, i64, vp, vp, vp, vp, vp, vp, vp],
    "trl_sac_v_loss": [vp, vp, vp, vp, vp, f32, i32, i64, vp, vp, vp, vp, vp, vp, vp, vp],
    "trl_twin_mse_loss": [vp, vp, vp, i64, vp, vp, vp, vp, vp, vp],
    "trl_twin_mse_loss_weighted": [vp, vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp],
    "trl_qr_dqn_loss": [vp, vp, vp, vp, vp, vp, i32, i32, i32, f32, f32, i32, vp, vp, vp, vp, vp, vp],
    "trl_bootstrapped_dqn_loss": [vp, vp, vp, vp, vp, vp, i64, i32, i32, f32, vp, vp, vp, vp, vp],
    "trl_bootstrapped_act": [vp, vp, vp, vp, vp, vp, vp, vp, u64, vp, vp, i64, i32, i32, f32, vp],
}
_RESTYPES = {"trl_last_error": ctypes.c_char_p, "trl_ppo_actor_scratch_doubles": ctypes.c_int64,
             "trl_ppo_categorical_actor_scratch_doubles": ctypes.c_int64,
             "trl_vmpo_categorical_scratch_doubles": ctypes.c_int64,
             "trl_offpolicy_scratch_doubles": ctypes.c_int64, "trl_bias_act_bwd_scratch_floats": ctypes.c_int64,
             "trl_skinny_tn_scratch_floats": ctypes.c_int64,
             "trl_skinny_dgrad_act_scratch_floats": ctypes.c_int64, "trl_comm_ll_recv_bytes": ctypes.c_int64}
# entry points that return a value rather than an error code
_VALUE_FUNCS = ("trl_abi_version", "trl_synth_env_smem_bytes", "trl_synth_env_num_ctas", "trl_cartpole_num_ctas",
                "trl_pendulum_num_ctas", "trl_comm_flag_bytes",
                "trl_comm_ipc_handle_bytes", "trl_comm_scratch_doubles", "trl_comm_ll_recv_bytes",
                "trl_ppo_actor_scratch_doubles", "trl_ppo_categorical_actor_scratch_doubles", "trl_vmpo_categorical_scratch_doubles",
                "trl_grad_sumsq_blocks", "trl_per_scratch_doubles")

_lib = None


class NativeLibraryError(RuntimeError):
    pass


def load():
    """dlopen the library once and type every entry point.  Raises if anything is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH) and os.environ.get("TORCHRL_B200_NO_AUTOBUILD") != "1":
        try:                                    # nvcc is part of the image: compile in-tree on first use
            from . import build as _build
            _build.build()
        except Exception as e:                  # noqa: BLE001
            raise NativeLibraryError("%s not found and the in-tree nvcc build failed (%s); there is no CPU "
                                     "fallback" % (LIB_PATH, e)) from e
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "%s not found: build it with `python -m torchrl_b200.build` (there is no CPU fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise NativeLibraryError("symbol %s missing from %s" % (name, LIB_PATH)) from e
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, ctypes.c_int)
    _lib = lib
    return lib


def check(rc, name):
    if rc != 0:
        msg = load().trl_last_error()
        raise RuntimeError("%s failed (rc=%d): %s" % (name, rc, msg.decode() if msg else ""))


_LAUNCHES = 0


def launch_count():
    """Kernels launched through the C ABI so far (graph replays add their captured count)."""
    return _LAUNCHES


def add_launches(n):
    global _LAUNCHES
    _LAUNCHES += int(n)


def call(name, *args, kernels=1):
    """Invoke a kernel-launching entry point, raise on error and count the `kernels` kernels it launched (the
    wrappers in ops.py know that number for each entry point and its arguments)."""
    global _LAUNCHES
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        check(rc, name)
    _LAUNCHES += kernels
