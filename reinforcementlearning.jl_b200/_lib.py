"""ctypes binding of libb200rl.so (include/b200rl.h).  No torch types cross this boundary.

The library is built in-tree by ``build.py`` (nvcc, sm_90a).  There is no CPU fallback: if
the shared object is missing, or no sm_90 (H100) device is usable, calls fail loudly."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# B200RL_LIB: development override (an A/B build from `build.py --variant`); the product path is the in-tree library
SO_PATH = os.environ.get("B200RL_LIB") or os.path.join(HERE, "libb200rl.so")

OK = 0
ERR_INVALID, ERR_CUDA, ERR_UNSUPPORTED, ERR_ACTION, ERR_NCCL, ERR_OOM, ERR_OVERFLOW = -1, -2, -3, -4, -5, -6, -7

ENV_CARTPOLE, ENV_PENDULUM, ENV_MOUNTAINCAR, ENV_CARTPOLE_CONTINUOUS, ENV_MOUNTAINCAR_CONTINUOUS, ENV_ACROBOT = 0, 1, 2, 3, 4, 5
F32, F64 = 0, 1
FIELD_STATE, FIELD_OBS, FIELD_REWARD, FIELD_TERMINAL, FIELD_T, FIELD_RNG, FIELD_FLAGS, FIELD_ACTION, FIELD_EPISODE_RETURN, FIELD_EPISODE_STATS = range(10)
FIELD_OBS_F32 = 10


class B200RLError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"b200rl status {status}: {msg}")
        self.status = status


class CartPoleParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("gravity", "masscart", "masspole", "totalmass", "halflength", "polemasslength",
                                          "forcemag", "dt", "thetathreshold", "xthreshold")] + [("max_steps", C.c_int64)]


class PendulumParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("max_speed", "max_torque", "g", "m", "l", "dt")] + [
        ("max_steps", C.c_int64), ("n_actions", C.c_int64), ("continuous", C.c_int32)]


class NetDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_in", "hidden", "act", "n_out", "kind")]


class OnPolicyConfig(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("gamma", "lambda_", "clip_range", "max_grad_norm", "w_actor", "w_critic", "w_entropy", "lr",
                                         "beta1", "beta2", "eps", "min_sigma", "max_sigma")] + [
        (n, C.c_int32) for n in ("normalize_advantage", "n_epochs", "n_microbatches", "update_freq", "algo")]


class DQNConfig(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("gamma", "lr", "beta1", "beta2", "eps", "max_grad_norm", "rho", "per_alpha", "per_beta",
                                         "per_eps")] + [(n, C.c_int32) for n in ("huber", "double_dqn", "target_update_freq")]


class Explorer(C.Structure):
    """b200rl_explorer: kind (0 :linear, 1 :exp, 2 speedy, 3 weighted softmax, 4 Gumbel softmax), the EpsilonGreedyExplorer
    fields, the step before the call and EpsilonSpeedyExplorer's beta."""
    _fields_ = [("eps_stable", C.c_double), ("eps_init", C.c_double), ("warmup_steps", C.c_int64), ("decay_steps", C.c_int64),
                ("step", C.c_int64), ("kind", C.c_int32), ("is_break_tie", C.c_int32), ("beta", C.c_double)]


class InsertSampleRatio(C.Structure):
    """b200rl_insert_sample_ratio: InsertSampleRatioController's ratio, threshold and counters."""
    _fields_ = [("ratio", C.c_double), ("threshold", C.c_int64), ("n_inserted", C.c_int64), ("n_sampled", C.c_int64)]


class EvalConfig(C.Structure):
    """b200rl_eval_config: mode 0 greedy | 1 sample, window length, records kept per env."""
    _fields_ = [(n, C.c_int32) for n in ("mode", "n_steps", "max_episodes")]


class MountainCarParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("min_pos", "max_pos", "max_speed", "goal_pos", "goal_velocity", "power", "gravity")] + [
        ("max_steps", C.c_int64)]


class AcrobotParams(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("link_length_a", "link_length_b", "link_mass_a", "link_mass_b", "link_com_pos_a", "link_com_pos_b", "link_moi",
                                          "max_torque_noise", "max_vel_a", "max_vel_b", "g", "dt")] + [("max_steps", C.c_int64), ("book", C.c_int32)]


_vp, _i32, _i64, _u64, _f32, _f64, _sz = C.c_void_p, C.c_int, C.c_int64, C.c_uint64, C.c_float, C.c_double, C.c_size_t
_pp = C.POINTER(C.c_void_p)

# name -> (restype, argtypes).  Must list every symbol include/b200rl.h declares
# (tests/test_abi.py checks header <-> table <-> exported symbols).
SIGNATURES = {
    "b200rl_init": (_i32, [_i32, _pp]),
    "b200rl_destroy": (None, [_vp]),
    "b200rl_last_error": (C.c_char_p, []),
    "b200rl_sync": (_i32, [_vp]),
    "b200rl_abi_version": (_i32, []),
    "b200rl_stream": (_i32, [_vp, _pp]),
    "b200rl_timer_start": (_i32, [_vp]),
    "b200rl_timer_stop_ms": (_i32, [_vp, C.POINTER(_f32)]),
    "b200rl_timer_record": (_i32, [_vp, _i32]),
    "b200rl_timer_elapsed_ms": (_i32, [_vp, _i32, _i32, C.POINTER(_f32)]),
    "b200rl_debug_phase_slots": (_i32, [_vp, _i32]),
    "b200rl_malloc": (_i32, [_vp, _sz, _pp]),
    "b200rl_free": (_i32, [_vp, _vp]),
    "b200rl_host_alloc": (_i32, [_vp, _sz, _pp]),
    "b200rl_host_free": (_i32, [_vp, _vp]),
    "b200rl_memcpy_h2d": (_i32, [_vp, _vp, _vp, _sz, _i32]),
    "b200rl_memcpy_d2h": (_i32, [_vp, _vp, _vp, _sz, _i32]),
    "b200rl_memset": (_i32, [_vp, _vp, _i32, _sz]),
    "b200rl_flush_l2": (_i32, [_vp]),
    "b200rl_launch_count": (_i32, [_vp, C.POINTER(_u64)]),
    "b200rl_env_create": (_i32, [_vp, _i32, _i32, _i64, _vp, _vp, _pp]),
    "b200rl_env_destroy": (_i32, [_vp]),
    "b200rl_env_set_max_timeout": (_i32, [_vp, _i64]),
    "b200rl_env_set_state_f32": (_i32, [_vp, _i32]),
    "b200rl_env_copy": (_i32, [_vp, _pp]),
    "b200rl_env_seed": (_i32, [_vp, _vp]),
    "b200rl_env_reset": (_i32, [_vp, _i32]),
    "b200rl_env_step": (_i32, [_vp, _vp, _i32, _i32]),
    "b200rl_env_step_random": (_i32, [_vp, _i32]),
    "b200rl_env_get": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_env_set": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_env_ptr": (_i32, [_vp, _i32, _pp]),
    "b200rl_env_check": (_i32, [_vp]),
    "b200rl_env_episode_stats": (_i32, [_vp, _vp, _i32]),
    "b200rl_env_episode_log": (_i32, [_vp, C.c_int32]),
    "b200rl_env_episode_log_flush": (_i32, [_vp, _vp, _i64]),
    "b200rl_env_episode_log_read": (_i32, [_vp, _vp, C.POINTER(_i64)]),
    "b200rl_gae_f32": (_i32, [_vp, _vp, _vp, _vp, _vp, _f32, _f32, _i64, _i64, _i32, _i32]),
    "b200rl_gae_f64": (_i32, [_vp, _vp, _vp, _vp, _vp, _f64, _f64, _i64, _i64, _i32, _i32]),
    "b200rl_discount_rewards_f32": (_i32, [_vp, _vp, _vp, _vp, _vp, _f32, _i64, _i64, _i32, _i32]),
    "b200rl_discount_rewards_f64": (_i32, [_vp, _vp, _vp, _vp, _vp, _f64, _i64, _i64, _i32, _i32]),
    "b200rl_discount_rewards_reduced_f32": (_i32, [_vp, _vp, _vp, _vp, _vp, _f32, _i64, _i64, _i32, _i32]),
    "b200rl_discount_rewards_reduced_f64": (_i32, [_vp, _vp, _vp, _vp, _vp, _f64, _i64, _i64, _i32, _i32]),
    "b200rl_traj_create": (_i32, [_vp, _i32, _i64, _i64, _i32, _f32, _vp, _i64, _pp]),
    "b200rl_traj_destroy": (_i32, [_vp]),
    "b200rl_traj_length": (_i32, [_vp, C.POINTER(_i64)]),
    "b200rl_traj_lane_lengths": (_i32, [_vp, _vp]),
    "b200rl_traj_n_sampleable": (_i32, [_vp, C.POINTER(_i64)]),
    "b200rl_traj_push_episode_start": (_i32, [_vp, _vp, _i32, _i32]),
    "b200rl_traj_field_bytes": (_i32, [_vp, _i32, C.POINTER(_sz)]),
    "b200rl_traj_get": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_traj_set": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_traj_push_state": (_i32, [_vp, _vp, _i32]),
    "b200rl_traj_push": (_i32, [_vp, _vp, _vp, _vp, _vp, _i32]),
    "b200rl_traj_push_env": (_i32, [_vp, _vp, _i32]),
    "b200rl_traj_sample": (_i32, [_vp, _f32]),
    "b200rl_traj_set_nstep": (_i32, [_vp, _i32, _f32]),
    "b200rl_traj_batch_get": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_traj_update_priority": (_i32, [_vp, _vp, _i32]),
    "b200rl_traj_total_priority": (_i32, [_vp, C.POINTER(_f32)]),
    "b200rl_net_nparams": (_i32, [_vp, C.POINTER(_i64)]),
    "b200rl_net_create": (_i32, [_vp, _vp, _vp, _pp]),
    "b200rl_net_destroy": (_i32, [_vp]),
    "b200rl_net_configure_optimizer": (_i32, [_vp, _f32, _f32, _f32, _f32, _f32]),
    "b200rl_net_set_critic_act": (_i32, [_vp, _i32]),
    "b200rl_net_get": (_i32, [_vp, _i32, _vp, _i64]),
    "b200rl_net_set": (_i32, [_vp, _i32, _vp, _i64]),
    "b200rl_net_ptr": (_i32, [_vp, _i32, _pp]),
    "b200rl_net_get_step": (_i32, [_vp, C.POINTER(_i64)]),
    "b200rl_net_set_step": (_i32, [_vp, _i64]),
    "b200rl_net_target_sync": (_i32, [_vp, _f32]),
    "b200rl_net_act": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200rl_net_values": (_i32, [_vp, _vp, _i64, _vp, _i32, _i32]),
    "b200rl_net_q_act": (_i32, [_vp, _vp, _i64, _vp, _f32, _vp]),
    "b200rl_net_q_explore": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp]),
    "b200rl_net_act_greedy": (_i32, [_vp, _vp, _i64, _vp, _i32]),
    "b200rl_evaluate": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200rl_evaluate_explore": (_i32, [_vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32]),
    "b200rl_eval_create": (_i32, [_vp, _vp, _i32, _vp]),
    "b200rl_eval_destroy": (_i32, [_vp]),
    "b200rl_eval_run_episodes": (_i32, [_vp, _vp, _vp, _i64, _i64, C.POINTER(_i64), C.POINTER(_i64)]),
    "b200rl_net_ac_step": (_i32, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _f32, _f32, _i32, _vp]),
    "b200rl_onpolicy_create": (_i32, [_vp, _vp, _vp, _vp, _vp, _pp]),
    "b200rl_onpolicy_destroy": (_i32, [_vp]),
    "b200rl_onpolicy_plan": (_i32, [_vp, _vp]),
    "b200rl_onpolicy_act": (_i32, [_vp]),
    "b200rl_onpolicy_push": (_i32, [_vp]),
    "b200rl_onpolicy_collect": (_i32, [_vp, _i32]),
    "b200rl_onpolicy_fill": (_i32, [_vp, C.POINTER(_i32), C.POINTER(_i32)]),
    "b200rl_onpolicy_update": (_i32, [_vp, _vp, _vp]),
    "b200rl_onpolicy_iterate": (_i32, [_vp, _i32, _vp]),
    "b200rl_onpolicy_graph_active": (_i32, [_vp, C.POINTER(_i32)]),
    "b200rl_onpolicy_run_episodes": (_i32, [_vp, _i64, _i64, _vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "b200rl_onpolicy_get": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_onpolicy_set": (_i32, [_vp, _i32, _vp, _sz]),
    "b200rl_onpolicy_export_state": (_i32, [_vp, _vp]),
    "b200rl_onpolicy_import_state": (_i32, [_vp, _vp]),
    "b200rl_onpolicy_time_kernel": (_i32, [_vp, _i32, _i32, C.POINTER(_f32)]),
    "b200rl_dqn_update": (_i32, [_vp, _vp, _vp, _vp]),
    "b200rl_dqn_last_td": (_i32, [_vp, _vp, _vp, _i64]),
    "b200rl_replay_create": (_i32, [_vp, _vp, _vp, _vp, _vp, _pp]),
    "b200rl_replay_run": (_i32, [_vp, _vp, _vp, _vp, _i64, _vp]),
    "b200rl_replay_run_episodes": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _vp, C.POINTER(_i64), C.POINTER(_i64)]),
    "b200rl_replay_graph_active": (_i32, [_vp, C.POINTER(_i32)]),
    "b200rl_replay_destroy": (_i32, [_vp]),
    "b200rl_set_tensor_cores": (_i32, [_i32]),
    "b200rl_set_fused_step": (_i32, [_i32]),
    "b200rl_comm_unique_id": (_i32, [_vp]),
    "b200rl_comm_init": (_i32, [_vp, _i32, _i32, _vp]),
    "b200rl_comm_allreduce_f32": (_i32, [_vp, _vp, _i64]),
    "b200rl_comm_p2p_export": (_i32, [_vp, _vp, _pp]),
    "b200rl_comm_p2p_open": (_i32, [_vp, _vp, _pp]),
    "b200rl_comm_p2p_attach": (_i32, [_vp, _vp]),
    "b200rl_ctx_pci_bus_id": (_i32, [_vp, _vp, _i32]),
    "b200rl_comm_p2p_set_exclusive": (_i32, [_vp, _i32]),
    "b200rl_comm_rank_world": (_i32, [_vp, C.POINTER(_i32), C.POINTER(_i32)]),
}

_LIB = None


def load():
    """dlopen libb200rl.so and attach the signatures.  Loading needs no GPU; calling does."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(SO_PATH):
        raise RuntimeError(
            f"{SO_PATH} is missing: build it with `python reinforcementlearning.jl_b200/build.py` "
            "(there is no CPU fallback for the b200rl hot path)")
    lib = C.CDLL(SO_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    _LIB = lib
    return lib


def check(status):
    if status != OK:
        raise B200RLError(status, load().b200rl_last_error().decode(errors="replace"))


def ptr(a):
    """void* of a numpy array (None -> NULL) or pass an int device pointer through."""
    if a is None:
        return None
    if isinstance(a, (int, np.integer)):
        return C.c_void_p(int(a))
    if isinstance(a, C.c_void_p):
        return a
    return a.ctypes.data_as(C.c_void_p)


class Context:
    """b200rl_ctx: one device + one stream."""

    def __init__(self, device=0):
        self.lib = load()
        h = C.c_void_p()
        check(self.lib.b200rl_init(device, C.byref(h)))
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200rl_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sync(self):
        check(self.lib.b200rl_sync(self.h))

    def rank_world(self):
        """(rank, world) of the ctx's communicator; (0, 1) without one (b200rl_comm_rank_world)."""
        r, w = C.c_int32(), C.c_int32()
        check(self.lib.b200rl_comm_rank_world(self.h, C.byref(r), C.byref(w)))
        return r.value, w.value

    def stream(self):
        s = C.c_void_p()
        check(self.lib.b200rl_stream(self.h, C.byref(s)))
        return s.value or 0

    def timer_start(self):
        check(self.lib.b200rl_timer_start(self.h))

    def timer_stop_ms(self):
        ms = C.c_float()
        check(self.lib.b200rl_timer_stop_ms(self.h, C.byref(ms)))
        return ms.value

    def timer_record(self, slot):
        check(self.lib.b200rl_timer_record(self.h, slot))

    def timer_elapsed_ms(self, slot_from, slot_to):
        ms = C.c_float()
        check(self.lib.b200rl_timer_elapsed_ms(self.h, slot_from, slot_to, C.byref(ms)))
        return ms.value

    def phase_slots(self, base_slot):
        check(self.lib.b200rl_debug_phase_slots(self.h, base_slot))

    def launch_count(self):
        n = C.c_uint64()
        check(self.lib.b200rl_launch_count(self.h, C.byref(n)))
        return n.value

    def flush_l2(self):
        check(self.lib.b200rl_flush_l2(self.h))

    def malloc(self, nbytes):
        p = C.c_void_p()
        check(self.lib.b200rl_malloc(self.h, nbytes, C.byref(p)))
        return p.value

    def free(self, dptr):
        check(self.lib.b200rl_free(self.h, C.c_void_p(dptr)))

    def h2d(self, dptr, arr, async_=False):
        if not (arr.flags.c_contiguous or arr.flags.f_contiguous):
            arr = np.ascontiguousarray(arr)   # F-ordered (Julia-shaped) arrays are copied as they lie in memory
        check(self.lib.b200rl_memcpy_h2d(self.h, C.c_void_p(dptr), ptr(arr), arr.nbytes, int(async_)))

    def d2h(self, arr, dptr, async_=False):
        assert arr.flags.c_contiguous or arr.flags.f_contiguous
        check(self.lib.b200rl_memcpy_d2h(self.h, ptr(arr), C.c_void_p(dptr), arr.nbytes, int(async_)))
        return arr

    def host_alloc(self, shape, dtype):
        """Pinned host numpy array (freed with host_free)."""
        dtype = np.dtype(dtype)
        n = int(np.prod(shape)) * dtype.itemsize
        p = C.c_void_p()
        check(self.lib.b200rl_host_alloc(self.h, n, C.byref(p)))
        buf = (C.c_char * max(n, 1)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
        return arr, p.value

    def host_free(self, address):
        check(self.lib.b200rl_host_free(self.h, C.c_void_p(address)))
