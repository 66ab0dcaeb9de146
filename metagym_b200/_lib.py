"""ctypes binding of libmgb200.so (include/mgb200.h).  There is no CPU fallback: if the library is missing or the
CUDA runtime cannot find a device, the entry points raise instead of silently computing somewhere else."""
import ctypes
import os

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, "libmgb200.so")

c_i32, c_i64, c_u64, c_f32, c_f64 = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64, ctypes.c_float, ctypes.c_double
vp = ctypes.c_void_p


class MgbError(RuntimeError):
    pass


class QuadCfg(ctypes.Structure):
    """mgb_quad_cfg (include/mgb200.h)."""
    _fields_ = [
        ("precision", c_f64), ("quality", c_f64), ("inv_inertia", c_f32 * 9), ("drag_m", c_f32 * 3),
        ("drag_f", c_f32 * 3), ("gravity_center", c_f32 * 3), ("ct", c_f64 * 3), ("mm", c_f64), ("jm", c_f64),
        ("phi", c_f64), ("ra", c_f64), ("fail_velocity", c_f64), ("fail_range", c_f64), ("fail_w", c_f64),
        ("propeller", c_f32 * 12), ("propeller_norm", c_f32 * 4), ("min_voltage", c_f64), ("max_voltage", c_f64),
        ("init_velocity", c_f32 * 3), ("init_velocity_noise", c_f64), ("init_angular_velocity", c_f32 * 3),
        ("init_angular_velocity_noise", c_f64), ("dt", c_f64), ("nt", c_i32), ("task", c_i32),
        ("healthy_reward", c_f64), ("z_offset", c_f64), ("integrator", c_i32), ("rk4_steps", c_i32),
    ]


class MazeTaskScalars(ctypes.Structure):
    """mgb_maze_task_scalars (include/mgb200.h)."""
    _fields_ = [("start", c_i32 * 2), ("goal", c_i32 * 2), ("cell_size", c_f64), ("wall_height", c_f64),
                ("agent_height", c_f64), ("initial_life", c_f64), ("max_life", c_f64), ("step_reward", c_f64),
                ("goal_reward", c_f64)]


class MazeSamplerCfg(ctypes.Structure):
    """mgb_maze_sampler_cfg (include/mgb200.h)."""
    _fields_ = [("allow_loops", c_i32), ("n_texts", c_i32), ("food_interval", c_i32), ("pad", c_i32),
                ("cell_size", c_f64), ("wall_height", c_f64), ("agent_height", c_f64), ("step_reward", c_f64),
                ("goal_reward", c_f64), ("food_reward", c_f64), ("initial_life", c_f64), ("max_life", c_f64),
                ("food_density", c_f64), ("crowd_ratio", c_f64)]


class MazeCfg(ctypes.Structure):
    """mgb_maze_cfg (include/mgb200.h)."""
    _fields_ = [("kind", c_i32), ("task_type", c_i32), ("n_cells", c_i32), ("max_steps", c_i32),
                ("view_grid", c_i32), ("res_h", c_i32), ("res_v", c_i32), ("obs_dtype", c_i32),
                ("max_vision", c_f64), ("fov", c_f64), ("l_focal", c_f64), ("text_size", c_f64)]


class Policy(ctypes.Structure):
    """mgb_policy (include/mgb200.h)."""
    _fields_ = [("params_dev", vp), ("n_hidden", c_i32), ("width", c_i32 * 3), ("activation", c_i32), ("mode", c_i32)]


class RnnPolicy(ctypes.Structure):
    """mgb_rnn_policy (include/mgb200.h)."""
    _fields_ = [("params_dev", vp), ("hidden", c_i32), ("feedback", c_i32), ("reset", c_i32), ("head_hidden", c_i32),
                ("head_width", c_i32), ("activation", c_i32), ("mode", c_i32), ("cell", c_i32)]


class Critic(ctypes.Structure):       # mgb_critic
    _fields_ = [("value_dev", vp), ("value_last_dev", vp), ("final_value_dev", vp), ("adv_dev", vp), ("ret_dev", vp),
                ("gamma", ctypes.c_float), ("lam", ctypes.c_float)]


class RnnSeq(ctypes.Structure):
    """mgb_rnn_seq (include/mgb200.h)."""
    _fields_ = [("cell", c_i32), ("hidden", c_i32), ("in_", c_i32), ("T", c_i32), ("n", c_i64), ("params_dev", vp),
                ("x_dev", vp), ("wipe_dev", vp), ("state0_dev", vp), ("h_dev", vp), ("gates_dev", vp), ("dh_dev", vp),
                ("dgi_dev", vp), ("dghn_dev", vp), ("dstate0_dev", vp)]


ACT_TANH, ACT_RELU = 0, 1            # MGB_ACT_*
POLICY_SAMPLE, POLICY_MEAN = 0, 1    # MGB_POLICY_*
RNN_RESET_EPISODE, RNN_RESET_TASK = 0, 1     # MGB_RNN_RESET_*
RNN_CELL_GRU, RNN_CELL_LSTM = 0, 1           # MGB_RNN_CELL_*
POLICY_MEMBER_WARP = 32                      # MGB_POLICY_MEMBER_WARP
QUAD_POLICY_CTA_ENVS = 64                    # MGB_QUAD_POLICY_CTA_ENVS
MAZE2D_POLICY_CTA_ENVS = 128                 # MGB_MAZE2D_POLICY_CTA_ENVS
QUAD_RNN_CTA_ENVS = 128                      # MGB_QUAD_RNN_CTA_ENVS
RNN_SEQ_CTA_ENVS = 128                       # MGB_RNN_SEQ_CTA_ENVS


# name -> (restype, argtypes); every function include/mgb200.h declares (tests/test_abi.py checks the two agree)
SIGNATURES = {
    "mgb_quad_create": (ctypes.c_int, [ctypes.POINTER(vp), c_i64, ctypes.POINTER(QuadCfg), ctypes.c_int, c_i64]),
    "mgb_quad_destroy": (None, [vp]),
    "mgb_quad_obs_dim": (ctypes.c_int, [vp]),
    "mgb_quad_num_envs": (c_i64, [vp]),
    "mgb_quad_set_options": (ctypes.c_int, [vp, ctypes.c_int, c_u64]),
    "mgb_quad_set_map": (ctypes.c_int, [vp, vp, c_i32, c_i32]),
    "mgb_quad_set_targets": (ctypes.c_int, [vp, vp, c_i32, vp]),
    "mgb_quad_make_targets": (ctypes.c_int, [vp, vp, c_i32, vp, vp]),
    "mgb_quad_reset": (ctypes.c_int, [vp, vp, vp, vp, vp]),
    "mgb_quad_step": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_quad_rollout": (ctypes.c_int, [vp, c_i32, vp, c_u64, vp, vp, vp, vp, vp]),
    "mgb_quad_step_host": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_quad_step_ex": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_quad_step_host_ex": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_quad_rollout_ex": (ctypes.c_int, [vp, c_i32, vp, c_u64, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_quad_rollout_policy": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), c_u64, vp, vp, vp, vp, vp, vp, vp, vp,
                                               vp]),
    "mgb_quad_rollout_population": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), c_i32, c_i64, c_u64, vp, vp, vp,
                                                   vp, vp, vp, vp, vp, vp]),
    "mgb_quad_rollout_critic": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), c_i32, c_i64, c_u64, vp, vp, vp, vp,
                                               vp, vp, vp, vp, ctypes.POINTER(Critic), vp]),
    "mgb_quad_rollout_rnn": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(RnnPolicy), c_u64, vp, vp, vp, vp, vp, vp, vp,
                                            vp, vp, vp, vp, vp]),
    "mgb_quad_rollout_rnn_population": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(RnnPolicy), c_i32, c_i64, c_u64, vp,
                                                       vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_quad_rollout_rnn_critic": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(RnnPolicy), c_i32, c_i64, c_u64, vp, vp,
                                                   vp, vp, vp, vp, vp, vp, vp, vp, vp, ctypes.POINTER(Critic), vp]),
    "mgb_quad_state": (ctypes.c_int, [vp, vp, vp, ctypes.c_int, vp]),
    "mgb_quad_launch_count": (c_i64, [vp]),
    "mgb_quad_step_kernel": (ctypes.c_char_p, [vp]),
    "mgb_maze_create": (ctypes.c_int, [ctypes.POINTER(vp), c_i64, ctypes.POINTER(MazeCfg), ctypes.c_int, c_i64]),
    "mgb_maze_destroy": (None, [vp]),
    "mgb_maze_obs_bytes_per_env": (c_i64, [vp]),
    "mgb_maze_set_textures": (ctypes.c_int, [vp, vp, c_i32, vp, c_i32]),
    "mgb_maze_set_task": (ctypes.c_int, [vp, c_i32, vp, vp, vp, vp, ctypes.POINTER(MazeTaskScalars), vp]),
    "mgb_maze_resample_tasks": (ctypes.c_int, [vp, vp, ctypes.POINTER(MazeSamplerCfg), c_u64, vp]),
    "mgb_maze_get_tasks": (ctypes.c_int, [vp, c_i32, vp, vp, vp, vp, vp, ctypes.POINTER(MazeTaskScalars)]),
    "mgb_maze_set_cache": (ctypes.c_int, [vp, ctypes.c_int]),
    "mgb_maze_cache_info": (ctypes.c_int, [vp, vp]),
    "mgb_maze_update_tasks": (ctypes.c_int, [vp, c_i32, vp, vp, vp, vp, vp, ctypes.POINTER(MazeTaskScalars), vp]),
    "mgb_maze_reset": (ctypes.c_int, [vp, vp, vp, vp]),
    "mgb_maze_step": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_maze_set_options": (ctypes.c_int, [vp, ctypes.c_int]),
    "mgb_maze_set_episodes_per_task": (ctypes.c_int, [vp, c_i32]),
    "mgb_maze_task_episodes": (ctypes.c_int, [vp, vp, vp]),
    "mgb_peer_alloc": (ctypes.c_int, [ctypes.c_int, c_u64, ctypes.POINTER(ctypes.c_void_p)]),
    "mgb_peer_free": (ctypes.c_int, [ctypes.c_int, vp]),
    "mgb_peer_export": (ctypes.c_int, [ctypes.c_int, vp, vp]),
    "mgb_peer_open": (ctypes.c_int, [ctypes.c_int, vp, ctypes.POINTER(ctypes.c_void_p)]),
    "mgb_peer_close": (ctypes.c_int, [ctypes.c_int, vp]),
    "mgb_quad_set_mirrors": (ctypes.c_int, [vp, ctypes.c_int, vp]),
    "mgb_maze_set_mirrors": (ctypes.c_int, [vp, ctypes.c_int, vp]),
    "mgb_quad_set_mirror_window": (ctypes.c_int, [vp, vp, c_u64]),
    "mgb_maze_set_mirror_window": (ctypes.c_int, [vp, vp, c_u64]),
    "mgb_quad_set_multicast": (ctypes.c_int, [vp, ctypes.c_int64]),
    "mgb_maze_set_multicast": (ctypes.c_int, [vp, ctypes.c_int64]),
    "mgb_maze_rollout": (ctypes.c_int, [vp, c_i32, vp, c_u64, vp, vp, vp, vp, vp, vp, ctypes.POINTER(MazeSamplerCfg),
                                        c_u64, vp]),
    "mgb_maze_set_expert": (ctypes.c_int, [vp, ctypes.c_int]),
    "mgb_maze_rollout_expert": (ctypes.c_int, [vp, c_i32, vp, ctypes.c_float, c_i32, c_u64, vp, vp, vp, vp, vp, vp, vp,
                                               vp]),
    "mgb_maze_step_expert": (ctypes.c_int, [vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_maze_expert": (ctypes.c_int, [vp, vp, vp, vp]),
    "mgb_maze_expert_table": (ctypes.c_int, [vp, c_i32, c_i32, vp, vp, vp]),
    "mgb_maze_rollout_policy": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), c_u64, ctypes.POINTER(MazeSamplerCfg),
                                               c_u64, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_maze_rollout_rnn": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(RnnPolicy), c_u64, ctypes.POINTER(MazeSamplerCfg),
                                            c_u64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]),
    "mgb_maze_rollout_population": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), c_i32, c_i64, c_u64,
                                                   ctypes.POINTER(MazeSamplerCfg), c_u64, vp, vp, vp, vp, vp, vp, vp,
                                                   vp, vp]),
    "mgb_maze_rollout_rnn_population": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(RnnPolicy), c_i32, c_i64, c_u64,
                                                       ctypes.POINTER(MazeSamplerCfg), c_u64, vp, vp, vp, vp, vp, vp,
                                                       vp, vp, vp, vp, vp, vp]),
    "mgb_maze_rollout_critic": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), c_i32, c_i64, c_u64,
                                               ctypes.POINTER(MazeSamplerCfg), c_u64, vp, vp, vp, vp, vp, vp, vp, vp,
                                               ctypes.POINTER(Critic), vp]),
    "mgb_maze_rollout_rnn_critic": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(RnnPolicy), c_i32, c_i64, c_u64,
                                                   ctypes.POINTER(MazeSamplerCfg), c_u64, vp, vp, vp, vp, vp, vp, vp,
                                                   vp, vp, vp, vp, ctypes.POINTER(Critic), vp]),
    "mgb_quad_evaluate": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), ctypes.POINTER(RnnPolicy), c_i32, c_i32,
                                         c_i64, c_u64, vp, vp, vp, vp, vp]),
    "mgb_maze_evaluate": (ctypes.c_int, [vp, c_i32, ctypes.POINTER(Policy), ctypes.POINTER(RnnPolicy), c_i32, c_i32,
                                         c_i64, c_u64, ctypes.POINTER(MazeSamplerCfg), c_u64, vp, vp, vp, vp, vp]),
    "mgb_rnn_seq_forward": (ctypes.c_int, [ctypes.POINTER(RnnSeq), vp]),
    "mgb_rnn_seq_backward": (ctypes.c_int, [ctypes.POINTER(RnnSeq), vp]),
    "mgb_maze_pose": (ctypes.c_int, [vp, vp, vp, vp]),
    "mgb_maze_state": (ctypes.c_int, [vp, vp, vp, vp]),
    "mgb_maze_launch_count": (c_i64, [vp]),
    "mgb_maze_god_view": (ctypes.c_int, [vp, c_i32, vp, c_i32, c_i32, vp, vp]),
    "mgb_maze_set_path": (ctypes.c_int, [vp, ctypes.c_int]),
    "mgb_maze_path": (ctypes.c_int, [vp, c_i32, vp, vp, vp, vp]),
    "mgb_quad_record_bytes": (c_i64, [vp]),
    "mgb_quad_snapshot": (ctypes.c_int, [vp, vp, vp]),
    "mgb_quad_restore": (ctypes.c_int, [vp, vp, c_i64, vp, vp]),
    "mgb_quad_counters": (ctypes.c_int, [vp, ctypes.POINTER(c_u64), ctypes.c_int]),
    "mgb_quad_fingerprint": (ctypes.c_int, [vp, ctypes.POINTER(c_u64)]),
    "mgb_maze_record_bytes": (c_i64, [vp]),
    "mgb_maze_snapshot": (ctypes.c_int, [vp, vp, vp]),
    "mgb_maze_restore": (ctypes.c_int, [vp, vp, c_i64, vp, vp]),
    "mgb_maze_counters": (ctypes.c_int, [vp, ctypes.POINTER(c_u64), ctypes.c_int]),
    "mgb_maze_fingerprint": (ctypes.c_int, [vp, ctypes.POINTER(c_u64)]),
    "mgb_last_error": (ctypes.c_char_p, []),
    "mgb_version": (ctypes.c_char_p, []),
    "mgb_device_count": (ctypes.c_int, []),
}

_lib = None


def load():
    """dlopen libmgb200.so and bind every symbol.  Raises MgbError when the library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MgbError("%s not found: build it with `python -m metagym_b200._build` (nvcc, sm_90a). "
                       "metagym_b200 has no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise MgbError("libmgb200: %s (code %d)" % (load().mgb_last_error().decode(), rc))


def current_stream(torch, device):
    """Raw cudaStream_t of torch's current stream on `device` (torch.device with an index)."""
    get = getattr(torch._C, "_cuda_getCurrentRawStream", None)
    if get is not None:
        return get(device.index)
    return torch.cuda.current_stream(device).cuda_stream


def ptr(t):
    """Device/host address of a torch tensor or numpy array (None -> NULL)."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    return t.ctypes.data
