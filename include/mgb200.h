/*
 * mgb200.h -- C ABI of libmgb200.so, the H100 (sm_90a) batched environment engine for the two MetaGym dynamics
 * hot paths (quadrotor 6-DoF integrator + task logic; MetaMaze grid step + raycast render).
 *
 * The reference (PaddlePaddle/MetaGym) is pure Python and has no FFI of its own; the boundary it exposes is the
 * gym.Env protocol.  Each entry point below therefore names the reference METHOD it replaces (file:line relative to
 * the reference tree), for a batch of n independent env instances.  The Python classes in metagym_b200/ bind these
 * symbols with ctypes and re-expose the reference's method names (INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error; mgb_last_error() returns a thread-local message.
 *   - *_dev pointers are device pointers owned by the caller (e.g. torch tensor.data_ptr()); *_host are host pointers.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).  Nothing synchronises the host except
 *     the *_host entry points, mgb_*_create/destroy and the functions documented as synchronous.
 *   - a handle is bound to one device and is not thread-safe; distinct handles are independent.
 *   - there is NO CPU fallback: without a usable CUDA device every create call fails with MGB_ERR_CUDA.
 */
#ifndef MGB200_H
#define MGB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MGB_OK 0
#define MGB_ERR_ARG (-1)
#define MGB_ERR_CUDA (-2)
#define MGB_ERR_STATE (-3)

/* ------------------------------------------------------------------------------------------------------------ */
/* Quadrotor                                                                                                      */
/* ------------------------------------------------------------------------------------------------------------ */

#define MGB_TASK_NO_COLLISION 0     /* env.py:216-218 */
#define MGB_TASK_HOVERING_CONTROL 1 /* env.py:222-243 */
#define MGB_TASK_VELOCITY_CONTROL 2 /* env.py:219-221 */

#define MGB_INTEGRATOR_REFERENCE 0
#define MGB_INTEGRATOR_RK4 1

#define MGB_FAIL_NONE 0
#define MGB_FAIL_RANGE 1    /* quadrotorsim.py:213-214 */
#define MGB_FAIL_VELOCITY 2 /* quadrotorsim.py:216-217 */
#define MGB_FAIL_ANGULAR 3  /* quadrotorsim.py:219-221 */

/* Numbers of QuadrotorSim._parse_cfg (quadrotorsim.py:50-109) + the Quadrotor ctor kwargs (env.py:46-69).
 * Doubles carry the python floats of the config exactly; the library rounds derived constants to float32 the way
 * numpy >= 2 does ("weak" python scalars take the float32 type of the array they meet). */
typedef struct mgb_quad_cfg {
    double precision;          /* config.json "precision": substep h                         */
    double quality;            /* config.json "quality": mass                                */
    float inv_inertia[9];      /* np.linalg.inv(float32 inertia), row-major (quadrotorsim.py:64) */
    float drag_m[3];           /* diag of _drag_coeff_momentum                               */
    float drag_f[3];           /* diag of _drag_coeff_force                                  */
    float gravity_center[3];
    double ct[3];              /* thrust CT0..2                                              */
    double mm, jm, phi, ra;    /* thrust Mm, Jm, phi, RA                                     */
    double fail_velocity, fail_range, fail_w;
    float propeller[12];       /* 4 x (x,y,z)                                                */
    float propeller_norm[4];   /* np.linalg.norm(float32 coord) (quadrotorsim.py:146)        */
    double min_voltage, max_voltage;
    float init_velocity[3];    /* config.json "init_velocity" x,y,z                          */
    double init_velocity_noise;
    float init_angular_velocity[3];
    double init_angular_velocity_noise;
    /* Quadrotor(...) kwargs, env.py:46-53 */
    double dt;
    int32_t nt;
    int32_t task;              /* MGB_TASK_*                                                 */
    double healthy_reward;
    double z_offset;           /* env.py:112 (5.0 for the flat map; 0 for velocity_control)  */
    /* Integrator.  MGB_INTEGRATOR_REFERENCE: int(dt/precision) semi-implicit Euler substeps, the reference's only
     * integrator (quadrotorsim.py:122-208) and the parity-checked default.  MGB_INTEGRATOR_RK4: classical RK4 on the
     * same continuous-time model, rk4_steps steps of dt/rk4_steps per env step -- BASELINE.json's "RK4 dt=0.005";
     * the reference has no counterpart, so it is validated by convergence only (DESIGN.md, row Q9). */
    int32_t integrator;
    int32_t rk4_steps;
} mgb_quad_cfg;

typedef struct mgb_quad mgb_quad;

/* Quadrotor.__init__ (env.py:46-114) for n_envs instances on `device`.  State starts at _zero_state
 * (quadrotorsim.py:20-28), ct = 0.  `env_index_base` is the global index of local env 0: per-env random streams are
 * keyed by the global index so that results do not depend on how envs are sharded over GPUs. */
int mgb_quad_create(mgb_quad **out, int64_t n_envs, const mgb_quad_cfg *cfg, int device, int64_t env_index_base);
void mgb_quad_destroy(mgb_quad *h);

/* Observation width: 16, or 19 for velocity_control (env.py:86-92). */
int mgb_quad_obs_dim(const mgb_quad *h);
int64_t mgb_quad_num_envs(const mgb_quad *h);

/* auto_reset != 0: an env whose step returns done is re-initialised in the same launch with counter-based noise
 * (Philox keyed by seed, global env index, episode count); obs then holds the first observation of the new episode
 * and final_obs (if given to mgb_quad_step) the terminal one.  auto_reset == 0: the reference behaviour -- state is
 * left as is and the caller resets (env.py:116).  Synchronous w.r.t. nothing; takes effect at the next launch. */
int mgb_quad_set_options(mgb_quad *h, int auto_reset, uint64_t seed);

/* Quadrotor.load_map + the map part of __init__ (env.py:97-114, 293-305): map_host [rows][cols] int32 with exactly one
 * -1 (the start cell, which becomes 0); x_offset / y_offset are its column / row.  Only the TRUTHINESS of the cells in
 * the window swept by a step matters to the reference's _check_collision (env.py:248-260: `z < np.any(taken_pos)`),
 * including python's negative-index slice semantics; both are reproduced.  NULL map = the flat default (env.py:295-298).
 * no_collision / hovering_control only.  Synchronous. */
int mgb_quad_set_map(mgb_quad *h, const int32_t *map_host, int32_t rows, int32_t cols);

/* Velocity targets of define_velocity_control_task (quadrotorsim.py:306-319): tbl [n_tasks][nt][3] float32 and the
 * task row of every local env, env2task [n_envs] int32.  Both are COPIED into the handle (synchronous).  The handle
 * stores the table time-major with one 16-byte row per (t, task), [nt][n_tasks] float4 (x, y, z, 0), so that a step
 * reads a row with one load and a warp of envs at the same t reads contiguous rows: 16 * nt * n_tasks bytes of device
 * memory, a third more than tbl (1 MB for 64 tasks at nt = 1000, 1.05 GB for 65 536 tasks). */
int mgb_quad_set_targets(mgb_quad *h, const float *tbl_dev, int32_t n_tasks, const int32_t *env2task_dev);

/* Runs define_velocity_control_task (quadrotorsim.py:306-319) on the device for n_tasks seeds: act_host [n_tasks][nt][4] float32 are the
 * np.random.uniform draws (host-replayed for RNG parity); tbl_dev [n_tasks][nt][3] receives global_velocity after
 * every step from the zero state.  Independent of the handle's env state. */
int mgb_quad_make_targets(mgb_quad *h, const float *act_dev, int32_t n_tasks, float *tbl_dev, void *stream);

/* Quadrotor.reset (env.py:116-125 -> quadrotorsim.py:239-258).  mask_dev [n] uint8 (NULL = all envs).
 * noise_dev [n][12] float64 = the twelve np.random.random() draws of one reset in reference order (sign_v[3],
 * mag_v[3], sign_w[3], mag_w[3]); NULL = counter-based draws.  ct is NOT touched (reference quirk, env.py:65,150).
 * obs_dev [n][obs_dim] (NULL = skip) receives the observation of every env (masked-out envs: current state). */
int mgb_quad_reset(mgb_quad *h, const uint8_t *mask_dev, const double *noise_dev, float *obs_dev, void *stream);

/* Quadrotor.step (env.py:127-165): int(dt/precision) substeps of QuadrotorSim._run_internal (quadrotorsim.py:122-221),
 * get_sensor/get_state (:260-293), reward / collision / done (env.py:211-260).
 *   act_dev  [n][4] float32           obs_dev [n][obs_dim] float32      rew_dev [n] float32     done_dev [n] uint8
 *   fail_dev [n] int32 or NULL  (MGB_FAIL_*: the reference raises, the batch reports done + code)
 *   final_obs_dev [n][obs_dim] or NULL (terminal observation of envs that finished, when auto_reset is on) */
int mgb_quad_step(mgb_quad *h, const float *act_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                  int32_t *fail_dev, float *final_obs_dev, void *stream);
/* mgb_quad_step with one more optional output (NULL: not produced, and the call is exactly mgb_quad_step):
 *   truncated_dev [n] uint8, written for every env: 1 iff done and the episode ended through the time limit alone,
 *     `ct == nt` (env.py:159-161).  A collision in the same step is terminal: its branch (env.py:144-150) clears ct
 *     before the time-limit check.  A failure (MGB_FAIL_*, where the reference raises) is terminal.  So
 *     terminated = done && !truncated; for velocity_control, truncated = done && fail == MGB_FAIL_NONE.
 * obs, rew, done, fail, final_obs and the env state are bit for bit what mgb_quad_step gives. */
int mgb_quad_step_ex(mgb_quad *h, const float *act_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                     int32_t *fail_dev, float *final_obs_dev, uint8_t *truncated_dev, void *stream);

/* T consecutive Quadrotor.step calls (env.py:127-165; the rollout loop of quadrotor/tests/test_env.py:22-28) in ONE launch
 * with the state held in registers (auto-reset semantics as configured).
 *   act_dev [T][n][4] or NULL: NULL draws U(min_voltage, max_voltage) actions from the counter-based generator
 *   (stream id `act_seed`), written to act_out_dev [T][n][4] if not NULL.
 *   obs_dev [T][n][obs_dim], rew_dev [T][n], done_dev [T][n]; any of them may be NULL to skip that output. */
int mgb_quad_rollout(mgb_quad *h, int32_t T, const float *act_dev, uint64_t act_seed, float *act_out_dev,
                     float *obs_dev, float *rew_dev, uint8_t *done_dev, void *stream);
/* mgb_quad_rollout with two optional outputs (both NULL: exactly mgb_quad_rollout):
 *   final_obs_dev [T][n][obs_dim] float32: row (t, e) is written only when done[t][e] = 1, with the observation an
 *     auto_reset-off handle would have returned at step t (the terminal one, env.py:163-165).  Rows with done = 0 are
 *     not written.  Needs auto_reset on (MGB_ERR_ARG otherwise).
 *   truncated_dev [T][n] uint8, written for every (t, e): as mgb_quad_step_ex's truncated_dev (env.py:144-161).
 * obs, rew, done, the drawn actions and the env state are bit for bit what mgb_quad_rollout gives.  Either output while
 * output mirrors or multicast are set is MGB_ERR_ARG. */
int mgb_quad_rollout_ex(mgb_quad *h, int32_t T, const float *act_dev, uint64_t act_seed, float *act_out_dev,
                        float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                        void *stream);

/* ---- policy-driven rollouts (DESIGN.md "Policy-driven rollouts") ------------------------------------------------
 * A multi-layer perceptron evaluated inside the rollout launch: the action of step t is drawn from the policy's output
 * on the observation the env holds before step t.
 *   params_dev: float32 on the handle's device, read at every launch (so a captured graph sees an in-place update).
 *     Layers in torch.nn.Linear order, first hidden layer to output layer: W [out][in] row-major, then b [out].  The
 *     input width is the obs dim, the output width 4.  The quadrotor buffer then ends with log_std [4].
 *   n_hidden 0..3, width[k] 1..64 for k < n_hidden, activation MGB_ACT_* (every hidden layer), mode MGB_POLICY_*.
 *   The maze buffer has no log_std: its four outputs are the logits of the actions 0..3.
 * Numerical contract: float32 throughout, each output a fused multiply-add chain from the bias over the inputs in index
 * order, accurate tanhf / expf / logf (no approximate instructions, no tensor cores).  Draws: Philox4x32-10, counter
 * (genv lo, genv hi, t_base + t, MGB_STREAM_POLICY = 0x400), key = seed. */
#define MGB_ACT_TANH 0
#define MGB_ACT_RELU 1
#define MGB_POLICY_SAMPLE 0   /* stochastic: Gaussian (quadrotor) / categorical (maze 2-D) */
#define MGB_POLICY_MEAN 1     /* deterministic: the mean (quadrotor) / argmax of the logits (maze 2-D) */
#define MGB_POLICY_MAX_HIDDEN 3
#define MGB_POLICY_MAX_WIDTH 64
/* Populations (the *_population entry points): envs per member are a multiple of MGB_POLICY_MEMBER_WARP and either
 * divide the policy kernel's CTA env count or are a multiple of it. */
#define MGB_POLICY_MEMBER_WARP 32
#define MGB_QUAD_POLICY_CTA_ENVS 64      /* quadrotor: 32 or a multiple of 64 envs per member */
#define MGB_MAZE2D_POLICY_CTA_ENVS 128   /* MetaMaze2D: 32, 64 or a multiple of 128 envs per member */
#define MGB_QUAD_RNN_CTA_ENVS 128        /* quadrotor, recurrent policies: 32, 64 or a multiple of 128 envs per member */

typedef struct mgb_policy {
    const float *params_dev;  /* packed float32 on the handle's device, read at every launch */
    int32_t n_hidden;         /* 0..3 hidden layers */
    int32_t width[3];         /* 1..64 each (entries past n_hidden are ignored) */
    int32_t activation;       /* MGB_ACT_*, the same for every hidden layer */
    int32_t mode;             /* MGB_POLICY_* */
} mgb_policy;

/* mgb_quad_rollout_ex with actions from a Gaussian MLP policy instead of a fixed tensor.
 *   Sampling: for the four Philox words (x, y, z, w), Box-Muller per pair: u1 = ((x >> 8) + 1) 2^-24 in (0, 1],
 *   u2 = (y >> 8) 2^-24, z0 = sqrt(-2 log u1) cos(2 pi u2), z1 = sqrt(-2 log u1) sin(2 pi u2); likewise z2, z3 from
 *   (z, w).  a_k = mean_k + exp(log_std_k) z_k, with no squashing or clipping (the step clamps voltages).
 *   logp = sum_k (-z_k^2 / 2 - log_std_k) - 2 log(2 pi).  MGB_POLICY_MEAN: a = mean, and logp_out must be NULL.
 *   act_out_dev [T][n][4] float32: the actions taken.  logp_out_dev [T][n] float32.  obs0_out_dev [n][obs_dim]: the
 *   observation the policy acted on at t = 0, computed from the handle's state; at t > 0 it acted on obs[t-1].
 *   obs, rew, done, final_obs, truncated: as mgb_quad_rollout_ex.  Every output may be NULL.
 * The env side is bit for bit mgb_quad_rollout_ex fed act_out.  The step counter advances by T; nothing is allocated,
 * and the call can be captured in a CUDA graph.  Refused (MGB_ERR_ARG, handle untouched): T <= 0, a NULL policy or
 * params_dev, n_hidden / width / activation / mode out of range, logp_out in mean mode, output mirrors or multicast
 * set, final_obs without auto_reset, and weights plus activations beyond the device's opt-in shared memory. */
int mgb_quad_rollout_policy(mgb_quad *h, int32_t T, const mgb_policy *pol, uint64_t seed, float *act_out_dev,
                            float *logp_out_dev, float *obs0_out_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                            float *final_obs_dev, uint8_t *truncated_dev, void *stream);

/* mgb_quad_rollout_policy with a population of `members` policies of pol's shape (DESIGN.md "Populations"): member m's
 * packed buffer starts at pol->params_dev + m member_stride floats, and with E = n / members it drives the envs
 * [m E, (m + 1) E) of the handle.  Every other input, output, draw (keyed by the global env index) and refusal is
 * mgb_quad_rollout_policy's, and members = 1 is that call exactly (the stride is then not read).  Also refused
 * (MGB_ERR_ARG, handle untouched): members < 1, n not a multiple of members, E neither 32 nor a multiple of
 * MGB_QUAD_POLICY_CTA_ENVS, member_stride below the packed length (with log_std), and the staged members of one CTA
 * with the activations beyond the device's opt-in shared memory. */
int mgb_quad_rollout_population(mgb_quad *h, int32_t T, const mgb_policy *pol, int32_t members, int64_t member_stride,
                                uint64_t seed, float *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                                float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                                uint8_t *truncated_dev, void *stream);

/* Quadrotor.step as the reference's numpy users call it (env.py:127-165: ndarray in, ndarray out).
 * Same as mgb_quad_step with HOST buffers: stages through pinned memory (or, for pinned caller buffers, lets the kernel
 * read/write host memory directly), copies inside the call, returns when the outputs are on the host (synchronous).
 * All work is enqueued on `stream` (the caller's current stream), so the step is ordered after a preceding
 * mgb_quad_reset / mgb_quad_rollout / mgb_quad_state on that stream.  fail_host [n] int32 and final_obs_host
 * [n][obs_dim] may be NULL; they report what mgb_quad_step's fail_dev / final_obs_dev report (quadrotorsim.py:212-221).
 * This is the call a numpy user of the reference API makes. */
int mgb_quad_step_host(mgb_quad *h, const float *act_host, float *obs_host, float *rew_host, uint8_t *done_host,
                       int32_t *fail_host, float *final_obs_host, void *stream);
/* mgb_quad_step_host with truncated_host [n] uint8 (NULL: not produced): what mgb_quad_step_ex's truncated_dev reports
 * (env.py:144-161), through the same zero-copy, copy and hybrid paths (a pageable truncated_host takes the copy path). */
int mgb_quad_step_host_ex(mgb_quad *h, const float *act_host, float *obs_host, float *rew_host, uint8_t *done_host,
                          int32_t *fail_host, float *final_obs_host, uint8_t *truncated_host, void *stream);

/* Checkpoint / inspection (quadrotorsim.py:30-48 _save_state/_restore_state): state_dev [n][22] float32 row-major
 * = p3 v3 w3 prop4 R9, ct_dev [n] int32.  load = 0 copies handle -> buffers, 1 buffers -> handle. */
int mgb_quad_state(mgb_quad *h, float *state_dev, int32_t *ct_dev, int load, void *stream);

/* Exact snapshot / restore of env state (DESIGN.md "Snapshot, restore and clone").  A record is a fixed-size,
 * 16-byte-aligned row of mgb_quad_record_bytes(h) bytes per env: the six float4 state planes of the env (22 state floats,
 * ct, episode counter) and its velocity task index.  Records carry no env index: the caller matches them to envs.
 *   mgb_quad_snapshot: rec_dev [n][B] receives the record of every local env.
 *   mgb_quad_restore: row_of_env_dev [n] int64 gives, for each local env e, the row of rec_dev [n_rec][B] to load into
 *     it; a row outside [0, n_rec) leaves env e untouched.  Rows must come from a handle with the same fingerprint.  A
 *     task index outside the handle's target table leaves env2task[e] as it was.
 * Both are stream-ordered kernels, with no host synchronisation and no allocation (capturable in a CUDA graph).
 *   mgb_quad_counters: set = 0 reads the handle's rollout action counter (the step index that keys device-drawn rollout
 *     actions) into *t_base, set = 1 writes it.  Host-only, immediate.
 *   mgb_quad_fingerprint: out[MGB_FINGERPRINT_WORDS] = what a handle restoring these records must share: out[0] config
 *     (mgb_quad_cfg, auto_reset, rng seed, record size), out[1] obstacle map, out[2] velocity-target table, out[3] 0. */
#define MGB_FINGERPRINT_WORDS 4
int64_t mgb_quad_record_bytes(const mgb_quad *h);
int mgb_quad_snapshot(mgb_quad *h, uint8_t *rec_dev, void *stream);
int mgb_quad_restore(mgb_quad *h, const uint8_t *rec_dev, int64_t n_rec, const int64_t *row_of_env_dev, void *stream);
int mgb_quad_counters(mgb_quad *h, uint64_t *t_base, int set);
int mgb_quad_fingerprint(const mgb_quad *h, uint64_t *out);

/* Number of kernel launches issued through this handle so far (bench.py reports it as gpu_launches). */
int64_t mgb_quad_launch_count(const mgb_quad *h);

/* Name of the kernel an mgb_quad_step launch of this handle takes at its batch size ("quad_step_wide_kernel<..>": one
 * CTA per SM for single-wave batches of up to 384 envs per SM, MGB_WIDE_KERNEL; "quad_stream_kernel<..>": persistent TMA-pipelined variant for multi-wave batches;
 * "quad_step_kernel<..>": 64-env CTAs otherwise; "quad_step2_kernel<..>": the packed two-envs-per-thread variant, MGB_PACKED=1).
 * Reporting only (bench.py's roofline.kernel); no reference counterpart. */
const char *mgb_quad_step_kernel(const mgb_quad *h);

/* ------------------------------------------------------------------------------------------------------------ */
/* MetaMaze (2D grid + discrete-3D raycast)                                                                       */
/* ------------------------------------------------------------------------------------------------------------ */

#define MGB_MAZE_2D 0          /* MazeCore2D, maze_2d.py:13          */
#define MGB_MAZE_DISCRETE_3D 1 /* MazeCoreDiscrete3D, maze_discrete_3d.py:17 */
#define MGB_MAZE_CONTINUOUS_3D 2 /* MazeCoreContinuous3D, maze_continuous_3d.py:16 (+ dynamics.py) */

#define MGB_MAZE_SURVIVAL 0 /* maze_base.py:52-57,72-88 */
#define MGB_MAZE_ESCAPE 1   /* maze_base.py:58-60,90-93 */

#define MGB_OBS_U8 0  /* min(value, 255) as uint8 (3-D only; reference values can reach ~350 on near-floor pixels) */
#define MGB_OBS_I32 1 /* exact reference values as int32 (ray_caster_utils.py:79)                                 */
#define MGB_OBS_F32 2 /* the same exact values as float32: the dtype observation_space declares (maze_env.py:37-39)  */

/* Scalars of one TaskConfig (maze_task.py:15-17,176-190). */
typedef struct mgb_maze_task_scalars {
    int32_t start[2];
    int32_t goal[2];
    double cell_size, wall_height, agent_height;
    double initial_life, max_life, step_reward, goal_reward;
} mgb_maze_task_scalars;

typedef struct mgb_maze_cfg {
    int32_t kind;        /* MGB_MAZE_*                                                      */
    int32_t task_type;   /* MGB_MAZE_SURVIVAL / ESCAPE                                      */
    int32_t n_cells;     /* maze side n (odd, maze_task.py:56-57); <= 31                    */
    int32_t max_steps;   /* maze_base.py:191-192                                            */
    int32_t view_grid;   /* 2-D: half window g, obs (2g+1)^2 (maze_2d.py:89-121)            */
    int32_t res_h;       /* 3-D: resolution_horizon                                         */
    int32_t res_v;       /* 3-D: resolution_vertical                                        */
    int32_t obs_dtype;   /* 3-D: MGB_OBS_*                                                  */
    double max_vision;   /* 12.0, maze_discrete_3d.py:22                                    */
    double fov;          /* 0.6 * 3.1415926, maze_discrete_3d.py:23                         */
    double l_focal;      /* 0.20, maze_discrete_3d.py:116                                   */
    double text_size;    /* 1.0, maze_discrete_3d.py:116                                    */
} mgb_maze_cfg;

typedef struct mgb_maze mgb_maze;

/* MetaMaze2D.__init__ / MetaMazeDiscrete3D.__init__ (maze_env.py:156-172, 17-42) for n_envs instances. */
int mgb_maze_create(mgb_maze **out, int64_t n_envs, const mgb_maze_cfg *cfg, int device, int64_t env_index_base);
void mgb_maze_destroy(mgb_maze *h);
int64_t mgb_maze_obs_bytes_per_env(const mgb_maze *h);

/* MazeTaskManager textures (maze_task.py:19-35): grounds [n_tex][ts][ts][3] (x-major like pygame.surfarray) and
 * ceil [ts][ts][3], HOST pointers, uint8 (the reference stores the same integers as float32).  ts must be 64. */
int mgb_maze_set_textures(mgb_maze *h, const uint8_t *grounds_host, int32_t n_tex, const uint8_t *ceil_host,
                          int32_t tex_size);

/* MazeBase.set_task (maze_base.py:19-38) for a table of n_tasks TaskConfigs and the task of every local env.
 * HOST pointers, copied (synchronous): walls/texts int8 [n_tasks][n][n], food_rewards float64 [n_tasks][n][n],
 * food_interval int32 [n_tasks][n][n], scalars [n_tasks], env2task int32 [n_envs]. */
int mgb_maze_set_task(mgb_maze *h, int32_t n_tasks, const int8_t *walls_host, const int8_t *texts_host,
                      const double *food_rewards_host, const int32_t *food_interval_host,
                      const mgb_maze_task_scalars *scalars_host, const int32_t *env2task_host);

/* MazeTaskSampler keyword arguments (maze_task.py:41-54; defaults in metagym_b200/metamaze.py). */
typedef struct mgb_maze_sampler_cfg {
    int32_t allow_loops, n_texts, food_interval, pad;
    double cell_size, wall_height, agent_height, step_reward;
    double goal_reward;         /* <= 0: the reference's default -sqrt(n) * n * step_reward (maze_task.py:163-166) */
    double food_reward, initial_life, max_life, food_density, crowd_ratio;
} mgb_maze_sampler_cfg;

/* Per-episode task resampling ON THE DEVICE (maze_task.py:41-190 at the scale of SURVEY.md 8f row 3): every env e with
 * mask_dev[e] != 0 (NULL: all envs) gets a freshly drawn maze written into its task-table slot and starts an episode on
 * it; one kernel, stream-ordered, no host involvement (typical use: mask = the `done` array of the previous step).  Draws
 * come from a counter-based generator keyed by (seed, global env index, how often the env has been resampled), so results
 * do not depend on sharding.  The distribution family is MazeTaskSampler's (spanning tree of the room lattice, loops down
 * to crowd_ratio, textures, start/goal, thinned food); it is NOT sample-identical to the reference, which draws from
 * Python's and numpy's global MT19937 streams.  Food values are clip(U * food_reward, 0.10, food_reward) in np.clip's
 * order and a food cell's interval is food_interval where its value is above 1e-3, else 0, as in MazeTaskSampler.  Needs
 * one table slot per env (mgb_maze_set_task with an injective env2task) and the direct renderer; food cells per task are
 * capped at the table's largest task.  Allocates nothing (mgb_maze_set_task allocates the resample counts), so it can be
 * captured in a CUDA graph. */
int mgb_maze_resample_tasks(mgb_maze *h, const uint8_t *mask_dev, const mgb_maze_sampler_cfg *cfg, uint64_t seed,
                            void *stream);

/* Read tasks back from the table (synchronous; inspection / tests): arrays as for mgb_maze_set_task, [count] long. */
int mgb_maze_get_tasks(mgb_maze *h, int32_t count, const int32_t *task_slots_host, int8_t *walls_host, int8_t *texts_host,
                       double *food_rewards_host, int32_t *food_interval_host, mgb_maze_task_scalars *scalars_host);

/* MetaMazeDiscrete3D renderer choice.  enabled = 1 (default): static layers of every (task, cell, heading) are rendered once
 * and memoised (pose cache, within MGB_MAZE_CACHE_GB), a step composes / copies; 0: every frame is ray-cast directly
 * (ray_caster_utils.py:66-209 per frame, like the reference) -- the mode for task tables that change every episode
 * (mgb_maze_resample_tasks).  The cache is laid out per task slot (S = 4 x the most free cells of a set_task task pose
 * slots, V variant frames each), so mgb_maze_update_tasks rebuilds only the replaced tasks. */
int mgb_maze_set_cache(mgb_maze *h, int enabled);

/* Pose-cache statistics after the first reset/step (reporting only; synchronises the device to read the counts of
 * tasks mgb_maze_update_tasks rebuilt back): out[0] cached poses, out[1] extra variant frames,
 * out[2] variant bits in use (poses whose image depends on k <= bits foods have all 2^k finished frames), out[3] bytes,
 * out[4..12] poses by k (0..7, and 8 = eight or more), out[13] 1 if the cache is in use; shared-memory plan of the last
 * direct-renderer launch: out[14] 1 if the crossing lists live in a global scratch, out[15] 1 if pipelined. */
int mgb_maze_cache_info(const mgb_maze *h, int64_t out[16]);

/* Per-episode task resampling (MazeBase.set_task on a fresh TaskConfig every episode, maze_base.py:19-38, at the scale of
 * SURVEY.md 8f row 3): replace `count` entries of the table mgb_maze_set_task built -- task_slots_host [count] indices into
 * it, the other arrays as for mgb_maze_set_task but [count] long -- STREAM-ORDERED and without any device synchronisation
 * (one pinned-staged copy + three small kernels on `stream`).  Every env whose env2task entry is one of the replaced slots
 * starts a new episode on its new task (agent at start, life = initial_life, food restored), like set_task + reset of that
 * env; other envs are untouched.  The table's shape is fixed by mgb_maze_set_task: a replacement may not have more food
 * cells than the table's largest task nor smaller cells than its smallest.  MetaMazeDiscrete3D on the pose cache: the
 * replaced tasks' poses and frames are rebuilt in place in the same stream order (FILL pass, signatures, device-planned
 * variant frames, bakes, pose records; no allocation), and a replacement may not have more free cells (start cell
 * included) than the largest task of mgb_maze_set_task, nor may a slot appear twice in one call.  Before the cache's first
 * build (set_task without reset yet) only the table changes, and the first build covers it. */
int mgb_maze_update_tasks(mgb_maze *h, int32_t count, const int32_t *task_slots_host, const int8_t *walls_host,
                          const int8_t *texts_host, const double *food_rewards_host, const int32_t *food_interval_host,
                          const mgb_maze_task_scalars *scalars_host, void *stream);

/* MazeBase.reset (maze_base.py:40-63, maze_discrete_3d.py:39-49).  mask_dev NULL = all.  obs_dev NULL = skip. */
int mgb_maze_reset(mgb_maze *h, const uint8_t *mask_dev, void *obs_dev, void *stream);

/* MetaMaze*.step (maze_env.py:59-75,129-146,189-206).  act_dev is typed by the handle kind:
 *   MetaMaze2D, MetaMazeDiscrete3D: [n] int32 in 0..3; DISCRETE_ACTIONS[a] (maze_env.py:14) -> do_action ->
 *   evaluation_rule (maze_base.py:65-95) -> update_observation (maze_2d.py:89-121 | maze_discrete_3d.py:113-127 +
 *   ray_caster_utils.py).
 *   MetaMazeContinuous3D: [n][2] float32 = (turn_rate, walk_speed), clipped to [-1, 1] like the reference
 *   (maze_continuous_3d.py:47-56, dynamics.py:58-92); ten 10 ms sub-steps of turn/walk with the soft wall-repulsion
 *   collision model, then evaluation_rule and the ray-cast observation (same renderer).  Typing follows what the reference
 *   computes for float32 actions (its action_space.sample()): float32 position, float64 heading.
 *   obs_dev: 2-D float32 [n][2g+1][2g+1]; 3-D uint8|int32|float32 [n][res_h][res_v][3];
 *   rew_dev [n] float64 (the reference returns python/np float64); done_dev [n] uint8.
 * With auto_reset on (mgb_maze_set_options) a finished env is reset in the same launch and obs holds the first
 * observation of the next episode.  Two optional outputs (NULL: not produced):
 *   final_obs_dev [n][obs of one env] in the obs dtype: for every env with done = 1 in this step, the observation an
 *     auto_reset-off handle would have returned (the terminal frame, life bar included).  Rows of envs that did not
 *     finish are left untouched.  Needs auto_reset on (MGB_ERR_ARG otherwise).
 *   truncated_dev [n] uint8, written for every env: 1 iff done and the episode ended only through the step limit
 *     (SURVIVAL: life >= 0; ESCAPE: not on the goal; steps > max_steps - 1), so terminated = done && !truncated.
 * obs, rew, done and the env state are bit for bit the same with or without them.  The fused uint8 step (pose cache)
 * moves the terminal frames in the same launch (final_obs 16-byte aligned; otherwise the two-kernel path runs); the other
 * 3-D paths render them in one more launch, one frame per finished env.  Stream-ordered, no host synchronisation,
 * capturable in a CUDA graph. */
int mgb_maze_step(mgb_maze *h, const void *act_dev, void *obs_dev, double *rew_dev, uint8_t *done_dev,
                  void *final_obs_dev, uint8_t *truncated_dev, void *stream);
int mgb_maze_set_options(mgb_maze *h, int auto_reset);

/* Trials of k episodes per maze (RL^2: the agent's memory is carried across the episodes of one maze).  k >= 1 makes
 * the handle a TRIAL handle; k = 0 (the default) leaves it as it is.  Must be called before the first mgb_maze_set_task,
 * which fixes the record layout; refused (MGB_ERR_ARG) afterwards and for k < 0.  Synchronous.
 * A trial handle keeps task_episodes[e]: the episodes env e has finished (done = 1) since it was last given a maze.
 *   Every done adds 1: mgb_maze_step, mgb_maze_rollout, mgb_maze_rollout_policy and mgb_maze_rollout_rnn.
 *   It goes to 0 where the env gets a maze: mgb_maze_set_task (all envs), mgb_maze_update_tasks (envs of the replaced
 *   slots), mgb_maze_resample_tasks (masked envs) and an in-launch draw.  mgb_maze_reset does not change it.
 *   With resample_cfg, an env that finishes at step t draws a new maze only when its count after step t reaches k (and
 *   the count returns to 0); otherwise it auto-resets on its old maze exactly as without resample_cfg, and its resample
 *   count is unchanged.  The rollout then equals, step for step, step + resample_tasks(m) + reset(mask = m) with
 *   m = done && task_episodes >= k.  The recurrent "task" reset rule zeroes the state where the env drew.
 *   Without resample_cfg a step or rollout takes the counts from done_dev, which may then not be NULL (MGB_ERR_ARG,
 *   handle untouched); one more small kernel follows the launch.  k = 1 gives exactly the outputs of a handle without
 *   trials.  Snapshot records gain one 16-byte block (mgb_maze_snapshot below).
 *   mgb_maze_task_episodes: the counts as int32 [n] into out_dev; stream-ordered, capturable in a CUDA graph.  Refused on
 *   a handle that is not a trial handle. */
int mgb_maze_set_episodes_per_task(mgb_maze *h, int32_t k);
int mgb_maze_task_episodes(mgb_maze *h, int32_t *out_dev, void *stream);

/* T consecutive mgb_maze_step calls (the random-action loops of metamaze/test.py:9-67) in ONE launch; auto-reset
 * semantics as configured, state left as T steps leave it.  The handle picks the engine:
 *   MetaMaze2D: agent state in registers.
 *   MetaMazeDiscrete3D without resample_cfg: the pose cache when it is in use (one CTA per env, step logic by one thread,
 *   frame by the CTA); otherwise, and always with resample_cfg, the direct renderer (every frame ray-cast).  Both give
 *   the same outputs, env state and step counter.
 *   MetaMazeContinuous3D: the direct renderer.
 *   act_dev [T][n] int32 in 0..3 (MetaMazeContinuous3D: float32 [T][n][2]) or NULL: NULL draws the actions from the
 *   counter-based generator (stream id act_seed, keyed by the global env index, counted across calls) -- uniform {0..3},
 *   or turn_rate and walk_speed uniform on [-1, 1) -- written to act_out_dev (same shape) if not NULL.
 *   obs_dev [T][n][obs of one env] (2-D: float32 [2g+1][2g+1]; 3-D: uint8, int32 or float32 [res_h][res_v][3]),
 *   rew_dev [T][n] float64, done_dev [T][n] uint8.  Any may be NULL, except on the direct renderer.
 * Two optional outputs per step (NULL: not produced):
 *   final_obs_dev [T][n][obs of one env] in the obs dtype: row (t, e) is written only when done[t][e] = 1, with the
 *     observation an auto_reset-off handle would have returned at step t (update_observation on the state
 *     evaluation_rule left: maze_2d.py:89-121; maze_discrete_3d.py:113-127 with the food it left and the life bar at the
 *     terminal life; maze_continuous_3d.py:47-56 then the ray-cast observation).  Rows with done = 0 are not written.
 *     Needs auto_reset on (MGB_ERR_ARG otherwise).
 *   truncated_dev [T][n] uint8, written for every (t, e): 1 iff done and the episode ended only through the step limit
 *     (maze_base.py:80,91-95,191-192).
 * obs, rew, done, the drawn actions, the generator's step counter, the env state and the pose are bit for bit the same
 * with or without them.  On the 3-D engines a finished env costs one more frame in the same launch.
 *   resample_cfg NULL: no resampling; the outputs and the env state are bit for bit those of T step() calls.
 *   resample_cfg set (the data-generation loop of meta-RL over an endless stream of tasks): when env e finishes at step t
 *   (done, auto-reset on), its reward, done, truncated[t][e] and final_obs[t][e] come from the old task; then it gets the
 *   task mgb_maze_resample_tasks(mask with only e set, resample_cfg, resample_seed) would give it -- written into its
 *   table slot, resample count + 1 -- and starts its next episode on it (start cell, initial_life, every food present):
 *   obs[t][e] is its first observation on the NEW maze.  That equals, step for step, step + resample_tasks(done) +
 *   reset(mask = done) (without the extra render).
 * MetaMaze2D without resample_cfg delivers obs, rew, done and act_out through output mirrors or multicast when they are
 * set (mgb_maze_set_mirrors, mgb_maze_set_multicast below).
 * Refused (MGB_ERR_ARG, handle untouched): T <= 0; final_obs without auto-reset; final_obs or truncated while output
 * mirrors or multicast are set; output mirrors or multicast on a 3-D handle or with resample_cfg; NULL obs, rew or done on
 * the direct renderer; a screen too large for the pose cache's group queue.  With resample_cfg also: auto-reset off,
 * every refusal of mgb_maze_resample_tasks (one slot per env, a discrete handle whose pose cache is in use, the cfg
 * checks) with the same messages, and on MetaMaze2D shared memory per CTA (two tiles of 128 windows plus four sampler
 * workspaces) beyond the device's opt-in limit (n = 31 needs view_grid <= 6).
 * Advances the step counter by T.  Stream-ordered, no host synchronisation, no allocation after the handle's first
 * reset() (which builds the pose cache and sizes the renderer's scratch): capturable in a CUDA graph. */
int mgb_maze_rollout(mgb_maze *h, int32_t T, const void *act_dev, uint64_t act_seed, void *act_out_dev,
                     void *obs_dev, double *rew_dev, uint8_t *done_dev, void *final_obs_dev, uint8_t *truncated_dev,
                     const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed, void *stream);

/* Expert (ESCAPE on MetaMaze2D and MetaMazeDiscrete3D; DESIGN.md §4d "Expert").  Per task slot, a breadth-first search
 * backwards from the goal over the step's own action model:
 *   MetaMaze2D: the states are the cells, the actions the four of DISCRETE_ACTIONS (maze_2d.py:21-34); a move into a
 *   wall or off the grid leaves the agent in place and still takes a step.  One heading plane.
 *   MetaMazeDiscrete3D: the states are (heading, cell), 4 n^2 of them; an action turns, then moves
 *   (maze_discrete_3d.py:51-81).
 *   dist(s): the fewest actions from s after which the agent stands on the goal cell (evaluation_rule ends the episode
 *   there, maze_base.py:90-93); 0 on the goal, 0xFFFF where the goal cannot be reached.
 *   mask(s): bit a set iff dist(next(s, a)) = dist(s) - 1; 0 on the goal and on unreachable states.
 * Tables: dist uint16 and mask uint8 [slot][planes][n][n] (planes: 1 for MetaMaze2D, 4 indexed by heading), entry
 * ((slot planes + ori) n + gx) n + gy.  Every integer, so the tables are exact.  They are rebuilt on the stream of the
 * call that changes the task table, for exactly the slots it changes: mgb_maze_set_task (every slot),
 * mgb_maze_update_tasks (the replaced slots), mgb_maze_resample_tasks (the drawn slots) and mgb_maze_restore (the slots
 * of the restored envs, when records carry their tasks).  None of them gains a host synchronisation.
 * Decision of step t of env e (global index genv = env_index_base + e) on a state with mask m: Philox4x32-10 counter
 * (genv lo, genv hi, t_base + t, MGB_STREAM_EXPERT = 0x800), key = seed, words r.x, r.y.  The choice set C is {0..3}
 * when (r.x >> 8) 2^-24 < eps (float32 compare) or m = 0, else the bits of m; the action is the j-th lowest member of
 * C, j = floor(r.y |C| / 2^32).  Mean mode (mode 1): no draw and no eps; the lowest member of m, or 0 where m = 0.
 *
 * mgb_maze_set_expert(h, on): makes h an expert handle.  Before the first mgb_maze_set_task only, like
 *   mgb_maze_set_episodes_per_task; refused afterwards, and with on for SURVIVAL or MetaMazeContinuous3D.
 * mgb_maze_rollout_expert: mgb_maze_rollout without resampling whose action at step t is act_dev[t] when act_dev is
 *   given, else the expert's decision on the state the env holds before step t (written to act_out_dev if not NULL).
 *   expert_out_dev [T][n] uint8 (or NULL): the mask of that state (DAgger labels).  The env side is bit for bit
 *   mgb_maze_rollout fed act_out: auto-reset, final_obs / truncated, trial counts, path recording; every engine
 *   (MetaMaze2D, the pose cache, the direct renderer) gives the same outputs.  mode 0 samples, mode 1 is the mean mode.
 *   obs_dev, rew_dev and done_dev are required.  Advances the step counter by T.
 * mgb_maze_step_expert: mgb_maze_step, then expert_out_dev [n] uint8: the mask of every env's state after the step,
 *   the one its next action acts on (what mgb_maze_expert returns then).
 * mgb_maze_expert: the mask (uint8 [n]) and, if dist_out_dev is not NULL, the dist (uint16 [n]) of every env's state.
 * mgb_maze_expert_table: the tables of slots [slot0, slot0 + count), mask uint8 and (if not NULL) dist uint16
 *   [count][planes][n][n].
 * All of them are stream-ordered, allocate nothing after the first reset() and can be captured in a CUDA graph.
 * Refused (MGB_ERR_ARG, handle untouched), with a message naming the reason: a handle that is not an expert handle,
 * SURVIVAL, MetaMazeContinuous3D, output mirrors or multicast set, eps not finite or outside [0, 1], a mode other than
 * 0 or 1, T <= 0, a NULL required output, final_obs without auto_reset, a slot range outside the table.
 * In-launch resampling is not offered: the kernels that draw a new maze into a slot cannot rebuild its tables.  So on an
 * expert handle every call with a resample_cfg (mgb_maze_rollout, mgb_maze_rollout_policy, mgb_maze_rollout_rnn, their
 * population and critic forms, mgb_maze_evaluate) is refused (MGB_ERR_ARG, handle untouched); mgb_maze_resample_tasks
 * between launches keeps the tables current. */
int mgb_maze_set_expert(mgb_maze *h, int on);
int mgb_maze_rollout_expert(mgb_maze *h, int32_t T, const int32_t *act_dev, float eps, int32_t mode, uint64_t seed,
                            int32_t *act_out_dev, uint8_t *expert_out_dev, void *obs_dev, double *rew_dev,
                            uint8_t *done_dev, void *final_obs_dev, uint8_t *truncated_dev, void *stream);
int mgb_maze_step_expert(mgb_maze *h, const int32_t *act_dev, void *obs_dev, double *rew_dev, uint8_t *done_dev,
                         void *final_obs_dev, uint8_t *truncated_dev, uint8_t *expert_out_dev, void *stream);
int mgb_maze_expert(mgb_maze *h, uint8_t *mask_out_dev, uint16_t *dist_out_dev, void *stream);
int mgb_maze_expert_table(mgb_maze *h, int32_t slot0, int32_t count, uint8_t *mask_out_dev, uint16_t *dist_out_dev,
                          void *stream);

/* mgb_maze_rollout of a MetaMaze2D handle (resample_cfg NULL: no resampling; set: in-launch resampling) with
 * actions from a categorical MLP policy (mgb_policy, "policy-driven rollouts" above; input width (2 view_grid + 1)^2,
 * the four outputs are the logits of actions 0..3, no log_std).
 *   Sampling: u = (x >> 8) 2^-24 of the first Philox word; the float32 softmax of the logits is accumulated in index
 *   order into c_0..c_2, and the action is the first k with u < c_k, else 3.  logp = l_a - logsumexp(l).
 *   MGB_POLICY_MEAN: the argmax, ties to the lowest index, and logp_out must be NULL.
 *   act_out_dev [T][n] int32, logp_out_dev [T][n] float32, obs0_out_dev [n][D] float32: the window the policy acted on
 *   at t = 0, computed from the handle's state; at t > 0 it acted on obs[t-1] (post auto-reset and resampling).
 *   obs, rew, done, final_obs, truncated: as mgb_maze_rollout.  Every output may be NULL.
 * The env side is bit for bit mgb_maze_rollout fed act_out.  The step counter advances
 * by T; nothing is allocated, and the call can be captured in a CUDA graph.  Refused (MGB_ERR_ARG, handle untouched):
 * a 3-D handle, T <= 0, a NULL policy or params_dev, n_hidden / width / activation / mode out of range, logp_out in mean
 * mode, output mirrors or multicast set, final_obs without auto_reset, resample_cfg where mgb_maze_rollout
 * refuses it (same reasons), and observation tiles, sampler workspaces, weights and activations of 128 envs beyond the
 * device's opt-in shared memory (a large view_grid with wide layers). */
int mgb_maze_rollout_policy(mgb_maze *h, int32_t T, const mgb_policy *pol, uint64_t seed,
                            const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed, int32_t *act_out_dev,
                            float *logp_out_dev, float *obs0_out_dev, float *obs_dev, double *rew_dev, uint8_t *done_dev,
                            float *final_obs_dev, uint8_t *truncated_dev, void *stream);

/* ---- recurrent policies (DESIGN.md "Recurrent policies") ----------------------------------------------------------
 * A GRU cell (torch.nn.GRUCell(in, H); cell = MGB_RNN_CELL_GRU) or an LSTM cell (torch.nn.LSTMCell(in, H); cell =
 * MGB_RNN_CELL_LSTM, below) followed by a head, evaluated inside a MetaMaze2D rollout launch.  The GRU's memory is a
 * caller-owned float32 state [n][S], S = H + 5 feedback, row e = [c (H), onehot(prev action) (4), (float)prev reward
 * (1)] (the last five only with feedback = 1).
 *   Input of step t: x_t = [obs (D = (2 view_grid + 1)^2), then with feedback the five feedback entries of the state].
 *   params_dev: float32 on the handle's device, read at every launch.  weight_ih [3H][in], weight_hh [3H][H], bias_ih
 *     [3H], bias_hh [3H] (gate order r, z, n; a cell without bias packs zeros), then the head in torch.nn.Linear order:
 *     W [4][H], b [4] (head_hidden = 0) or W1 [w][H], b1 [w], W2 [4][w], b2 [4] (head_hidden = 1, w = head_width,
 *     hidden activation MGB_ACT_*).
 *   Step t: h_t = GRU(x_t, c_t); the action is drawn from head(h_t) exactly as mgb_maze_rollout_policy draws it from
 *     its logits (categorical head, MGB_STREAM_POLICY, counter (genv, t_base + t)).  Then, if done[t] and the reset rule
 *     fires, the whole state row becomes zero; otherwise c_{t+1} = h_t and the feedback entries become
 *     (onehot(a_t), (float)r_t).  MGB_RNN_RESET_EPISODE fires on every done; MGB_RNN_RESET_TASK fires where the env drew
 *     a new maze in this launch (a rollout with resample_cfg), so without resampling it never fires inside a launch and
 *     the caller zeroes the rows of envs it gives a new task (set_task, update_tasks, resample_tasks).
 * Numerical contract (float32, no tensor cores, no approximate instructions; u = 2^-24):
 *   gi_k[j] = fma chain from bias_ih[kH + j] over x_t[i], i = 0..in-1 in index order: acc = fmaf(W_ih[kH + j][i], x_i, acc);
 *   gh_k[j] likewise from bias_hh[kH + j] over c_t[i], i = 0..H-1.  k = r, z, n.
 *   r = 1 / (1 + expf(-(gi_r + gh_r))), z likewise: the two chains are added in one float32 add, then expf (at most 2
 *     ulp), one add and one correctly rounded division.
 *   n = tanhf(fmaf(r, gh_n, gi_n)) (one rounding inside, tanhf at most 2 ulp).
 *   h' = fmaf(z, c, (1 - z) n): 1 - z and its product with n are rounded, then one fused multiply-add.
 *   The head is the MLP of mgb_policy on h_t (fma chains from the bias, accurate tanhf).
 * LSTM (cell = MGB_RNN_CELL_LSTM): everything above holds except the following.
 *   State [n][S], S = 2H + 5 feedback, row e = [h (H), c (H), onehot(prev action) (4), (float)prev reward (1)].
 *   params_dev: weight_ih [4H][in], weight_hh [4H][H], bias_ih [4H], bias_hh [4H] (torch's gate order i, f, g, o; a
 *     cell without bias packs zeros), then the head as for the GRU.
 *   Step t: (h_t, c'_t) = LSTM(x_t, (h_{t-1}, c_{t-1})); the action is drawn from head(h_t) as for the GRU.  Then, if
 *     done[t] and the reset rule fires, the whole state row (h, c and feedback) becomes zero; otherwise h and c carry
 *     and the feedback entries become (onehot(a_t), (float)r_t).  hid_out holds h_t.
 *   gi_k[j] = fma chain from bias_ih[kH + j] over x_t[i], i = 0..in-1 in index order; gh_k[j] likewise from
 *     bias_hh[kH + j] over h_{t-1}[i], i = 0..H-1.  k = i, f, g, o.  v_k = gi_k + gh_k in one float32 add.
 *   i = 1 / (1 + expf(-v_i)), f and o likewise (expf at most 2 ulp, one add, one correctly rounded division);
 *     g = tanhf(v_g) (at most 2 ulp).
 *   c' = fmaf(f, c, i g): the product i g is rounded, then one fused multiply-add.
 *   h' = o tanhf(c'): tanhf at most 2 ulp, then one rounded product. */
#define MGB_RNN_RESET_EPISODE 0   /* zero the state row at every done */
#define MGB_RNN_RESET_TASK 1      /* zero it where the env drew a new maze in this launch (in-launch resampling) */
#define MGB_RNN_MAX_HIDDEN 64
#define MGB_RNN_CELL_GRU 0        /* torch.nn.GRUCell */
#define MGB_RNN_CELL_LSTM 1       /* torch.nn.LSTMCell */

typedef struct mgb_rnn_policy {
    const float *params_dev;  /* packed float32 on the handle's device, read at every launch */
    int32_t hidden;           /* H, 1..64 */
    int32_t feedback;         /* 0 or 1: the input ends with onehot(prev action) and prev reward */
    int32_t reset;            /* MGB_RNN_RESET_* */
    int32_t head_hidden;      /* 0: Linear(H, 4); 1: Linear(H, w), activation, Linear(w, 4) */
    int32_t head_width;       /* w, 1..64 when head_hidden = 1 (ignored otherwise) */
    int32_t activation;       /* MGB_ACT_* of the head's hidden layer */
    int32_t mode;             /* MGB_POLICY_* */
    int32_t cell;             /* MGB_RNN_CELL_* (0, the GRU, for callers that predate the field) */
} mgb_rnn_policy;

/* mgb_maze_rollout_policy with a recurrent policy (mgb_rnn_policy above) on a MetaMaze2D handle with auto_reset on.
 *   state_dev [n][S] float32: read at launch start, written back in place at launch end (4-byte aligned, not NULL).
 *   state0_out_dev [n][S]: the state as read.  hid_out_dev [T][n][H]: h_t.  Both may be NULL.
 *   act_out, logp_out, obs0_out, obs, rew, done, final_obs, truncated, seed, resample_cfg, resample_seed: as
 *   mgb_maze_rollout_policy.  The env side is bit for bit mgb_maze_rollout fed act_out.  The step counter advances by
 *   T; nothing is allocated, and the call can be captured in a CUDA graph.  Refused (MGB_ERR_ARG; the handle, its step
 *   counter and the state untouched): everything mgb_maze_rollout_policy refuses, a NULL or misaligned state_dev,
 *   auto_reset off, hidden / feedback / reset / head_hidden / head_width / activation / mode out of range, an unknown
 *   cell, and observation tiles, sampler workspaces, weights and activations of 128 envs beyond the device's opt-in
 *   shared memory (a large view_grid with a wide cell; DESIGN.md "Recurrent policies" lists what fits). */
int mgb_maze_rollout_rnn(mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, uint64_t seed,
                         const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                         float *state_dev, float *state0_out_dev, float *hid_out_dev,
                         int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                         float *obs_dev, double *rew_dev, uint8_t *done_dev,
                         float *final_obs_dev, uint8_t *truncated_dev, void *stream);

/* mgb_maze_rollout_policy and mgb_maze_rollout_rnn with a population of `members` policies of pol's shape (DESIGN.md
 * "Populations"): member m's packed buffer starts at pol->params_dev + m member_stride floats, and with E = n / members
 * it drives the envs [m E, (m + 1) E) of the handle (its rows of state_dev too).  Every other input, output, draw
 * (keyed by the global env index) and refusal is that of the single-policy call, and members = 1 is that call exactly
 * (the stride is then not read).  Also refused (MGB_ERR_ARG; the handle, its step counter and the state untouched):
 * members < 1, n not a multiple of members, E not 32, 64 or a multiple of MGB_MAZE2D_POLICY_CTA_ENVS, member_stride
 * below the packed length, and the staged members of one CTA with the tiles and activations beyond the device's opt-in
 * shared memory. */
int mgb_maze_rollout_population(mgb_maze *h, int32_t T, const mgb_policy *pol, int32_t members, int64_t member_stride,
                                uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                                int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev, float *obs_dev,
                                double *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                                void *stream);
int mgb_maze_rollout_rnn_population(mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                                    int64_t member_stride, uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg,
                                    uint64_t resample_seed, float *state_dev, float *state0_out_dev, float *hid_out_dev,
                                    int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev, float *obs_dev,
                                    double *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                                    void *stream);

/* ---- value heads and GAE (DESIGN.md "Value heads and GAE") -------------------------------------------------------
 * The *_critic entry points are the population calls (members = 1: the single policy) with a critic: the packed
 * buffer's output layer has 5 rows, W [5][k] then b [5], rows 0..3 the actor's outputs and row 4 the value V (k: the
 * last hidden width, the obs dim with no hidden layer, H or the head's hidden width for the recurrent head).  The
 * quadrotor's log_std [4] still follows.  Rows 0..3, and with them every action, logp and env output, are bit for bit
 * those of the same call on the buffer without row 4.  V is the fma chain of row 4 from its bias, like the others.
 *   value_dev [T][n] float32 (not NULL): V(s_t) on the input step t acts on (obs0 at t = 0).
 *   value_last_dev [n]: V(s_T) on the observation and carried state the launch leaves behind; it equals value[0] of the
 *     next launch bit for bit when nothing touches the handle or the state in between.
 *   final_value_dev [T][n]: V of the terminal observation, written only where the cut fires (below) on a truncated step;
 *     other entries keep what they held.  Recurrent: the cell steps once more from the memory before the wipe (h_t, and
 *     the LSTM's c'_t) on [terminal window, onehot(a_t), (float)r_t].
 *   The cut is where the policy's memory is wiped: every done for an MLP and MGB_RNN_RESET_EPISODE, and where the env drew
 *     a new maze in this launch for MGB_RNN_RESET_TASK.
 *   adv_dev, ret_dev [T][n] (both or neither; they need rew, done, truncated and final_value): GAE(gamma, lambda) over
 *     the launch, float32, each operation rounded to nearest, no contraction; r_t is the reward rounded once to float32.
 *     gl = gamma lambda; for t = T-1 .. 0: nv = cut_t ? (truncated_t ? final_value_t : 0)
 *     : (t = T-1 ? value_last : value_{t+1}); delta = (r_t + gamma nv) - v_t; A_t = delta + (cut_t ? 0 : gl A_{t+1}),
 *     A_T = 0; ret_t = A_t + v_t.
 *   Every other argument is the population call's.  Refused (MGB_ERR_ARG; the handle, its step counter and the state
 *   untouched): everything the population call refuses, a NULL critic, auto_reset off, a NULL value_dev, adv / ret
 *   without each other or without rew, done, truncated and final_value, gamma or lambda not finite or outside [0, 1],
 *   and the footprint beyond the device's opt-in shared memory. */
typedef struct mgb_critic {
    float *value_dev;         /* [T][n], not NULL */
    float *value_last_dev;    /* [n] or NULL */
    float *final_value_dev;   /* [T][n] or NULL */
    float *adv_dev;           /* [T][n] or NULL */
    float *ret_dev;           /* [T][n] or NULL */
    float gamma;              /* discount, [0, 1] */
    float lambda;             /* GAE lambda, [0, 1] */
} mgb_critic;

int mgb_quad_rollout_critic(mgb_quad *h, int32_t T, const mgb_policy *pol, int32_t members, int64_t member_stride,
                            uint64_t seed, float *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                            float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                            uint8_t *truncated_dev, const mgb_critic *critic, void *stream);
int mgb_maze_rollout_critic(mgb_maze *h, int32_t T, const mgb_policy *pol, int32_t members, int64_t member_stride,
                            uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                            int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev, float *obs_dev,
                            double *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                            const mgb_critic *critic, void *stream);
int mgb_maze_rollout_rnn_critic(mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                                int64_t member_stride, uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg,
                                uint64_t resample_seed, float *state_dev, float *state0_out_dev, float *hid_out_dev,
                                int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev, float *obs_dev,
                                double *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                                const mgb_critic *critic, void *stream);

/* ---- recurrent quadrotor policies (DESIGN.md "Recurrent quadrotor policies") ---------------------------------------
 * The cells of "recurrent policies" above (mgb_rnn_policy, unchanged) with a Gaussian head, driving a quadrotor handle
 * with auto_reset on.  The packed buffer is the maze's (the cell, then the head, with its value row for the critic)
 * followed by log_std [4], always, as for mgb_quad_rollout_policy.
 *   Input of step t: x_t = [obs_t (D = 16, or 19 for velocity_control), then with feedback a_{t-1} (4), r_{t-1} (1)]:
 *     the raw action the policy drew (as stored in act_out, not clamped) and the float32 reward.  The feedback entries
 *     of the state row hold them; S = H + 5 (GRU) or 2H + 5 (LSTM), as on the maze.
 *   Step t: h_t from the cell exactly as on the maze; mean = head(h_t); the action is drawn exactly as
 *     mgb_quad_rollout_policy draws it (Philox counter (genv, t_base + t, MGB_STREAM_POLICY), Box-Muller, the same
 *     logp), so one seed gives the same z for every quadrotor policy.  Then the whole state row (h, c and feedback) is
 *     zeroed at every done (reset must be MGB_RNN_RESET_EPISODE: a quadrotor task never changes inside a launch);
 *     otherwise h and c carry and the feedback becomes (a_t, r_t).
 *   state_dev [n][S] float32: read at launch start, written back in place at launch end (4-byte aligned, not NULL).
 *   state0_out_dev [n][S]: the state as read.  hid_out_dev [T][n][H]: h_t.  Both may be NULL.
 *   act_out, logp_out, obs0_out, obs, rew, done, final_obs, truncated, seed: as mgb_quad_rollout_policy.  The env side
 *   is bit for bit mgb_quad_rollout_ex fed act_out.  The step counter advances by T; nothing is allocated, and the call
 *   can be captured in a CUDA graph.
 *   Populations: as mgb_quad_rollout_population, with E = n / members 32, 64 or a multiple of MGB_QUAD_RNN_CTA_ENVS.
 *   Critic: as mgb_quad_rollout_critic; final_value comes from the memory before the wipe (h_t, and the LSTM's c'_t):
 *     the cell steps once more on [terminal obs, a_t, r_t].
 * Refused (MGB_ERR_ARG; the handle, its step counter and the state untouched): everything mgb_quad_rollout_policy (and
 * the population and critic calls) refuse, reset other than MGB_RNN_RESET_EPISODE, auto_reset off, a NULL or
 * misaligned state_dev, hidden / feedback / head_hidden / head_width / activation / mode out of range, an unknown cell,
 * and weights, observation tiles and columns of MGB_QUAD_RNN_CTA_ENVS envs beyond the device's opt-in shared memory
 * (the message gives the byte count; DESIGN.md "Recurrent quadrotor policies" lists what fits). */
int mgb_quad_rollout_rnn(mgb_quad *h, int32_t T, const mgb_rnn_policy *pol, uint64_t seed, float *state_dev,
                         float *state0_out_dev, float *hid_out_dev, float *act_out_dev, float *logp_out_dev,
                         float *obs0_out_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                         uint8_t *truncated_dev, void *stream);
int mgb_quad_rollout_rnn_population(mgb_quad *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                                    int64_t member_stride, uint64_t seed, float *state_dev, float *state0_out_dev,
                                    float *hid_out_dev, float *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                                    float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                                    uint8_t *truncated_dev, void *stream);
int mgb_quad_rollout_rnn_critic(mgb_quad *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                                int64_t member_stride, uint64_t seed, float *state_dev, float *state0_out_dev,
                                float *hid_out_dev, float *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                                float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                                uint8_t *truncated_dev, const mgb_critic *critic, void *stream);

/* ---- whole-episode evaluation (DESIGN.md "Whole-episode evaluation") -----------------------------------------------
 * Per-episode returns of a policy in ONE launch: every env steps until its `episodes`-th done and then stops.  One entry
 * point per engine serves every policy kind.
 *   Policy: exactly one of mlp (as mgb_*_rollout_policy) and rnn (as mgb_*_rollout_rnn) is set.  members = 1: a single
 *     policy; otherwise member m drives the envs [m E, (m + 1) E), E = n / members under the population calls' rules
 *     (member_stride as there).  state_dev [n][S] goes with rnn only, read at launch start and written back at launch
 *     end as in mgb_*_rollout_rnn.  value_row = 1: the packed output layer has the critic's fifth row (the *_critic
 *     layout); it is skipped, never evaluated.  seed keys the policy's draws; mode MGB_POLICY_MEAN draws nothing.
 *   Stopping rule: let t = 0, 1, ... count env e's steps in this launch.  Step t is, bit for bit, step t of the policy
 *     rollout with the same handle state, policy, seed, carried state and resample_cfg: the same Philox counter
 *     (genv, t_base + t), auto-reset, in-launch resampling (MetaMaze2D), trial counting and path recording.  Env e stops
 *     after its episodes-th done, at step L_e; its state (the quadrotor's rigid body, ct and episode counter; the
 *     maze's agent, life, food, steps, task slot, resample count, trial count and path) and its row of state_dev are
 *     then what a rollout of exactly L_e steps leaves, so successive calls score consecutive episodes.
 *   Outputs, [episodes][n] (episode-major, like the rollouts' [T][n]), none NULL:
 *     return_dev: the float64 sum in step order of episode j's rewards (the steps after done number j - 1, up to and
 *       including done number j; episode 0 starts at launch start).  Quadrotor rewards are float32 widened one by one.
 *     length_dev: the steps of episode j.  truncated_dev: the rollout's truncated flag at that done (1 only when the
 *       episode ended through the time limit alone).
 *   Episode 0 is counted from whatever state the env holds at launch start: reset() first for clean episodes (the
 *   quadrotor's reset() leaves ct alone, as the reference's does).  Each episode ends within the time limit (nt on the
 *   quadrotor, max_steps on the maze), so the launch takes at most B = episodes x limit steps, and the step counter
 *   advances by B.  No host synchronisation and no allocation; the call can be captured in a CUDA graph.
 * Refused (MGB_ERR_ARG; the handle, its step counter and the state untouched): everything the matching rollout call
 * refuses, auto_reset off, episodes < 1, B above 2^31 - 1, both or neither of mlp / rnn, state_dev NULL with rnn or set
 * with mlp, value_row other than 0 or 1, a NULL output, a 3-D maze handle, and output mirrors or multicast set. */
int mgb_quad_evaluate(mgb_quad *h, int32_t episodes, const mgb_policy *mlp, const mgb_rnn_policy *rnn,
                      int32_t value_row, int32_t members, int64_t member_stride, uint64_t seed, float *state_dev,
                      double *return_dev, int32_t *length_dev, uint8_t *truncated_dev, void *stream);
int mgb_maze_evaluate(mgb_maze *h, int32_t episodes, const mgb_policy *mlp, const mgb_rnn_policy *rnn,
                      int32_t value_row, int32_t members, int64_t member_stride, uint64_t seed,
                      const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed, float *state_dev,
                      double *return_dev, int32_t *length_dev, uint8_t *truncated_dev, void *stream);

/* ---- recurrent cell sequences (DESIGN.md "Fused unroll") ----------------------------------------------------------
 * The learner's side of the recurrent policies: the cell of mgb_rnn_policy run over T given steps of n envs, forward and
 * backward, with no env and no head.  A PPO update recomputes h_t with autograd from a rollout's inputs; the head, the
 * log-softmax and the weight gradients are batched GEMMs over all T n rows and stay with the caller.
 *   params_dev: weight_ih [G H][in], weight_hh [G H][H], bias_ih [G H], bias_hh [G H] (G = 3 for the GRU, 4 for the LSTM;
 *     zeros for a cell without bias): the cell part of mgb_rnn_policy's packed buffer.
 *   x_dev [T][in][n]: the cell's input of step t for env e at (t in + i) n + e.
 *   wipe_dev [T][n] uint8: nonzero where the state is zeroed after step t (the reset rule of the rollout that made x).
 *   state0_dev [n][HC]: the memory going into step 0, HC = H (GRU: h) or 2H (LSTM: h, c).
 *   h_dev [T][n][H]: h_t.
 * mgb_rnn_seq_forward: for t = 0 .. T-1, (h, c) = cell(x_t, memory), the memory being state0 at t = 0, zeros where
 *   wipe[t-1] and (h_{t-1}, c_{t-1}) otherwise; the arithmetic of "Recurrent policies" above, so h_t equals the rollout's
 *   hid_out bit for bit on equal inputs.  With gates_dev [T][S][H][n] (S = 4) it also saves what the backward reads, unit
 *   j of env e at ((t S + s) H + j) n + e: the GRU's r, z, n and W_hn h_{t-1} + b_hn, the LSTM's i, f, g, o; the LSTM
 *   saves c_t as s = 4 (S = 5).  gates_dev NULL saves nothing.  Reads params, x, wipe, state0; writes h (and gates).
 * mgb_rnn_seq_backward: from dh_dev [T][n][H] = dL/dh_t and the saved gates (and h for the GRU), walks t = T-1 .. 0 and
 *   writes the gate pre-activation gradients dgi_dev [T][G H][n] (gate block k, unit j of env e at ((t G + k) H + j) n + e;
 *   = dL/d(W_ih x + b_ih)), for the GRU dghn_dev [T][H][n], the n block of dL/d(W_hh h + b_hh), whose r and z blocks
 *   equal dgi's, and dstate0_dev [n][HC].  The gradient carried into step t-1 is dropped where wipe[t-1].  Each env is
 *   summed in a fixed order by one thread: no atomics, the result is deterministic.  Reads params, wipe, state0, h (GRU),
 *   gates and dh; writes dgi, dghn and dstate0.
 * Both are stream-ordered, allocate nothing and can be captured in a CUDA graph; offsets are 64-bit.  The CTA holds
 * MGB_RNN_SEQ_CTA_ENVS envs.  Refused (MGB_ERR_ARG, nothing written): a NULL seq, an unknown cell, hidden outside 1..64,
 * in, T or n below 1, a NULL pointer the call reads or writes, and a footprint beyond the current device's opt-in shared
 * memory (forward: the cell's staged weights and the columns x, c, h of the CTA's envs; backward: weight_hh and two
 * columns; DESIGN.md "Fused unroll" restates both). */
#define MGB_RNN_SEQ_CTA_ENVS 128
typedef struct mgb_rnn_seq {
    int32_t cell;             /* MGB_RNN_CELL_* */
    int32_t hidden;           /* H, 1..64 */
    int32_t in;               /* inputs per step, >= 1 */
    int32_t T;                /* steps, >= 1 */
    int64_t n;                /* envs, >= 1 */
    const float *params_dev;  /* cell weights, above */
    const float *x_dev;       /* [T][in][n] (forward) */
    const uint8_t *wipe_dev;  /* [T][n] */
    const float *state0_dev;  /* [n][HC] */
    float *h_dev;             /* [T][n][H]: written by the forward, read by the GRU's backward */
    float *gates_dev;         /* [T][S][H][n]: written by the forward (or NULL), read by the backward */
    const float *dh_dev;      /* [T][n][H] (backward) */
    float *dgi_dev;           /* [T][G H][n] (backward) */
    float *dghn_dev;          /* [T][H][n] (backward, GRU) */
    float *dstate0_dev;       /* [n][HC] (backward) */
} mgb_rnn_seq;

int mgb_rnn_seq_forward(const mgb_rnn_seq *seq, void *stream);
int mgb_rnn_seq_backward(const mgb_rnn_seq *seq, void *stream);

/* Continuous pose (maze_continuous_3d.py:47-56, dynamics.py:71-92): pos_dev [n][2] float32 (_agent_loc), ori_dev [n]
 * float64 (_agent_ori). */
int mgb_maze_pose(mgb_maze *h, float *pos_dev, double *ori_dev, void *stream);

/* Inspection (info["steps"] maze_env.py:73; _agent_grid, _agent_ori_index, _life of maze_base.py:40-63): agent [n][4]
 * int32 = grid_x, grid_y, ori_index, steps; life [n] float64. */
int mgb_maze_state(mgb_maze *h, int32_t *agent_dev, double *life_dev, void *stream);
int64_t mgb_maze_launch_count(const mgb_maze *h);

/* God view (the right-hand panel that MazeBase.render_init + render_update draw, maze_base.py:100-157, with the agent
 * marker of maze_2d.py:73-75 / maze_discrete_3d.py:88-99 / maze_continuous_3d.py:63-74) of `count` envs in one launch:
 * white floor, black walls, the ESCAPE goal in green, SURVIVAL food as (f, 255, f) with f = int(255 - 255 food) on the
 * live food state, then the agent (2-D: red cell; 3-D: green disc and heading line).  The text labels are not drawn.
 *   envs_dev [count] int32 local env indices, or NULL for envs 0 .. count-1 (count <= n_envs); an index outside
 *     [0, n_envs) gives an all-zero frame.
 *   view_size S in [1, 4096]: the reference's render_scale; cell size S / n_cells, need not be an integer.
 *   out_dev [count][S][S][3] uint8, IMAGE ROWS TOP TO BOTTOM: out[k][y][x] is pygame pixel (x, y) of the panel, as a saved
 *     PNG shows it.  This is transposed against the x-major observation arrays ([res_h][res_v][3]).
 * mode: MGB_GOD_LIVE (the current state; nothing needs recording) or MGB_GOD_TRAJECTORY (the picture of
 *   MazeBase.render_trajectory with additional=None, maze_base.py:159-189: white fill, walls and ESCAPE goal, a red agent
 *   rect at the current cell for every kind, SURVIVAL food over it, then red width-3 lines between the centres of
 *   consecutive cells of the env's current-episode path; needs mgb_maze_set_path, else MGB_ERR_ARG).  Pixel rules:
 *   DESIGN.md "God view".  Stream-ordered, no host synchronisation, no allocation: capturable in a CUDA graph. */
#define MGB_GOD_LIVE 0
#define MGB_GOD_TRAJECTORY 1
int mgb_maze_god_view(mgb_maze *h, int32_t count, const int32_t *envs_dev, int32_t view_size, int32_t mode,
                      uint8_t *out_dev, void *stream);

/* Path recording (MazeBase._agent_trajectory, maze_base.py:44,67), off by default; call after mgb_maze_create, like
 * mgb_maze_set_options.  enabled = 1 allocates [max_steps + 1][n_envs] int8 cell pairs, step-major; every kernel that
 * leaves env e with step count s then stores the agent's cell as entry (s, e), so the current episode's path is entries
 * 0 .. min(s, max_steps).  Steps past max_steps (auto_reset off, stepping on after done) are not stored.  Switching it on
 * mid-episode records the current cell; earlier entries read (-1, -1).  Observations, rewards, dones and state are
 * bit-identical with recording on and off.  Synchronous; enabled = 0 frees the buffer.
 *   mgb_maze_path: cells_out [count][max_steps + 1][2] int8 (entries at and past len_out[k] are not written) and len_out
 *   [count] int32 of envs envs_dev (as for mgb_maze_god_view; an index outside [0, n_envs) has length 0).  Stream-ordered,
 *   no host synchronisation. */
int mgb_maze_set_path(mgb_maze *h, int enabled);
int mgb_maze_path(mgb_maze *h, int32_t count, const int32_t *envs_dev, int8_t *cells_out, int32_t *len_out, void *stream);

/* Exact snapshot / restore of env state, as mgb_quad_snapshot / mgb_quad_restore (same row map and stream rules).  A
 * record of mgb_maze_record_bytes(h) bytes (after mgb_maze_set_task) holds agent (int4), life, the env's resample count,
 * its task-table slot, the continuous pose, the food stamps of every food slot and -- when the handle owns one table
 * slot per env and can re-task envs on the device (injective env2task, direct renderer) -- the whole task of the env's
 * slot.  Restore then writes that task into the destination env's own slot; otherwise the table is shared, the fingerprint
 * covers it, and restore points env2task[e] at the record's slot.  mgb_maze_restore is synchronous the first time it
 * finds the pose cache to be built (like the first reset); after that it is stream-ordered.  A recording handle
 * (mgb_maze_set_path) appends the env's path entries to its records (2 (max_steps + 1) bytes, padded to 16).  A trial
 * handle (mgb_maze_set_episodes_per_task) has one more 16-byte block after the food stamps: its episode count (u32) and
 * zero padding; the task and the path entries follow it.
 *   mgb_maze_fingerprint: out[0] config (mgb_maze_cfg, auto_reset, table shape, path recording, episodes per task,
 *     record layout), out[1] textures,
 *     out[2] the shared task table (0 when records carry their tasks), out[3] 1 when records carry their tasks. */
int64_t mgb_maze_record_bytes(const mgb_maze *h);
int mgb_maze_snapshot(mgb_maze *h, uint8_t *rec_dev, void *stream);
int mgb_maze_restore(mgb_maze *h, const uint8_t *rec_dev, int64_t n_rec, const int64_t *row_of_env_dev, void *stream);
int mgb_maze_counters(mgb_maze *h, uint64_t *t_base, int set);
int mgb_maze_fingerprint(const mgb_maze *h, uint64_t *out);

/* ------------------------------------------------------------------------------------------------------------ */
const char *mgb_last_error(void);
const char *mgb_version(void);
/* Number of CUDA devices visible, or <0 when the runtime cannot initialise (no fallback exists). */
int mgb_device_count(void);

/* ---- peer memory: the rollout kernels as their own all-gather (NVLink stores, no NCCL on the data) -----------------
 * Replaces the `comm.allgather(trajectories)` a distributed learner would do around N copies of the reference's
 * env.step loop (SURVEY.md 8e).  One receive arena per rank, allocated with mgb_peer_alloc, exported as a 64-byte
 * cudaIpcMemHandle, opened by every other rank of the node; mgb_*_set_mirrors then makes the fused rollout kernels
 * store each output at `ptr` and at `ptr + byte_delta[i]`, i < count <= MGB_MAX_MIRRORS. */
#define MGB_MAX_MIRRORS 7
#define MGB_PEER_HANDLE_BYTES 64
int mgb_peer_alloc(int device, uint64_t bytes, void **ptr_out);
int mgb_peer_free(int device, void *ptr);
int mgb_peer_export(int device, void *ptr, uint8_t handle_out[MGB_PEER_HANDLE_BYTES]);
int mgb_peer_open(int device, const uint8_t handle[MGB_PEER_HANDLE_BYTES], void **ptr_out);
int mgb_peer_close(int device, void *ptr);
int mgb_quad_set_mirrors(mgb_quad *h, int count, const int64_t *byte_delta);
int mgb_maze_set_mirrors(mgb_maze *h, int count, const int64_t *byte_delta);
/* Guard: while mirrors (or multicast) are on, a rollout whose obs/rew/done/act_out pointers are not all inside
 * [base, base + bytes) -- this rank's slot of the arena the deltas were computed for -- is refused with MGB_ERR_ARG
 * instead of storing to `pointer + delta` somewhere else.  bytes = 0 removes the guard. */
int mgb_quad_set_mirror_window(mgb_quad *h, const void *base, uint64_t bytes);
int mgb_maze_set_mirror_window(mgb_maze *h, const void *base, uint64_t bytes);
/* NVSwitch multicast variant: the rollout outputs are stored ONLY at `ptr + byte_delta` with multimem.st, where
 * byte_delta = (multicast mapping base - local arena base) of a multicast object every rank has bound its arena to
 * (cuMulticast*; torch.distributed._symmetric_memory does that plumbing).  The switch replicates each store into every
 * rank's arena, this rank's included.  0 switches it off.  Needs num_envs % 4 == 0. */
int mgb_quad_set_multicast(mgb_quad *h, int64_t byte_delta);
int mgb_maze_set_multicast(mgb_maze *h, int64_t byte_delta);

#ifdef __cplusplus
}
#endif
#endif /* MGB200_H */
