// MetaMaze hot path for sm_90a: 2-D grid step (one thread = one env) and discrete-3D step + first-person raycast
// render (one persistent CTA per SM, textures staged ONCE into shared memory by TMA bulk copy, every env's maze tile
// staged by TMA + mbarrier, pixels leave through double-buffered shared-memory chunks and TMA bulk stores).
//
// Replaces (reference file:line, PaddlePaddle/MetaGym):
//   MazeBase.set_task / reset / evaluation_rule      metagym/metamaze/envs/maze_base.py:19-95, 191-202
//   MazeCore2D.do_action / update_observation        metagym/metamaze/envs/maze_2d.py:21-34, 89-121
//   MazeCoreDiscrete3D.turn / move / do_action / update_observation
//                                                    metagym/metamaze/envs/maze_discrete_3d.py:39-81, 113-127
//   DDA_2D / maze_view                               metagym/metamaze/envs/ray_caster_utils.py:11-62, 66-209
//
// Exactness: grid state, done flags, float64 rewards/life and the rendered integers are bit-identical to the reference.
// The renderer therefore computes pixel geometry in float64 with the reference's operation order, float32 column
// tables, truncating float->int conversions and NO fused multiply-add (this file is compiled with -fmad=false).
// Food respawn is evaluated lazily from per-food "eaten at step s" stamps (SURVEY.md 8a): a cell eaten at step s is
// edible again at the check of step t iff t > s + interval and visible after step t iff t >= s + interval, which is
// what maze_base.py:74-75,83-88 does with its whole-grid countdown arrays.
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <memory>
#include <new>
#include <type_traits>
#include <utility>
#include <vector>

#include "mgb_common.cuh"
#include "mgb_policy.cuh"

namespace {

constexpr int kMaxN = 31;
constexpr int kNever = INT_MIN / 2;
constexpr int kRenderThreads = 512;
constexpr int kGeoThreads = 128;            // direct renderer, pipelined: threads that prepare the next env's records
constexpr int kMaxHitsCap = 2 * kMaxN - 1;   // a ray enters at most 2 n - 1 cells of an n x n grid

// shared-memory workspace of one warp of the task sampler (maze_sample_task): per cell a 32-bit value draw, a 16-bit order
// entry and a wall/food byte, then one union-find byte per room; rounded up to 16
__host__ __device__ constexpr int sampler_ws_bytes(int n) { return (7 * n * n + ((n - 1) / 2) * ((n - 1) / 2) + 15) / 16 * 16; }
constexpr int kSamplerWsMax = sampler_ws_bytes(kMaxN);

struct TaskHdr {                 // 104 bytes, head of every task blob
    int32_t start[2], goal[2];
    double cell_size, wall_height, agent_height, initial_life, max_life, step_reward, goal_reward;
    int32_t n_food;
    int32_t cls;                 // index of the (agent_height, wall_height) class -> pose-independent eff table
    // x / d == x * (1/d) exactly when d is a power of two: the renderer's divisions by cell_size (2.0) and
    // text_size / cell_size (0.5) then cost one multiply instead of a ~40-instruction IEEE division.
    double inv_cell, inv_t2c;
    int32_t cell_pow2, t2c_pow2;
};

struct MazeConst {
    int kind, task_type, n, max_steps, view_grid, res_h, res_v, obs_dtype;
    int n_tex, ts;
    int f_max;                   // food slots per env
    int max_hits;                // transparent crossings kept per column
    int run_px;                  // pixels per warp run (768 B of output): one bulk store per run
    int text_pow2;               // text_size is a power of two
    double inv_text;
    int n_cls;                   // height classes with a precomputed eff table (0 = compute per pixel)
    int pipe;                    // direct renderer: two record sets, geometry of env e + 1 under the pixels of env e
    int hits_in_global;          // large screens: the per-column crossing lists live in a global scratch, not smem
    int blob_bytes;              // bytes of one task blob (multiple of 16)
    int off_walls, off_texts, off_fidx, off_fval, off_fint;   // offsets inside a blob
    double max_vision, l_focal, text_size;
    double half_h, half_v, pixel_size;                        // host-computed like ray_caster_utils.py:68-70
    // life bar (maze_discrete_3d.py:42-45)
    double lb_sx, lb_sy, lb_w, lb_l;
};

struct SamplerCfg {          // mgb_maze_sampler_cfg + derived fields (sampler_cfg)
    int allow_loops, n_texts, food_interval, cls;
    double cell_size, wall_height, agent_height, step_reward, goal_reward, food_reward, initial_life, max_life, food_density,
        crowd_ratio;
};

struct MazeArgs {
    int64_t n, n_pad, env_base;
    int4 *agent;                 // gx, gy, ori, steps
    double *life;
    int32_t *eaten;              // [f_max][n_pad]
    const int32_t *env2task;
    const uint8_t *blobs;        // [n_tasks][blob_bytes]
    const uint32_t *tex;         // packed 0x00BBGGRR, (n_tex + 1) * ts * ts, ceiling last
    const float *coltab;         // [4][3][res_h]: cos_hp, cos_abs, sin_abs per heading
    const double *efftab;        // [n_cls][res_h * res_v]: distance(d_v) / cos_hp(d_h), pose independent
    const double *fogtab;        // [n_cls][res_h * res_v]: alpha = clip(2 eff / max_vision - 1, 0, 1) of that distance
    // pose cache (memoised static layers, see maze3d_compose_kernel)
    const int4 *poses;           // FILL: [n_slots] task, gx, gy, ori
    const int32_t *pose_index;   // [n_tasks][n*n*4] -> slot or -1
    const void *pose_rec;        // [n_tasks][n*n*4] PoseRec (pose_index + c_fmask + c_vbase merged), nullptr: use the three tables
    uint32_t *c_px;              // [n_slots][H*V]   10-bit R | G<<10 | B<<20 | in_wall<<30
    uint8_t *c_fid;              // [n_slots][H*V]   food slot of the floor/ceiling cell under the pixel, 0xFF none
    uint8_t *c_rgb8;             // [n_slots][H*V*3] finished uint8 pixel with EVERY food of the task present (baked)
    uint32_t *c_px_all;          // int32 mode: [n_slots][H*V] packed like c_px, every food present (baked)
    uint64_t *c_fmask;           // [n_slots][2] food slots that can change this pose's image at all
    // variant frames (uint8 SURVIVAL): a pose whose image depends on k <= kVariantBits foods has all 2^k finished frames
    // baked, so a step never recomputes a pixel -- it picks the frame of the foods currently visible
    const int32_t *c_vbase;      // [n_slots] index of the pose's first extra frame in c_var8, or -1 (all-present frame only)
    uint8_t *c_var8;             // [n_tasks * V][H*V*3]; variant v of a pose = frame c_vbase + v, v = the visible foods'
                                 // bits compacted in ascending slot order; the all-visible variant is c_rgb8[slot] itself
    const void *bake_desc;       // bake mode over variant frames: [n_items] BakeDesc (slot, presence mask)
    int bake;                    // compose kernel: items are pose slots, output goes to c_rgb8 / c_px_all
    uint8_t *c_gsig;             // [n_slots][H*V/4] per 4-pixel group: signature of the foods that can tint it
    uint8_t *c_colhits;          // [n_slots][H]     transparent crossings recorded for the column
    void *c_hits;                // [n_slots][H][max_hits] HitRec
    void *dyn;                   // [n] EnvDyn, written by the logic kernel, read by the compose kernel
    void *hit_scratch;           // [grid][H][max_hits] HitRec when c.hits_in_global
    const int32_t *act;
    const float *act_c;          // continuous maze: [n][2] (turn_rate, walk_speed)
    float2 *cpos;                // continuous maze: position (float32, dynamics.py:75)
    double *cori;                // continuous maze: heading (python float)
    const double *coltab_d;      // [2][res_h]: cos_hp, sin_hp in float64 (heading independent)
    void *obs;
    double *rew;
    uint8_t *done;
    const uint8_t *mask;
    int do_step;                 // 0: observe only (reset), 1: step then observe
    int do_parts;                // compose kernel: image slices per env
    int T;                       // maze2d rollout: steps per launch
    uint64_t act_seed;
    uint32_t t_base;
    int32_t *act_out;
    MgbMirrors mir;              // maze2d rollout: every output is also stored at ptr + mir.delta[i]
    int auto_reset;
    float *act_out_c;            // continuous-maze rollout: drawn actions [T][n][2] (last, so the other kernels' parameter
                                 // offsets do not move)
    // terminal observations of auto-reset steps (mgb_maze_step).  The step logic of a finished env appends its terminal
    // state to a compact list before env_reset; a second pass renders the list into final_obs[fin_env[i]].
    uint8_t *truncated;          // [n] 1: done only through the step limit; nullptr: not produced
    void *final_obs;             // 2-D: [n][2g+1][2g+1] float32, written by the step kernel itself; 3-D: set on the list pass
    int32_t *fin_count;          // [1] list length (zeroed before the step); nullptr: no list
    int32_t *fin_env;            // [n] env of list entry i
    void *fin_dyn;               // pose cache: [n] EnvDyn of the terminal state
    int4 *fin_agent;             // direct renderer: terminal gx, gy, ori, steps ...
    double *fin_life;            // ... life
    int32_t *fin_eaten;          // ... food stamps [f_max][n_pad]
    int32_t *fin_task;           // ... task slot
    float2 *fin_cpos;            // ... continuous position
    double *fin_cori;            // ... continuous heading
    // path recording (mgb_maze_set_path): [max_steps + 1][n_pad] grid cells, step-major.  Whenever a kernel leaves env e
    // with step count s, entry (s, e) holds the agent's cell; nullptr: recording off, nothing is stored
    char2 *path;
    // pose-cache build of a region of the task table (ensure_pose_cache: every task; mgb_maze_update_tasks: the replaced
    // ones).  Task slot t owns the pose slots [t S, t S + S) and the variant frames [t V, t V + V); a region kernel's item i
    // is entry i % region_ext of task region[i / region_ext] (region_ext = S or V), the FILL pass renders the pose slots
    // fill_slot[0 .. n).  Unused pose slots have poses[slot].x = -1; a task's frames past task_frames[t] are unused.
    const int32_t *region;       // [K] task slots
    const int32_t *fill_slot;    // [n] pose slots of the region's tasks
    const int32_t *task_frames;  // [n_tasks] variant frames planned for each task
    int region_ext;
    int pose_stride, var_stride; // S, V
    int var_bits;                // variant bits of the table: a task takes the largest bits <= var_bits whose frames fit V
};

// in-launch task resampling (maze3d_kernel<.., RS> and maze2d_rollout_kernel<0, .., RS>, mgb_maze_rollout with a
// sampler cfg): an env whose episode ends gets the task mgb_maze_resample_tasks would draw for it.  A
// parameter of those kernels after MazeArgs, so that no other parameter offsets move.  Trial handles
// (mgb_maze_set_episodes_per_task) also pass `count`: an env then draws only when it finishes its k-th episode on its
// maze (rs_draws); with count null every finished env draws.
struct MazeResample {
    SamplerCfg cfg;
    uint64_t seed;
    uint32_t *epoch;             // [n] resample count of every env
    uint32_t *count;             // [n] episodes each env has finished on its current maze, or null
    int32_t k;                   // episodes per maze (count set)
};

// A finished env's trial bookkeeping: its count goes up by one, and it draws a new maze (count back to 0) at the k-th
__device__ __forceinline__ bool rs_draws(const MazeResample &rs, uint32_t &cnt)
{
    if (!rs.count) return true;
    cnt += 1;
    const bool draw = cnt >= (uint32_t)rs.k;
    if (draw) cnt = 0;
    return draw;
}

__device__ __noinline__ void maze_sample_task(const MazeConst &c, const SamplerCfg &sc, uint64_t seed, int64_t genv,
                                              uint32_t *epoch, uint8_t *ws, uint8_t *b);

struct Env {
    int gx, gy, ori, steps;
    double life;
};

__device__ __forceinline__ const TaskHdr *blob_hdr(const uint8_t *b) { return reinterpret_cast<const TaskHdr *>(b); }

__device__ __forceinline__ void maze_evaluate(const MazeConst &c, const uint8_t *blob, int32_t *eaten, int64_t estride,
                                              Env &e, double &reward, int &done);

// action + evaluation_rule for one env (single thread).  `eaten` is strided by `estride` (SoA in HBM).
__device__ __forceinline__ void maze_logic(const MazeConst &c, const uint8_t *blob, int32_t *eaten, int64_t estride,
                                           Env &e, int action, double &reward, int &done)
{
    const TaskHdr *th = blob_hdr(blob);
    const int8_t *walls = reinterpret_cast<const int8_t *>(blob + c.off_walls);
    const int n = c.n;
    action &= 3;
    if (c.kind == MGB_MAZE_2D) {                                  // maze_2d.py:21-34 with DISCRETE_ACTIONS (dx, dy)
        int tx = e.gx + (action == 0 ? -1 : (action == 1 ? 1 : 0));
        int ty = e.gy + (action == 2 ? -1 : (action == 3 ? 1 : 0));
        if (tx < 0) tx += n;                                      // numpy negative index; unreachable (border walls)
        if (ty < 0) ty += n;
        if (tx < n && ty < n && walls[tx * n + ty] < 1) { e.gx = tx; e.gy = ty; }
    } else {                                                      // maze_discrete_3d.py:51-81, (turn, move)
        const int turn = action == 0 ? -1 : (action == 1 ? 1 : 0);
        const int mv = action == 2 ? -1 : (action == 3 ? 1 : 0);
        e.ori = (e.ori + turn + 4) & 3;
        int tx = e.gx, ty = e.gy;
        if (e.ori == 0) tx += mv; else if (e.ori == 1) ty += mv; else if (e.ori == 2) tx -= mv; else ty -= mv;
        if (tx >= 0 && tx < n && ty >= 0 && ty < n && walls[tx * n + ty] == 0) { e.gx = tx; e.gy = ty; }
    }
    maze_evaluate(c, blob, eaten, estride, e, reward, done);
}

// MazeBase.evaluation_rule (maze_base.py:65-95) on the agent's current cell
__device__ __forceinline__ void maze_evaluate(const MazeConst &c, const uint8_t *blob, int32_t *eaten, int64_t estride,
                                              Env &e, double &reward, int &done)
{
    const TaskHdr *th = blob_hdr(blob);
    const int n = c.n;
    e.steps += 1;                                                 // maze_base.py:66
    const bool over = e.steps > c.max_steps - 1;                  // :191-192
    if (c.task_type == MGB_MAZE_SURVIVAL) {
        double r = 0.0;
        const int8_t *fidx = reinterpret_cast<const int8_t *>(blob + c.off_fidx);
        const int f = fidx[e.gx * n + e.gy];
        if (f >= 0) {
            const double val = reinterpret_cast<const double *>(blob + c.off_fval)[f];
            const int itv = reinterpret_cast<const int32_t *>(blob + c.off_fint)[f];
            const int ea = eaten[f * estride];
            const bool present = (ea == kNever) || (e.steps > ea + itv);
            if (present && val > 1.0e-2) {                        // :71-75
                r = val;
                eaten[f * estride] = e.steps;
            }
        }
        e.life = e.life + (r + th->step_reward);                  // :78
        e.life = e.life < th->max_life ? e.life : th->max_life;   // :79
        done = (e.life < 0.0) || over;                            // :80
        reward = r;
    } else {
        const int goal = (e.gx == th->goal[0] && e.gy == th->goal[1]);
        reward = th->step_reward + (double)goal * th->goal_reward;   // :91-92
        done = goal || over;
    }
}

__device__ __forceinline__ void env_reset(const MazeConst &c, const uint8_t *blob, int32_t *eaten, int64_t estride,
                                          Env &e)
{
    const TaskHdr *th = blob_hdr(blob);
    e.gx = th->start[0]; e.gy = th->start[1]; e.ori = 0; e.steps = 0;
    e.life = th->initial_life;
    for (int f = 0; f < c.f_max; ++f) eaten[f * estride] = kNever;
}

// the episode that just ended (done) ended only through the step limit: SURVIVAL alive, ESCAPE off the goal (maze_base.py:80,
// 91-95, 191-192).  Evaluated on the state evaluation_rule left, before any reset.
__device__ __forceinline__ uint8_t maze_truncated(const MazeConst &c, const uint8_t *blob, const Env &e)
{
    const TaskHdr *th = blob_hdr(blob);
    const bool over = e.steps > c.max_steps - 1;
    const bool terminal = c.task_type == MGB_MAZE_SURVIVAL ? e.life < 0.0 : (e.gx == th->goal[0] && e.gy == th->goal[1]);
    return (uint8_t)(over && !terminal);
}

// _agent_trajectory (maze_base.py:44,67): the agent's cell becomes entry (steps, e) of the path record.  The entry index is
// the step count the env carries, so an episode's path is entries 0 .. steps; steps past the capacity (an env without
// auto-reset stepped on after done) are not stored.
__device__ __forceinline__ void path_store(const MazeConst &c, const MazeArgs &a, int64_t e, const Env &s)
{
    if (a.path && s.steps <= c.max_steps) a.path[(int64_t)s.steps * a.n_pad + e] = make_char2((char)s.gx, (char)s.gy);
}

// current transparent value of cell (i, j): SURVIVAL = remaining food (alias at maze_base.py:57), ESCAPE = goal one-hot
__device__ __forceinline__ double food_now(const MazeConst &c, const uint8_t *blob, const int32_t *eaten,
                                           int64_t estride, int steps, int cell)
{
    const int8_t *fidx = reinterpret_cast<const int8_t *>(blob + c.off_fidx);
    const int f = fidx[cell];
    if (f < 0) return 0.0;
    const int itv = reinterpret_cast<const int32_t *>(blob + c.off_fint)[f];
    const int ea = eaten[f * estride];
    const bool visible = (ea == kNever) || (steps >= ea + itv);
    return visible ? reinterpret_cast<const double *>(blob + c.off_fval)[f] : 0.0;
}

// ---------------------------------------------------------------------------------------------------------------
// ESCAPE expert (include/mgb200.h "Expert", DESIGN.md §4d): per task slot, the fewest actions to the goal from every
// state and the set of actions that realise it, by breadth-first search backwards from the goal over the step's own move
// rules.  A state is s = (ori n + gx) n + gy (MetaMaze2D: ori = 0, one plane).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kExpertWarps = 2;
constexpr int kExpertStates = 4 * kMaxN * kMaxN;
constexpr uint16_t kExpertFar = 0xFFFF;      // the goal cannot be reached

__host__ __device__ constexpr int expert_planes(int kind) { return kind == MGB_MAZE_2D ? 1 : 4; }

// The state action `action` leads to from s: the move of maze_logic, restated on a state index
__device__ __forceinline__ int expert_next(const MazeConst &c, const int8_t *walls, int s, int action)
{
    const int n = c.n, nn = n * n;
    int ori = s / nn, gx = (s - ori * nn) / n, gy = s - ori * nn - gx * n;
    if (c.kind == MGB_MAZE_2D) {
        int tx = gx + (action == 0 ? -1 : (action == 1 ? 1 : 0));
        int ty = gy + (action == 2 ? -1 : (action == 3 ? 1 : 0));
        if (tx < 0) tx += n;
        if (ty < 0) ty += n;
        if (tx < n && ty < n && walls[tx * n + ty] < 1) { gx = tx; gy = ty; }
    } else {
        const int turn = action == 0 ? -1 : (action == 1 ? 1 : 0);
        const int mv = action == 2 ? -1 : (action == 3 ? 1 : 0);
        ori = (ori + turn + 4) & 3;
        int tx = gx, ty = gy;
        if (ori == 0) tx += mv; else if (ori == 1) ty += mv; else if (ori == 2) tx -= mv; else ty -= mv;
        if (tx >= 0 && tx < n && ty >= 0 && ty < n && walls[tx * n + ty] == 0) { gx = tx; gy = ty; }
    }
    return (ori * n + gx) * n + gy;
}

// The states from which `action` may lead to t, or -1: `which` 0 is the state that stays (3-D: the turned heading on
// t's cell), 1 the state that moved into t.  A superset: the caller keeps a candidate only if expert_next maps it to t.
__device__ __forceinline__ int expert_pred(const MazeConst &c, int t, int action, int which)
{
    const int n = c.n, nn = n * n;
    const int ot = t / nn, x = (t - ot * nn) / n, y = t - ot * nn - x * n;
    if (c.kind == MGB_MAZE_2D) {       // staying in place reaches t from t itself, which the search has already visited
        if (which == 0) return -1;
        const int dx = action == 0 ? -1 : (action == 1 ? 1 : 0), dy = action == 2 ? -1 : (action == 3 ? 1 : 0);
        return ((x - dx + n) % n) * n + (y - dy + n) % n;     // the wrap of a negative index (maze_logic) included
    }
    const int turn = action == 0 ? -1 : (action == 1 ? 1 : 0);
    const int mv = action == 2 ? -1 : (action == 3 ? 1 : 0);
    const int o = (ot - turn + 4) & 3;
    if (which == 0) return (o * n + x) * n + y;
    if (mv == 0) return -1;
    const int sx = x - mv * (ot == 0 ? 1 : (ot == 2 ? -1 : 0)), sy = y - mv * (ot == 1 ? 1 : (ot == 3 ? -1 : 0));
    return sx >= 0 && sx < n && sy >= 0 && sy < n ? (o * n + sx) * n + sy : -1;
}

// One warp per item: the tables of task slot map[i] (map null: slot i), for the items with sel[i] set (sel null: all)
// whose record row[i] lies in [0, n_rec) (row null: all).  Breadth-first from the goal's states with the queue, the
// distance plane and the walls in shared memory: each state enters the queue once, when a lane claims it (16-bit
// compare-and-swap) as a verified predecessor of a state of the level before.
__global__ void __launch_bounds__(32 * kExpertWarps) maze_expert_kernel(const __grid_constant__ MazeConst c,
                                                                        const uint8_t *blobs, int64_t count,
                                                                        const int32_t *map, const uint8_t *sel,
                                                                        const int64_t *row, int64_t n_rec,
                                                                        uint16_t *dist, uint8_t *mask)
{
    __shared__ uint16_t s_dist[kExpertWarps][kExpertStates];
    __shared__ uint16_t s_queue[kExpertWarps][kExpertStates];
    __shared__ int8_t s_walls[kExpertWarps][kMaxN * kMaxN];
    __shared__ int s_tail[kExpertWarps];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * kExpertWarps + w;
    if (i >= count) return;                                        // warp-uniform exits
    if (sel && !sel[i]) return;
    if (row && (row[i] < 0 || row[i] >= n_rec)) return;
    const int64_t slot = map ? map[i] : i;
    const uint8_t *blob = blobs + slot * c.blob_bytes;
    const int n = c.n, nn = n * n, P = expert_planes(c.kind), S = P * nn;
    const int goal = blob_hdr(blob)->goal[0] * n + blob_hdr(blob)->goal[1];
    uint16_t *d = s_dist[w], *q = s_queue[w];
    int8_t *walls = s_walls[w];
    for (int k = lane; k < nn; k += 32) walls[k] = reinterpret_cast<const int8_t *>(blob + c.off_walls)[k];
    for (int k = lane; k < S; k += 32) d[k] = k % nn == goal ? 0 : kExpertFar;
    if (lane < P) q[lane] = (uint16_t)(lane * nn + goal);
    if (lane == 0) s_tail[w] = P;
    __syncwarp();
    for (int lo = 0, hi = P; lo < hi;) {
        for (int k = lo + lane; k < hi; k += 32) {
            const int t = q[k];
            const uint16_t nd = (uint16_t)(d[t] + 1);
            for (int act = 0; act < 4; ++act)
                for (int which = 0; which < 2; ++which) {
                    const int sp = expert_pred(c, t, act, which);
                    if (sp < 0 || d[sp] != kExpertFar || expert_next(c, walls, sp, act) != t) continue;
                    if (atomicCAS(reinterpret_cast<unsigned short *>(d + sp), kExpertFar, nd) == kExpertFar)
                        q[atomicAdd(&s_tail[w], 1)] = (uint16_t)sp;
                }
        }
        __syncwarp();
        lo = hi;
        hi = *reinterpret_cast<volatile int *>(&s_tail[w]);
        __syncwarp();                                              // every lane has read the level's end
    }
    for (int k = lane; k < S; k += 32) {
        const uint16_t dk = d[k];
        uint8_t m = 0;
        if (dk != 0 && dk != kExpertFar)
            for (int act = 0; act < 4; ++act) m |= (uint8_t)(d[expert_next(c, walls, k, act)] == dk - 1) << act;
        dist[slot * S + k] = dk;
        mask[slot * S + k] = m;
    }
}

// What an expert rollout (the EXP instantiations) reads and writes besides MazeArgs: a parameter after the others, empty
// in every other instantiation, so that no existing parameter offset moves
struct MazeExpert {
    const uint8_t *mask;         // [slots][planes][n][n]
    uint8_t *out;                // [T][n]: the mask of the state acted on, or null
    float eps;                   // mixing rate
    int mean;                    // 1: the lowest action of the choice set, no draw
    uint64_t seed;
};
struct MazeNoExpert {};
template <bool EXP>
using MazeExpertOr = std::conditional_t<EXP, MazeExpert, MazeNoExpert>;

// the entry of an env in state s on task slot `slot`
__device__ __forceinline__ int64_t expert_index(const MazeConst &c, int64_t slot, const Env &s)
{
    const int P = expert_planes(c.kind);
    return ((slot * P + (P == 4 ? s.ori : 0)) * c.n + s.gx) * c.n + s.gy;
}

__device__ __forceinline__ uint8_t expert_mask(const MazeConst &c, const uint8_t *mask, int64_t slot, const Env &s)
{
    return mask[expert_index(c, slot, s)];
}

// the tables' entries of every env's current state (mgb_maze_expert, mgb_maze_step_expert)
__global__ void maze_expert_state_kernel(const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a,
                                         const uint8_t *mask, const uint16_t *dist, uint8_t *mask_out, uint16_t *dist_out)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const int4 ag = a.agent[e];
    const Env s = {ag.x, ag.y, ag.z, ag.w, 0.0};
    const int64_t k = expert_index(c, a.env2task[e], s);
    mask_out[e] = mask[k];
    if (dist_out) dist_out[e] = dist[k];
}

// The expert's action on a state with mask m (include/mgb200.h): the choice set is {0..3} when r.x's 24-bit uniform is
// below eps or m is empty, else m; the action is set bit number floor(r.y k / 2^32) of the k in the choice set, or its
// lowest bit in mean mode
__device__ __forceinline__ int expert_action(const MazeExpert &x, uint8_t m, int64_t genv, uint32_t t)
{
    uint32_t set = m ? m : 0xFu, j = 0;
    if (!x.mean) {
        const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32), t, MGB_STREAM_EXPERT),
                                          make_uint2((uint32_t)x.seed, (uint32_t)(x.seed >> 32)));
        if (mgb_u01(r.x) < x.eps) set = 0xFu;
        j = (uint32_t)(((uint64_t)r.y * (uint32_t)__popc(set)) >> 32);
    }
    for (; j; --j) set &= set - 1;
    return __ffs(set) - 1;
}


// ---------------------------------------------------------------------------------------------------------------
// MetaMazeContinuous3D dynamics (dynamics.py:16-92), float32/float64 typing of the numba + numpy original for float32
// actions: see oracle/maze_oracle.c (mo_vector_move_with_collision) for the line-by-line restatement this mirrors.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float sum2f(float a, float b) { float c = 0.0f; c += a; c += b; return c; }

__device__ float nearest_point_dev(const float pos[2], float l1x, float l1y, float l2x, float l2y, float np_out[2])
{
    float ux = l2x - l1x, uy = l2y - l1y;
    const float edge_norm = sqrtf(sum2f(ux * ux, uy * uy));
    const double den = 1.0e-6 > (double)edge_norm ? 1.0e-6 : (double)edge_norm;
    ux = (float)((double)ux / den); uy = (float)((double)uy / den);
    const float dist_1 = sum2f((pos[0] - l1x) * ux, (pos[1] - l1y) * uy);
    float qx, qy;
    if (dist_1 > edge_norm) { qx = l2x; qy = l2y; }
    else if (dist_1 < 0) { qx = l1x; qy = l1y; }
    else { qx = l1x + dist_1 * ux; qy = l1y + dist_1 * uy; }
    const float a = pos[0] - qx, b = pos[1] - qy;
    np_out[0] = qx; np_out[1] = qy;
    return sqrtf(sum2f(a * a, b * b));
}

__device__ void collision_force_dev(const float dv[2], double cell_size, double col_dist, float out[2])
{
    double dist = (double)sqrtf(sum2f(dv[0] * dv[0], dv[1] * dv[1]));
    const double eff = col_dist / cell_size;
    out[0] = out[1] = 0.0f;
    if (dist > 0.708 + eff) return;
    if (fabsf(dv[0]) < 0.5f && fabsf(dv[1]) < 0.5f) {
        const float k = (float)(0.50 / (dist > 1.0e-6 ? dist : 1.0e-6) * (0.708 + eff - dist) * cell_size);
        out[0] = k * dv[0]; out[1] = k * dv[1];
        return;
    }
    const bool x_pos = (dv[0] + dv[1] > 0), y_pos = (dv[1] - dv[0] > 0);
    float np[2];
    if (x_pos && y_pos) dist = (double)nearest_point_dev(dv, 0.5f, 0.5f, -0.5f, 0.5f, np);
    else if (!x_pos && y_pos) dist = (double)nearest_point_dev(dv, -0.5f, 0.5f, -0.5f, -0.5f, np);
    else if (!x_pos && !y_pos) dist = (double)nearest_point_dev(dv, -0.5f, -0.5f, 0.5f, -0.5f, np);
    else dist = (double)nearest_point_dev(dv, 0.5f, -0.5f, 0.5f, 0.5f, np);
    if (eff < dist) return;
    float ox = dv[0] - np[0], oy = dv[1] - np[1];
    const float on = sqrtf(sum2f(ox * ox, oy * oy));
    const double inv = 1.0 / (1.0e-6 > (double)on ? 1.0e-6 : (double)on);
    ox = (float)((double)ox * inv); oy = (float)((double)oy * inv);
    const float k = (float)(0.50 * (eff - dist) * cell_size);
    out[0] = k * ox; out[1] = k * oy;
}

// do_action (maze_continuous_3d.py:47-53): clip, scale, ten sub-steps of vector_move + collision forces
__device__ void continuous_move(const MazeConst &c, const uint8_t *blob, float tr, float ws, float pos[2], double &ori_io)
{
    const TaskHdr *th = blob_hdr(blob);
    const int8_t *walls = reinterpret_cast<const int8_t *>(blob + c.off_walls);
    const int n = c.n;
    const double cell_size = th->cell_size;
    float turn = tr < -1.0f ? -1.0f : (tr > 1.0f ? 1.0f : tr);
    turn = turn * (float)3.1415926;
    float walk = ws < -1.0f ? -1.0f : (ws > 1.0f ? 1.0f : ws);
    if (walk < 0) walk = walk * 0.5f;
    float tx = pos[0], ty = pos[1];
    double ori = ori_io;
    for (int it = 0; it < 10; ++it) {                       // int(100 * 0.10), dynamics.py:76
        double fin = ori + (double)turn * 0.01;
        const double off_ori = 0.5 * (fin + ori);
        const double off = (double)walk * 0.01;
        const float dx = (float)(cos(off_ori) * off), dy = (float)(sin(off_ori) * off);
        while (fin > 6.2831852) fin -= 6.2831852;
        while (fin < 0) fin += 6.2831852;
        ori = fin;
        const float ex = tx + dx, ey = ty + dy;
        const float cs = (float)cell_size;
        const float ecx = ex / cs, ecy = ey / cs;
        float cx = 0.0f, cy = 0.0f;
        for (int i = -1; i < 2; ++i)
            for (int j = -1; j < 2; ++j) {
                const int wi = i + (int)ecx, wj = j + (int)ecy;
                if (wi > -1 && wi < n && wj > -1 && wj < n && walls[wi * n + wj] > 0) {
                    const float dv[2] = {ecx - floorf(ecx) - (float)(i + 0.5), ecy - floorf(ecy) - (float)(j + 0.5)};
                    float f[2];
                    collision_force_dev(dv, cell_size, 0.20, f);   // collision_dist = 0.20, maze_continuous_3d.py:20
                    cx += f[0]; cy += f[1];
                }
            }
        tx = cx + ex; ty = cy + ey;
    }
    pos[0] = tx; pos[1] = ty;
    ori_io = ori;
}

// ---------------------------------------------------------------------------------------------------------------
// state-only kernels
// ---------------------------------------------------------------------------------------------------------------
// Envs start a new episode: every env, or only those with a.mask[e] set, or (task_flags) only those whose task-table slot
// was just replaced (set_task leaves an env at its start state, maze_env.py:44-50).
__global__ void maze_reset_kernel(const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a,
                                  const uint8_t *task_flags)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    if (a.mask && !a.mask[e]) return;
    const int task = a.env2task[e];
    if (task_flags && !task_flags[task]) return;
    const uint8_t *blob = a.blobs + (int64_t)task * c.blob_bytes;
    Env s;
    env_reset(c, blob, a.eaten + e, a.n_pad, s);
    a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
    a.life[e] = s.life;
    path_store(c, a, e, s);
    if (c.kind == MGB_MAZE_CONTINUOUS_3D) {             // get_cell_center(start), heading 0 (maze_base.py:41,50)
        const TaskHdr *th = blob_hdr(blob);
        a.cpos[e] = make_float2((float)(s.gx * th->cell_size + 0.5 * th->cell_size),
                                (float)(s.gy * th->cell_size + 0.5 * th->cell_size));
        a.cori[e] = 0.0;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// 2-D: one thread per env; observation tile of the CTA leaves through shared memory + one bulk store
// ---------------------------------------------------------------------------------------------------------------
constexpr int k2dThreads = 128;
static_assert(k2dThreads == MGB_MAZE2D_POLICY_CTA_ENVS, "include/mgb200.h publishes the policy CTA's env count");

__global__ void __launch_bounds__(k2dThreads) maze2d_kernel(const __grid_constant__ MazeConst c,
                                                            const __grid_constant__ MazeArgs a)
{
    extern __shared__ __align__(128) float tile2d[];
    const int64_t e0 = (int64_t)blockIdx.x * k2dThreads;
    const int64_t e = e0 + threadIdx.x;
    const int W = 2 * c.view_grid + 1, D = W * W;
    const int rows = (int)((a.n - e0) < k2dThreads ? (a.n - e0) : k2dThreads);
    if (e < a.n) {
        const uint8_t *blob = a.blobs + (int64_t)a.env2task[e] * c.blob_bytes;
        const TaskHdr *th = blob_hdr(blob);
        const int4 ag = a.agent[e];
        Env s = {ag.x, ag.y, ag.z, ag.w, a.life[e]};
        int32_t *eaten = a.eaten + e;
        // update_observation, maze_2d.py:89-121
        auto observe = [&](float *row) {
            const int8_t *walls = reinterpret_cast<const int8_t *>(blob + c.off_walls);
            const int n = c.n, g = c.view_grid;
            for (int p = 0; p < W; ++p)
                for (int q = 0; q < W; ++q) {
                    const int x = s.gx - g + p, y = s.gy - g + q;
                    float v = -1.0f;
                    if (x >= 0 && x < n && y >= 0 && y < n) {
                        v = (float)(-(int)walls[x * n + y]);
                        if (c.task_type == MGB_MAZE_SURVIVAL)
                            v = (float)((double)v + food_now(c, blob, eaten, a.n_pad, s.steps, x * n + y));
                        else
                            v = (float)((double)v + ((x == th->goal[0] && y == th->goal[1]) ? 1.0 : 0.0));
                    }
                    row[p * W + q] = v;
                }
            if (c.task_type == MGB_MAZE_SURVIVAL) row[g * W + g] = (float)s.life;
        };
        if (a.do_step) {
            double reward;
            int done;
            maze_logic(c, blob, eaten, a.n_pad, s, a.act[e], reward, done);
            a.rew[e] = reward;
            a.done[e] = (uint8_t)done;
            if (a.truncated) a.truncated[e] = maze_truncated(c, blob, s);
            if (done && a.final_obs) observe(reinterpret_cast<float *>(a.final_obs) + e * D);   // the terminal window
            if (done && a.auto_reset) env_reset(c, blob, eaten, a.n_pad, s);
            a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
            a.life[e] = s.life;
            path_store(c, a, e, s);
        }
        observe(tile2d + threadIdx.x * D);
    }
    float *dst = reinterpret_cast<float *>(a.obs) + e0 * D;
    const uint32_t bytes = (uint32_t)rows * (uint32_t)D * 4u;
    if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
        mgb_fence_proxy_async();
        __syncthreads();
        if (threadIdx.x == 0) {
            mgb_bulk_store(dst, tile2d, bytes);
            mgb_bulk_commit();
            mgb_bulk_wait_read<0>();   // smem must outlive the copy; the kernel boundary flushes the writes
        }
    } else {
        __syncthreads();
        for (int i = threadIdx.x; i < rows * D; i += blockDim.x) dst[i] = tile2d[i];
    }
}


// update_observation (maze_2d.py:89-121) of one env into row: the terminal windows of maze2d_rollout_kernel<0, true>.  The
// rollout's observation tile writes the same loop out: routed through a shared helper, the instantiations without FIN
// were scheduled differently (same instructions, other order), and they are kept exactly as they were.
__device__ __forceinline__ void maze2d_window(const MazeConst &c, const uint8_t *blob, const int32_t *eaten,
                                              int64_t estride, const Env &s, float *row)
{
    const TaskHdr *th = blob_hdr(blob);
    const int8_t *walls = reinterpret_cast<const int8_t *>(blob + c.off_walls);
    const int n = c.n, g = c.view_grid, W = 2 * g + 1;
    for (int p = 0; p < W; ++p)
        for (int q = 0; q < W; ++q) {
            const int x = s.gx - g + p, y = s.gy - g + q;
            float v = -1.0f;
            if (x >= 0 && x < n && y >= 0 && y < n) {
                v = (float)(-(int)walls[x * n + y]);
                if (c.task_type == MGB_MAZE_SURVIVAL)
                    v = (float)((double)v + food_now(c, blob, eaten, estride, s.steps, x * n + y));
                else
                    v = (float)((double)v + ((x == th->goal[0] && y == th->goal[1]) ? 1.0 : 0.0));
            }
            row[p * W + q] = v;
        }
    if (c.task_type == MGB_MAZE_SURVIVAL) row[g * W + g] = (float)s.life;
}

// T MetaMaze2D steps in one launch: the agent (cell, step counter, life) stays in registers, food stamps stay in their
// SoA slots, each step's observation tile of the CTA leaves through double-buffered shared memory + one bulk store.
// XM: 0 plain, 1 peer mirrors, 2 multicast-only stores (see quad_rollout_kernel).  FIN (XM == 0 only, final_obs / truncated):
// also store the truncation byte of every (t, e), and the terminal window of every env that finished at step t to
// final_obs + (t n + e) D, both before env_reset; rows of envs that did not finish are not written.  REC: path recording on
// (a.path set); the instantiations without it have no store and no test of a.path in their loop.
// RS (XM == 0 only, a sampler cfg): an env that finishes at step t gets the task mgb_maze_resample_tasks would
// draw for it (after its reward, done, truncation byte and terminal window, all on the old task) and restarts on it, so
// obs[t] is its first window on the new maze.  The sampler is warp-collective: the done ballot is taken by all 32 lanes
// (the tail warp's lanes past n included), the warp draws one task per finished lane in lane order into that lane's table
// slot with its workspace behind the two tiles, and after a __syncwarp each owner resets on its new blob.  Each warp then
// publishes its own 32 rows of the tile with its own bulk store, so no step waits at a CTA barrier for another warp's
// carving.
// POL (XM == 0 only, mgb_maze_rollout_policy): the action of step t is drawn from the MLP policy `pol` (mgb_policy.cuh,
// categorical head) on the window the env holds before step t.  Each step copies the window row it leaves in the tile
// (post auto-reset and resampling) into the thread's column of the activation buffers, which follow the tiles and the
// sampler workspaces in dynamic shared memory at pol.smem_off, behind the staged weights; at t = 0 the window of the
// loaded state.  A population's CTA stages the one member that drives its envs, or its head.copies members back to back,
// each warp reading its own (mgb_population_stage).  The step arithmetic after the action is the code the other
// instantiations run.
// POL == kPolGru or kPolLstm (mgb_maze_rollout_rnn): the policy is the recurrent `pol` (MgbRnn, mgb_policy.cuh).  Its
// region at pol.smem_off holds the staged cell and head (of each staged member), then the columns x, c, h0, h1 and w.  The obs rows of x are
// filled as for the MLP; at t = 0 the state row fills h0, c and the feedback rows of x.  Step t computes h1 from
// (x, h0, c), updating c in place, and acts on head(h1), whose hidden layer goes to w (GRU) or the dead h0 (LSTM).
// After the step the carry swaps h0 and h1 and writes (onehot(a), (float)r) into the feedback rows, or zeroes h, c and
// the feedback where done and the reset rule fires; the state row is stored after step T - 1.
// VAL (POL and FIN only, mgb_maze_rollout_critic / mgb_maze_rollout_rnn_critic): the head's output layer has the value
// row.  Step t stores V(s_t).  Where the cut (the carry's wipe) fires on a truncated step, the terminal window goes into
// the x column and the policy runs once more on it, before the wipe (the recurrent cell from h_t and c'_t with the
// step's feedback, writing into the dead h0 column; the LSTM's head then uses the dead h1): that is final_value.  The task rule's cut is stored in adv for the epilogue.  After the loop (and after the state row is
// stored, since the LSTM cell updates c in place) one more pass gives value_last, and the epilogue (mgb_gae) walks the
// thread's column.
// VAL, step t of the thread's active env, after maze_logic and before env_reset: decides the cut from done and the
// trial draw, stores the task rule's cut into adv, and where the cut fires on a truncated step stores V of the terminal
// window (written into `row`, then the x column) into final_value.  Besides `row` and the x column's obs rows, which
// the step refills, it clobbers only what the carry then wipes: the h columns, c and the feedback rows.
template <int POL>
__device__ __forceinline__ void maze2d_terminal_value(const MazeConst &c, const MazeArgs &a, const mgb_critic &cr,
                                                      const MgbPolicyPlan<POL> &pol, const float *pol_w, float *pol_x,
                                                      float *pol_y, float *hid_prev, float *hid_new, float *cst,
                                                      const uint8_t *blob, const int32_t *eaten, const Env &s, int t,
                                                      int64_t e, int D, int done, int action, double reward,
                                                      uint32_t draw, float *row)
{
    constexpr bool RNN = POL == kPolGru || POL == kPolLstm;
    bool cut = done;
    if constexpr (RNN) {
        cut = done && (pol.reset == MGB_RNN_RESET_EPISODE || draw);
        if (pol.reset == MGB_RNN_RESET_TASK && cr.adv_dev) cr.adv_dev[(int64_t)t * a.n + e] = cut ? 1.f : 0.f;
    }
    if (!(cut && maze_truncated(c, blob, s))) return;
    maze2d_window(c, blob, eaten, a.n_pad, s, row);
    for (int k = 0; k < D; ++k) pol_x[k * k2dThreads + threadIdx.x] = row[k];
    const MgbMlp &head = mgb_policy_head(pol);
    float logits[4], v;
    mgb_population_weights(head, pol_w, pol.staged, [&](const float *w) {
        if constexpr (RNN) {
            if (pol.feedback) {
                float *fb = pol_x + D * k2dThreads + threadIdx.x;
                for (int k = 0; k < 4; ++k) fb[k * k2dThreads] = k == action ? 1.f : 0.f;
                fb[4 * k2dThreads] = (float)reward;
            }
            mgb_rnn_cell(pol, w, pol_x, hid_new, cst, hid_prev, k2dThreads, threadIdx.x);
            mgb_mlp_forward<true>(head, w + pol.s_head, hid_prev, POL == kPolLstm ? hid_new : pol_y, k2dThreads,
                                  threadIdx.x, logits, &v);
        } else {
            mgb_mlp_forward<true>(pol, w, pol_x, pol_y, k2dThreads, threadIdx.x, logits, &v);
        }
    });
    if (cr.final_value_dev) cr.final_value_dev[(int64_t)t * a.n + e] = v;
}

// VAL declares a minimum of one resident CTA per SM (.minnctapersm 1; 0 emits nothing, so the other instantiations are
// compiled as before): with ptxas's default register target the MLP kernel without RS spilled 8 bytes and the LSTM one
// with RS 84 bytes, where their value-less counterparts do not spill; with it none spills.
// EVAL (POL only, not FIN or VAL; mgb_maze_evaluate): whole-episode evaluation.  a.T is the step bound; the thread
// steps its env until its cr.episodes-th done and then stops, its state as that step left it.  It keeps the episode's
// return, length and index in registers and stores them at each done (mgb_eval_step); no per-step output is stored.  The
// window row in the tile is the thread's own scratch (the policy's next input), so the loop has no CTA barrier; a warp
// leaves it when all its envs have finished.  With RS a finished lane still takes part in the warp's draws (maze_sample_task
// is warp-cooperative) and changes nothing.  Without RS a trial handle's counts go up by the episodes at the end.
// EVAL keeps the counterpart's bounds, except with RS and the LSTM: at ptxas's default register target it took 128
// registers and spilled 80 bytes, where its counterpart takes 143 and does not spill; with one resident CTA per SM
// declared, as VAL does, it takes 168 and none spills.
// EXP (XM == 0, not RS or POL; mgb_maze_rollout_expert): the action of step t is act[t] when given, else the expert's
// (expert_action, from the mask of the state the env holds before step t); the mask goes to x.out [T][n].
template <int XM, bool FIN, bool REC, bool RS = false, int POL = 0, bool VAL = false, bool EVAL = false, bool EXP = false>
__global__ void __launch_bounds__(k2dThreads, VAL || (EVAL && RS && POL == kPolLstm) ? 1 : 0) maze2d_rollout_kernel(
    const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a, const __grid_constant__ MazeResample rs,
    const __grid_constant__ MgbPolicyPlan<POL> pol, const __grid_constant__ MgbCriticOrEval<EVAL> cr,
    const __grid_constant__ MazeExpertOr<EXP> x)
{
    constexpr bool RNN = POL == kPolGru || POL == kPolLstm;
    static_assert(!VAL || (POL && FIN), "value heads run on the policy rollouts with terminal outputs");
    static_assert(!EVAL || (POL && !FIN && !VAL), "evaluation runs a policy and stores only per-episode results");
    static_assert(!EXP || (XM == 0 && !RS && !POL), "expert rollouts are not mirrored, resampled or policy-driven");
    static_assert(!RS || XM == 0, "resampling rollouts are not mirrored");
    extern __shared__ __align__(128) float tile2d[];
    const int64_t e0 = (int64_t)blockIdx.x * k2dThreads;
    const int64_t e = e0 + threadIdx.x;
    const int W = 2 * c.view_grid + 1, D = W * W;
    const int rows = (int)((a.n - e0) < k2dThreads ? (a.n - e0) : k2dThreads);
    const bool active = e < a.n;
    const uint8_t *blob = nullptr;
    const TaskHdr *th = nullptr;
    const int8_t *walls = nullptr;
    Env s = {0, 0, 0, 0, 0.0};
    uint32_t tcount = 0;                                // RS on a trial handle: episodes finished on the current maze
    int32_t *eaten = a.eaten + e;
    if (active) {
        blob = a.blobs + (int64_t)a.env2task[e] * c.blob_bytes;
        th = blob_hdr(blob);
        walls = reinterpret_cast<const int8_t *>(blob + c.off_walls);
        const int4 ag = a.agent[e];
        s.gx = ag.x; s.gy = ag.y; s.ori = ag.z; s.steps = ag.w; s.life = a.life[e];
        if (RS && rs.count) tcount = rs.count[e];
    }
    const uint2 akey = make_uint2((uint32_t)a.act_seed, (uint32_t)(a.act_seed >> 32));
    const int64_t genv = a.env_base + e;
    const int n = c.n, g = c.view_grid;
    const float *pol_w = nullptr;                                   // the staged weights (mgb_population_weights)
    float *pol_x = nullptr, *pol_y = nullptr;                       // the input, the hidden layer
    float *hid_prev = nullptr, *hid_new = nullptr, *cst = nullptr;  // RNN: the columns h0, h1 and c
    const MgbMlp &head = mgb_policy_head(pol);                      // the plan of the categorical head
    if constexpr (POL) {
        static_assert(XM == 0, "policy rollouts are not mirrored");
        pol_x = tile2d + pol.smem_off + head.copies * pol.staged;
        if constexpr (RNN) {
            cst = pol_x + pol.in * k2dThreads;
            hid_prev = cst + pol.C() * k2dThreads;
            hid_new = hid_prev + pol.Hr * k2dThreads;
            pol_y = hid_new + pol.Hr * k2dThreads;     // w; the LSTM's head uses the dead h0 instead
        } else {
            pol_y = pol_x + pol.maxw * k2dThreads;
        }
        pol_w = tile2d + pol.smem_off;
        mgb_population_stage(pol, tile2d + pol.smem_off, e0, rows, k2dThreads);
        if (active) {       // the window of the loaded state: what the preceding reset() / step() returned
            float *row = tile2d + threadIdx.x * D;
            maze2d_window(c, blob, eaten, a.n_pad, s, row);
            for (int k = 0; k < D; ++k) pol_x[k * k2dThreads + threadIdx.x] = row[k];
            if (head.obs0_out)
                for (int k = 0; k < D; ++k) head.obs0_out[e * D + k] = row[k];
            if constexpr (RNN) {        // [h, c, feedback]
                const int S = pol.HC() + 5 * pol.feedback;
                const float *st = pol.state + e * S;
                for (int k = 0; k < pol.H; ++k) hid_prev[k * k2dThreads + threadIdx.x] = st[k];
                for (int k = 0; k < pol.C(); ++k) cst[k * k2dThreads + threadIdx.x] = st[pol.H + k];
                for (int k = pol.HC(); k < S; ++k) pol_x[(D + k - pol.HC()) * k2dThreads + threadIdx.x] = st[k];
                if (pol.state0_out)
                    for (int k = 0; k < S; ++k) pol.state0_out[e * S + k] = st[k];
            }
        }
        __syncthreads();    // the staged weights (the RS loop has no CTA barrier)
    }
    bool live = active;                 // EVAL: the env has episodes left
    double ev_ret = 0.0;                // EVAL: the return, length and index of the current episode
    int ev_len = 0, ev_ep = 0;
    for (int t = 0; t < a.T; ++t) {
        float *tile = tile2d + (size_t)(t & 1) * k2dThreads * D;
        if constexpr (EVAL) {
            if (!__any_sync(0xffffffffu, live)) break;
        } else if constexpr (RS) {                          // per warp: the warp's rows and their store are its own
            if ((threadIdx.x & 31) == 0) mgb_bulk_wait_read<1>();
            __syncwarp();
        } else {
            if (threadIdx.x == 0) mgb_bulk_wait_read<1>();  // the store issued two steps ago has read this tile
            __syncthreads();
        }
        uint32_t done_byte = 0, draw = 0;                  // draw (RS): the env finished and draws a new maze
        if (EVAL ? live : active) {
            int action;
            if constexpr (POL) {
                float logits[4], v;
                mgb_population_weights(head, pol_w, pol.staged, [&](const float *w) {
                    if constexpr (RNN) {
                        mgb_rnn_cell(pol, w, pol_x, hid_prev, cst, hid_new, k2dThreads, threadIdx.x);
                        if (pol.hid_out)
                            for (int k = 0; k < pol.H; ++k)
                                pol.hid_out[((int64_t)t * a.n + e) * pol.H + k] = hid_new[k * k2dThreads + threadIdx.x];
                        if constexpr (POL == kPolLstm) pol_y = hid_prev;   // dead until the carry makes it the next h
                        mgb_mlp_forward<VAL>(head, w + pol.s_head, hid_new, pol_y, k2dThreads, threadIdx.x, logits, &v);
                    } else {
                        mgb_mlp_forward<VAL>(pol, w, pol_x, pol_y, k2dThreads, threadIdx.x, logits, &v);
                    }
                });
                const float lp = mgb_categorical_action(head, genv, a.t_base + (uint32_t)t, logits, action);
                if (a.act_out) a.act_out[(int64_t)t * a.n + e] = action;
                if (head.logp_out) head.logp_out[(int64_t)t * a.n + e] = lp;
                if constexpr (VAL) cr.value_dev[(int64_t)t * a.n + e] = v;
            } else if constexpr (EXP) {
                const uint8_t m = expert_mask(c, x.mask, a.env2task[e], s);
                if (a.act) action = a.act[(int64_t)t * a.n + e];
                else {
                    action = expert_action(x, m, genv, a.t_base + (uint32_t)t);
                    if (a.act_out) a.act_out[(int64_t)t * a.n + e] = action;
                }
                if (x.out) x.out[(int64_t)t * a.n + e] = m;
            } else if (a.act) action = a.act[(int64_t)t * a.n + e];
            else {
                const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32),
                                                             a.t_base + (uint32_t)t, MGB_STREAM_ACTION), akey);
                action = (int)(r.x >> 30);                   // uniform over {0, 1, 2, 3}
                if (a.act_out) {
                    if (XM == 2) mgb_mc_st(mgb_shift(a.act_out + (int64_t)t * a.n + e, a.mir.delta[0]), (int32_t)action);
                    else a.act_out[(int64_t)t * a.n + e] = action;
                    if (XM == 1) mgb_mirror_store(a.mir, a.act_out + (int64_t)t * a.n + e, (int32_t)action);
                }
            }
            double reward;
            int done;
            maze_logic(c, blob, eaten, a.n_pad, s, action, reward, done);
            if (FIN) {
                static_assert(!FIN || XM == 0, "terminal rows and truncation flags are not mirrored");
                if (a.truncated) a.truncated[(int64_t)t * a.n + e] = maze_truncated(c, blob, s);
                if (done && a.final_obs)
                    maze2d_window(c, blob, eaten, a.n_pad, s, reinterpret_cast<float *>(a.final_obs) + ((int64_t)t * a.n + e) * D);
            }
            if constexpr (VAL) {    // the cut needs the trial draw before the reset
                if (RS && done) draw = (uint32_t)rs_draws(rs, tcount);
                maze2d_terminal_value<POL>(c, a, cr, pol, pol_w, pol_x, pol_y, hid_prev, hid_new, cst, blob, eaten, s, t,
                                           e, D, done, action, reward, draw, tile + threadIdx.x * D);
            }
            if constexpr (EVAL) live = mgb_eval_step(cr, a.n, e, reward, done, done && maze_truncated(c, blob, s), ev_ret,
                                                     ev_len, ev_ep);
            if (done && a.auto_reset) env_reset(c, blob, eaten, a.n_pad, s);
            if (!VAL && RS && done) draw = (uint32_t)rs_draws(rs, tcount);
            if (REC) path_store(c, a, e, s);
            if (a.rew && !EVAL) {
                if (XM == 2) mgb_mc_st(mgb_shift(a.rew + (int64_t)t * a.n + e, a.mir.delta[0]), reward);
                else a.rew[(int64_t)t * a.n + e] = reward;
                if (XM == 1) mgb_mirror_store(a.mir, a.rew + (int64_t)t * a.n + e, reward);
            }
            done_byte = (uint32_t)done;
            if (a.done && XM != 2 && !EVAL) {
                a.done[(int64_t)t * a.n + e] = (uint8_t)done;
                if (XM == 1) mgb_mirror_store(a.mir, a.done + (int64_t)t * a.n + e, (uint8_t)done);
            }
            if (a.obs || POL) {     // POL: the row is also the policy's next input
                float *row = tile + threadIdx.x * D;
                for (int p = 0; p < W; ++p)
                    for (int q = 0; q < W; ++q) {
                        const int x = s.gx - g + p, y = s.gy - g + q;
                        float v = -1.0f;
                        if (x >= 0 && x < n && y >= 0 && y < n) {
                            v = (float)(-(int)walls[x * n + y]);
                            if (c.task_type == MGB_MAZE_SURVIVAL)
                                v = (float)((double)v + food_now(c, blob, eaten, a.n_pad, s.steps, x * n + y));
                            else
                                v = (float)((double)v + ((x == th->goal[0] && y == th->goal[1]) ? 1.0 : 0.0));
                        }
                        row[p * W + q] = v;
                    }
                if (c.task_type == MGB_MAZE_SURVIVAL) row[g * W + g] = (float)s.life;
            }
            if constexpr (RNN) {
                // carry: the task rule fires where the env draws a new maze, which only RS does
                const bool wipe = done && (pol.reset == MGB_RNN_RESET_EPISODE || draw);
                if (wipe) {
                    for (int k = 0; k < pol.H; ++k) hid_new[k * k2dThreads + threadIdx.x] = 0.f;
                    for (int k = 0; k < pol.C(); ++k) cst[k * k2dThreads + threadIdx.x] = 0.f;
                }
                if (pol.feedback) {
                    float *fb = pol_x + D * k2dThreads + threadIdx.x;
                    for (int k = 0; k < 4; ++k) fb[k * k2dThreads] = !wipe && k == action ? 1.f : 0.f;
                    fb[4 * k2dThreads] = wipe ? 0.f : (float)reward;
                }
                float *const tmp = hid_prev;
                hid_prev = hid_new;
                hid_new = tmp;
            }
        }
        if constexpr (RS) {
            // auto-reset is on (the host requires it).  The step above left every finished env reset on its old task, with
            // that task's window in the tile and its path entry 0 stored; that step code stays as the other instantiations
            // compile it, and the few envs that draw redo the three on the new task here.  A finished env of a trial
            // handle that does not draw keeps what the step left: its next episode on the old maze.
            uint32_t fin = __ballot_sync(0xffffffffu, draw != 0);
            if (fin) {
                uint8_t *ws = reinterpret_cast<uint8_t *>(tile2d + 2 * k2dThreads * D) +
                              (threadIdx.x >> 5) * sampler_ws_bytes(c.n);
                const int64_t lane0_env = e - (threadIdx.x & 31);
                for (; fin; fin &= fin - 1) {
                    const int64_t el = lane0_env + (__ffs(fin) - 1);
                    maze_sample_task(c, rs.cfg, rs.seed, a.env_base + el, rs.epoch + el, ws,
                                     const_cast<uint8_t *>(a.blobs) + (int64_t)a.env2task[el] * c.blob_bytes);
                }
                __syncwarp();   // the new blobs, written by every lane, are read by their owners below
                if (draw) {
                    env_reset(c, blob, eaten, a.n_pad, s);
                    if (REC) path_store(c, a, e, s);
                    if (a.obs || POL) maze2d_window(c, blob, eaten, a.n_pad, s, tile + threadIdx.x * D);
                }
            }
        }
        if constexpr (POL) {        // the policy's input at step t + 1: the row this thread left in the tile
            if (EVAL ? live : active)
                for (int k = 0; k < D; ++k) pol_x[k * k2dThreads + threadIdx.x] = tile[threadIdx.x * D + k];
        }
        if (EVAL) {                 // no observation leaves the CTA
        } else if (XM == 2) {
            if (a.done) mgb_mc_st_bytes(mgb_shift(a.done + (int64_t)t * a.n + e, a.mir.delta[0]), done_byte, active);
            if (a.obs) {
                __syncthreads();
                mgb_mc_copy_tile(mgb_shift(reinterpret_cast<float *>(a.obs) + ((int64_t)t * a.n + e0) * D, a.mir.delta[0]),
                                 tile, (uint32_t)rows * (uint32_t)D * 4u);
            }
        } else if constexpr (RS) {
            // the warp's rows: 32 D 4 bytes, a multiple of 16, except in the tail warp
            const int w0 = threadIdx.x & ~31, lane = threadIdx.x & 31;
            const int wrows = rows - w0 < 32 ? rows - w0 : 32;
            if (a.obs && wrows > 0) {
                float *dst = reinterpret_cast<float *>(a.obs) + ((int64_t)t * a.n + e0 + w0) * D;
                const float *src = tile + w0 * D;
                const uint32_t bytes = (uint32_t)wrows * (uint32_t)D * 4u;
                if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
                    mgb_fence_proxy_async();
                    __syncwarp();
                    if (lane == 0) {
                        mgb_bulk_store(dst, src, bytes);
                        mgb_bulk_commit();
                    }
                } else {
                    __syncwarp();
                    for (int i = lane; i < wrows * D; i += 32) dst[i] = src[i];
                }
            }
        } else if (a.obs) {
            float *dst = reinterpret_cast<float *>(a.obs) + ((int64_t)t * a.n + e0) * D;
            const uint32_t bytes = (uint32_t)rows * (uint32_t)D * 4u;
            if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
                mgb_fence_proxy_async();
                __syncthreads();
                if (threadIdx.x == 0) {
                    mgb_bulk_store(dst, tile, bytes);
                    if (XM == 1) mgb_mirror_bulk_store(a.mir, dst, tile, bytes);
                    mgb_bulk_commit();
                }
            } else {
                __syncthreads();
                for (int i = threadIdx.x; i < rows * D; i += blockDim.x) {
                    dst[i] = tile[i];
                    if (XM == 1) mgb_mirror_store(a.mir, dst + i, tile[i]);
                }
            }
        }
    }
    if (active) {
        a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
        a.life[e] = s.life;
        if (RS && rs.count) rs.count[e] = tcount;
        if (EVAL && !RS && rs.count) rs.count[e] += (uint32_t)ev_ep;     // what maze_count_done_kernel adds
    }
    if constexpr (RNN) {
        if (active) {
            const int S = pol.HC() + 5 * pol.feedback;
            float *st = pol.state + e * S;
            for (int k = 0; k < pol.H; ++k) st[k] = hid_prev[k * k2dThreads + threadIdx.x];
            for (int k = 0; k < pol.C(); ++k) st[pol.H + k] = cst[k * k2dThreads + threadIdx.x];
            for (int k = pol.HC(); k < S; ++k) st[k] = pol_x[(D + k - pol.HC()) * k2dThreads + threadIdx.x];
        }
    }
    if constexpr (VAL) {
        if (active) {       // V(s_T), then GAE over the thread's column
            float logits[4], v;
            mgb_population_weights(head, pol_w, pol.staged, [&](const float *w) {
                if constexpr (RNN) {
                    mgb_rnn_cell(pol, w, pol_x, hid_prev, cst, hid_new, k2dThreads, threadIdx.x);
                    mgb_mlp_forward<true>(head, w + pol.s_head, hid_new, POL == kPolLstm ? hid_prev : pol_y, k2dThreads,
                                          threadIdx.x, logits, &v);
                } else {
                    mgb_mlp_forward<true>(pol, w, pol_x, pol_y, k2dThreads, threadIdx.x, logits, &v);
                }
            });
            if (cr.value_last_dev) cr.value_last_dev[e] = v;
            bool task_rule = false;
            if constexpr (RNN) task_rule = pol.reset == MGB_RNN_RESET_TASK;
            if (cr.adv_dev) mgb_gae(cr, a.T, a.n, e, v, a.rew, a.done, a.truncated, task_rule);
        }
    }
    if constexpr (RS) {
        if ((threadIdx.x & 31) == 0) mgb_bulk_wait_read<0>();
    } else {
        if (threadIdx.x == 0) mgb_bulk_wait_read<0>();
    }
}

// ---------------------------------------------------------------------------------------------------------------
// discrete 3-D: persistent CTA, step logic + raycast render
// ---------------------------------------------------------------------------------------------------------------
struct ColRec {                  // one screen column (ray), 64 bytes
    double cos_hp, cos_abs, sin_abs;   // float32 table values promoted (ray_caster_utils.py:82-92)
    double light, oma, ratio;          // wall shading: |cos/sin|, 1 - alpha, hit_dist * cos_hp / l_focal
    int16_t v_s, v_e;                  // wall span [v_s, v_e)
    int16_t ti, text_id;               // texture column, texture id
    int16_t n_hits, wall;              // transparent crossings, wall hit within max_vision
    int32_t pad;
};
struct RowRec {                  // one screen row, 24 bytes
    double distance, light;
    int32_t kind;                // 0 none, 1 floor, 2 ceiling
    int32_t pad;
};
struct HitRec {                  // one transparent crossing of a column, 16 bytes
    double tf;
    int16_t v_s, v_e;
    int32_t fid;                 // food slot of the crossed cell (pose cache: presence is decided per env, per step)
};
struct EnvDyn {                  // per env, per step: what the static pose layers must be combined with, 40 bytes
    int32_t slot;                // pose-cache slot of (task, cell, heading)
    int32_t bar_end;             // life bar end column (python slice semantics already applied)
    uint64_t present[2];         // bit f: food slot f is currently visible
    int32_t task, pad;           // pad: 8-bit signature of the missing foods that can tint this pose (0 = frame is final)
    int32_t vframe, pad2;        // >= 0: finished frame c_var8[vframe]; -1: c_rgb8[slot] (+ the tints `pad` asks for)
};
// what make_dyn needs to know about a pose, in ONE 32-byte record indexed like pose_index (two 16-byte loads issued together
// instead of the dependent chain pose_index -> c_fmask[slot] -> c_vbase[slot])
struct PoseRec {
    int32_t slot;                // pose-cache slot, -1: wall cell (never an agent pose)
    int32_t vbase;               // first variant frame of the pose, -1: none
    uint64_t fmask[2];           // food slots that can change this pose's image
    uint64_t pad;
};
struct BakeDesc {                // one variant frame to bake
    int32_t slot, pad;
    uint64_t present[2];
};
constexpr int kVariantBitsMax = 7;

// finished uint8 frame the env's observation starts from
__device__ __forceinline__ const uint8_t *frame_of(const MazeArgs &a, const EnvDyn &d, size_t frame_bytes)
{
    return d.vframe >= 0 ? a.c_var8 + (size_t)d.vframe * frame_bytes : a.c_rgb8 + (size_t)d.slot * frame_bytes;
}

__device__ __forceinline__ int trunc_i(double x) { return (int)x; }   // cvt.rzi: python/numba int()
// 32-bit observation word of a pixel value: the integer itself (MGB_OBS_I32, what the reference's array holds) or the same
// value as float32 (MGB_OBS_F32, the dtype the reference's observation_space declares, maze_env.py:37-39)
#define MGB_OBS_WORD(c, v) ((c).obs_dtype == MGB_OBS_F32 ? __float_as_int((float)(v)) : (v))

// rgb = light * (alpha * FAR_RGB + (1 - alpha) * texel), FAR_RGB = 0 (ray_caster_utils.py:7,118)
__device__ __forceinline__ void shade(int rgb[3], double light, double oma, uint32_t texel)
{
    rgb[0] = trunc_i(light * (oma * (double)(texel & 0xffu)));
    rgb[1] = trunc_i(light * (oma * (double)((texel >> 8) & 0xffu)));
    rgb[2] = trunc_i(light * (oma * (double)((texel >> 16) & 0xffu)));
}
// rgb = (1 - tf) * rgb + tf * (0, 255, 0)  (ray_caster_utils.py:8,121-123)
__device__ __forceinline__ void blend(int rgb[3], double tf)
{
    const double k = 1.0 - tf;
    rgb[0] = trunc_i(k * (double)rgb[0] + tf * 0.0);
    rgb[1] = trunc_i(k * (double)rgb[1] + tf * 255.0);
    rgb[2] = trunc_i(k * (double)rgb[2] + tf * 0.0);
}

__device__ __forceinline__ size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Terminal state of a finished env for the direct renderer's list pass: everything geometry() reads of an env (pose, life,
// food stamps, task).  Called before env_reset, which clears the stamps the terminal frame still shows.
__device__ __forceinline__ void push_terminal_state(const MazeConst &c, const MazeArgs &a, int64_t e, const Env &s,
                                                    const int32_t *eaten, float2 cp, double co)
{
    const int i = atomicAdd(a.fin_count, 1);
    a.fin_env[i] = (int32_t)e;
    a.fin_task[i] = a.env2task[e];
    a.fin_agent[i] = make_int4(s.gx, s.gy, s.ori, s.steps);
    a.fin_life[i] = s.life;
    for (int f = 0; f < c.f_max; ++f) a.fin_eaten[f * a.n_pad + i] = eaten[f * a.n_pad];
    if (c.kind == MGB_MAZE_CONTINUOUS_3D) { a.fin_cpos[i] = cp; a.fin_cori[i] = co; }
}

// FILL = false: render the observation of every env directly (step logic + ray cast + paint).
// FILL = true : render the STATIC layers of every cached pose (task, cell, heading) once, at set_task time: colours
//               before any transparency, the food slot under every floor/ceiling pixel, every POSSIBLE transparent
//               crossing of every column.  maze3d_compose_kernel then turns a pose + the env's current food state
//               into the exact observation with integer work only (the float64 geometry is memoised).
// ROLL = true (FILL = false, both 3-D kinds): T steps per launch.  A work item is (env, t), env-major: a CTA runs
//               t = 0..T-1 of env blockIdx.x, then of env blockIdx.x + gridDim.x, ...; so the pipelined order prepares
//               step t + 1 under the pixels of step t.  The pixel phase reads only its record set's snapshot (transparent
//               map, pose, life-bar end), never the env state that the next item's step logic is rewriting.
// FIN (ROLL only, mgb_maze_rollout_continuous_ex): the step logic of item (env, t) also stores truncated[t][env].  When the
//               env finished and final_obs is wanted it does NOT reset: the item's record set is built from the terminal
//               state and its pixels go to final_obs[t][env]; the next item is then (env, t, reset), whose geometry runs
//               env_reset, stores the state and builds the record set of the new episode's first frame for obs[t][env].
//               The destination travels with the record set; whether a reset item follows is published in shared memory
//               before the trip's closing barrier, so every thread takes the same next item.
// ROLL: mgb_maze_rollout of a 3-D handle off the pose cache; a discrete item reads the action
//               act[t][env] or draws it like maze3d_rollout_kernel.
// RS (ROLL only, mgb_maze_rollout with a sampler cfg): an item that resets its env (the item itself, or with FIN its
//               reset item) first gives the env a new task: warp 0 of the geometry group draws it into the item's tile
//               buffer (maze_sample_task), copies the tile to the env's table slot and fences the generic writes against
//               the bulk copies that load the slot later; thread 0 then resets the env on the new tile.  The next item's
//               tile is requested only after that (sequential mode), since it may be the same env.
// EXP (ROLL, not RS; mgb_maze_rollout_expert): the step logic of (e, t), which runs in the geometry phase, takes act[t]
// when given, else the expert's action on the state env e holds before step t, and stores that state's mask into
// x.out [T][n]; the pipeline order is the open-loop rollout's.
template <bool FILL, bool ROLL, bool FIN = false, bool RS = false, bool EXP = false>
__global__ void __launch_bounds__(kRenderThreads, 1) maze3d_kernel(const __grid_constant__ MazeConst c,
                                                                   const __grid_constant__ MazeArgs a,
                                                                   const __grid_constant__ MazeResample rs,
                                                                   const __grid_constant__ MazeExpertOr<EXP> x)
{
    static_assert(!FIN || (ROLL && !FILL), "terminal frames are a rollout output");
    static_assert(!RS || (ROLL && !FILL), "tasks are resampled in a rollout");
    static_assert(!EXP || (ROLL && !FILL && !RS), "expert rollouts run without resampling");
    extern __shared__ __align__(128) uint8_t smem[];
    // list pass (final_obs set): items are the entries of the terminal list the step logic just wrote; a CTA without one
    // leaves before it stages the textures
    const int64_t n_items = !FILL && !FIN && a.final_obs ? (int64_t)*a.fin_count : a.n;
    if ((int64_t)blockIdx.x >= n_items) return;
    const int n = c.n, H = c.res_h, V = c.res_v, ts = c.ts;
    const int tex_words = (c.n_tex + 1) * ts * ts;
    // ---- shared memory carve-up (mirrors maze3d_smem_bytes on the host)
    size_t off = 0;
    uint32_t *s_tex = reinterpret_cast<uint32_t *>(smem + off);          off = align_up(off + (size_t)tex_words * 4, 128);
    // record sets: [0] always, [1] when the direct renderer pipelines geometry of env e + 1 under the pixels of env e (c.pipe)
    const int nbuf = (!FILL && c.pipe) ? 2 : 1;
    uint8_t *s_blob2[2];
    double *s_transp2[2];
    ColRec *s_col2[2];
    RowRec *s_row2[2];
    HitRec *s_hit2[2];
    for (int b = 0; b < 2; ++b) {                                         // maze tiles: always two (this env's + the next one's in flight)
        s_blob2[b] = smem + off;                                          off = align_up(off + c.blob_bytes, 128);
    }
    for (int b = 0; b < 2; ++b) {
        if (b < nbuf) {
            s_transp2[b] = reinterpret_cast<double *>(smem + off);       off = align_up(off + (size_t)n * n * 8, 128);
            s_col2[b] = reinterpret_cast<ColRec *>(smem + off);          off = align_up(off + (size_t)H * sizeof(ColRec), 128);
            s_row2[b] = reinterpret_cast<RowRec *>(smem + off);          off = align_up(off + (size_t)V * sizeof(RowRec), 128);
            if (c.hits_in_global) s_hit2[b] = reinterpret_cast<HitRec *>(a.hit_scratch) + ((size_t)blockIdx.x * nbuf + b) * H * c.max_hits;
            else { s_hit2[b] = reinterpret_cast<HitRec *>(smem + off); off = align_up(off + (size_t)H * c.max_hits * sizeof(HitRec), 128); }
        } else {
            s_transp2[b] = s_transp2[0]; s_col2[b] = s_col2[0]; s_row2[b] = s_row2[0]; s_hit2[b] = s_hit2[0];
        }
    }
    double *s_rowc = reinterpret_cast<double *>(smem + off);             off = align_up(off + (size_t)V * 8, 128);
    const int px_bytes = c.obs_dtype == MGB_OBS_U8 ? 3 : 12;
    const int run_bytes = c.run_px * px_bytes;                           // 768
    const int n_slots = c.obs_dtype == MGB_OBS_U8 ? 2 : 1;               // int32 runs are 4x larger: single slot
    uint8_t *s_out = smem + off;                                          off = align_up(off + (size_t)(kRenderThreads / 32) * n_slots * run_bytes, 128);
    uint64_t *s_bar = reinterpret_cast<uint64_t *>(smem + off);          off += 32;
    int *s_env2[2];                                                       // [0..3] gx gy ori steps, [4] lifebar end
    double *s_pose2[2];                                                   // continuous maze: x, y, sin(ori), cos(ori)
    s_env2[0] = reinterpret_cast<int *>(smem + off);      s_pose2[0] = reinterpret_cast<double *>(smem + off + 32);
    s_env2[1] = reinterpret_cast<int *>(smem + off + 64); s_pose2[1] = reinterpret_cast<double *>(smem + off + 96);
    int *s_runctr = reinterpret_cast<int *>(smem + off + 128);            // [b]: next column run of record set b (pipelined mode)
    // FIN: [2 + bb] = 1 when the item whose geometry used tile buffer bb is followed by its reset item (one slot per trip
    // parity: a slot is rewritten two trips later, after every thread has read it); the destination of record set b is the
    // pointer at s_env2[b] + 6 (bytes 24..31 of the record set's int block)
    int *s_split = s_runctr + 2;
    uint8_t *s_rsws = smem + off + 144;                                   // RS: the sampler's workspace (sampler_ws_bytes)

    const int tid = threadIdx.x;
    // screen-row centre above the horizon, half_v - (d_v + 0.5) * pixel_size: the wall texel's row term (:184), pose independent
    for (int d_v = tid; d_v < V; d_v += blockDim.x) s_rowc[d_v] = c.half_v - (d_v + 0.5) * c.pixel_size;
    if (tid == 0) {
        mgb_mbar_init(&s_bar[0], 1);   // textures
        mgb_mbar_init(&s_bar[1], 1);   // task blob, buffer 0
        mgb_mbar_init(&s_bar[2], 1);   // task blob, buffer 1
        mgb_fence_mbar_init();
    }
    __syncthreads();
    // ---- textures: ONE bulk (TMA) copy per CTA for the whole launch, in <= 64 KB pieces
    if (tid == 0) {
        const uint32_t total = (uint32_t)tex_words * 4u;
        mgb_mbar_expect_tx(&s_bar[0], total);
        for (uint32_t o = 0; o < total; o += 65536u) {
            const uint32_t len = total - o < 65536u ? total - o : 65536u;
            mgb_bulk_load(reinterpret_cast<uint8_t *>(s_tex) + o, reinterpret_cast<const uint8_t *>(a.tex) + o, len,
                          &s_bar[0]);
        }
    }
    uint32_t blob_phase = 0;      // bit b: parity of buffer b's mbarrier
    bool tex_ready = false;
    int run_parity = 0;

    // ---- maze tiles (walls, texture ids, food table) arrive by TMA one env ahead of their use
    auto slot_of = [&](int64_t e) -> int64_t { return FILL ? (int64_t)a.fill_slot[e] : e; };   // FILL: item -> pose slot
    auto load_blob = [&](int64_t e, int b) {
        const int task_id = FILL ? a.poses[slot_of(e)].x : a.env2task[e];
        const uint8_t *src = a.blobs + (int64_t)task_id * c.blob_bytes;
        mgb_mbar_expect_tx(&s_bar[1 + b], (uint32_t)c.blob_bytes);
        mgb_bulk_load(b ? s_blob2[1] : s_blob2[0], src, (uint32_t)c.blob_bytes, &s_bar[1 + b]);
    };

    // ---- per-env geometry: tile, pose, transparent map, row table, one DDA ray per column -> record set `b`.  Run by `gn`
    // threads (gt = index among them) that synchronise among themselves: the whole CTA (__syncthreads), or -- pipelined
    // direct renderer -- the first kGeoThreads threads (named barrier 2) while every warp paints the previous env.
    // Tile buffer bb: loaded here (pipelined mode: the other buffer is being read by the pixel warps), or already requested by
    // the previous call, which prefetches `next_e` into the other buffer after its own wait (sequential mode).  FIN:
    // geo_reset marks the reset item of (e, t).
    bool geo_reset = false;
    auto geometry = [&](int64_t e, int t, int b, int bb, int gt, int gn, bool named, bool load_here, int64_t next_e) {
        auto gsync = [&]() { if (named) asm volatile("bar.sync 2, %0;" ::"n"(kGeoThreads) : "memory"); else __syncthreads(); };
        uint8_t *s_blob = (bb ? s_blob2[1] : s_blob2[0]);
        double *s_transp = (b ? s_transp2[1] : s_transp2[0]);
        ColRec *s_col = (b ? s_col2[1] : s_col2[0]);
        RowRec *s_row = (b ? s_row2[1] : s_row2[0]);
        HitRec *s_hit = (b ? s_hit2[1] : s_hit2[0]);
        int *s_env = (b ? s_env2[1] : s_env2[0]);
        double *s_pose = (b ? s_pose2[1] : s_pose2[0]);
        if (gt == 0) { if (load_here) load_blob(e, bb); s_runctr[b] = 0; }
        mgb_mbar_wait(&s_bar[1 + bb], (blob_phase >> bb) & 1u);
        blob_phase ^= 1u << bb;
        // FIN, sequential: when env e finishes here its reset item comes next and needs e's tile, not next_e's; which one is
        // known only after the step logic, so a prefetch of another env waits for it
        // RS, sequential: the next item may be this env on the task it is about to draw, so every prefetch waits for the draw
        const bool late = RS ? !load_here : (FIN && !load_here && !geo_reset && next_e != e);
        if (gt == 0 && next_e >= 0 && !late) load_blob(next_e, bb ^ 1);
        const TaskHdr *th = blob_hdr(s_blob);
        bool rs_env = false;                                             // RS: env e starts an episode on a new task
        // ---- step logic (one thread), then publish agent pose to the CTA
        if (FILL) {
            if (gt == 0) {
                const int4 ps = a.poses[slot_of(e)];
                s_env[0] = ps.y; s_env[1] = ps.z; s_env[2] = ps.w; s_env[3] = 0; s_env[4] = 0;
            }
        } else if (gt == 0) {
            const int4 ag = a.agent[e];
            Env s = {ag.x, ag.y, ag.z, ag.w, a.life[e]};
            int32_t *eaten = a.eaten + e;
            const bool cont = c.kind == MGB_MAZE_CONTINUOUS_3D;
            float cp[2] = {0.f, 0.f};
            double co = 0.0;
            if (cont) { const float2 p2 = a.cpos[e]; cp[0] = p2.x; cp[1] = p2.y; co = a.cori[e]; }
            if (a.do_step) {
                double reward;
                int done;
                const int64_t o = ROLL ? (int64_t)t * a.n + e : e;       // [T][n] outputs and actions of a rollout
                bool split = false;                                      // FIN: terminal frame now, reset item next
                if (FIN && geo_reset) {
                    done = 1;                                            // the reset that the step logic of (e, t) deferred
                } else {
                    if (cont) {
                        float tr, ws;
                        if (ROLL && !a.act_c) {   // uniform on [-1, 1): 2 u - 1 is exact for every 24-bit u01
                            const int64_t genv = a.env_base + e;
                            const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32),
                                                                         a.t_base + (uint32_t)t, MGB_STREAM_ACTION),
                                                              make_uint2((uint32_t)a.act_seed, (uint32_t)(a.act_seed >> 32)));
                            tr = 2.0f * mgb_u01(r.x) - 1.0f;
                            ws = 2.0f * mgb_u01(r.y) - 1.0f;
                            if (a.act_out_c) { a.act_out_c[2 * o] = tr; a.act_out_c[2 * o + 1] = ws; }
                        } else {
                            tr = a.act_c[2 * o]; ws = a.act_c[2 * o + 1];
                        }
                        continuous_move(c, s_blob, tr, ws, cp, co);
                        const float csf = (float)th->cell_size;                 // get_loc_grid, maze_base.py:199-202
                        s.gx = (int)(cp[0] / csf); s.gy = (int)(cp[1] / csf);
                        maze_evaluate(c, s_blob, eaten, a.n_pad, s, reward, done);
                    } else if (!ROLL) {
                        maze_logic(c, s_blob, eaten, a.n_pad, s, a.act[e], reward, done);
                    } else {
                        int action;
                        if constexpr (EXP) {
                            const uint8_t m = expert_mask(c, x.mask, a.env2task[e], s);
                            if (a.act) action = a.act[o];
                            else {
                                action = expert_action(x, m, a.env_base + e, a.t_base + (uint32_t)t);
                                if (a.act_out) a.act_out[o] = action;
                            }
                            if (x.out) x.out[o] = m;
                        } else if (a.act) action = a.act[o];
                        else {      // the draw of maze3d_rollout_kernel / maze2d_rollout_kernel
                            const int64_t genv = a.env_base + e;
                            const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32),
                                                                         a.t_base + (uint32_t)t, MGB_STREAM_ACTION),
                                                              make_uint2((uint32_t)a.act_seed, (uint32_t)(a.act_seed >> 32)));
                            action = (int)(r.x >> 30);
                            if (a.act_out) a.act_out[o] = action;
                        }
                        maze_logic(c, s_blob, eaten, a.n_pad, s, action, reward, done);
                    }
                    a.rew[o] = reward;
                    a.done[o] = (uint8_t)done;
                    if (a.truncated) a.truncated[o] = maze_truncated(c, s_blob, s);
                    if (done && a.fin_count) push_terminal_state(c, a, e, s, eaten, make_float2(cp[0], cp[1]), co);
                    split = FIN && done && a.final_obs && a.auto_reset;
                }
                if (done && a.auto_reset && !split) {
                    if (RS) {       // the episode ends here (with FIN, at its reset item): count it, and draw at the k-th
                        uint32_t cnt = rs.count ? rs.count[e] : 0u;
                        rs_env = rs_draws(rs, cnt);
                        if (rs.count) rs.count[e] = cnt;
                    }
                    env_reset(c, s_blob, eaten, a.n_pad, s);
                    if (cont) {
                        cp[0] = (float)(s.gx * th->cell_size + 0.5 * th->cell_size);
                        cp[1] = (float)(s.gy * th->cell_size + 0.5 * th->cell_size);
                        co = 0.0;
                    }
                }
                a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
                a.life[e] = s.life;
                path_store(c, a, e, s);
                if (cont) { a.cpos[e] = make_float2(cp[0], cp[1]); a.cori[e] = co; }
                if (FIN) {
                    s_split[bb] = split;
                    *reinterpret_cast<uint8_t **>(s_env + 6) =
                        reinterpret_cast<uint8_t *>(split ? a.final_obs : a.obs) + (size_t)o * H * V * px_bytes;
                    const int64_t ne = split ? e : next_e;
                    if (!RS && late && ne >= 0) load_blob(ne, bb ^ 1);
                }
            }
            if (cont) {          // publish the pose: position promoted from float32, sin/cos of the float64 heading
                s_pose[0] = (double)cp[0]; s_pose[1] = (double)cp[1]; s_pose[2] = sin(co); s_pose[3] = cos(co);
            }
            s_env[0] = s.gx; s_env[1] = s.gy; s_env[2] = s.ori; s_env[3] = s.steps;
            // life bar extent, maze_discrete_3d.py:118-126 (python slice semantics on the end index)
            int ex = trunc_i(c.lb_sx + s.life / th->max_life * c.lb_l);
            if (ex < 0) { ex += H; if (ex < 0) ex = 0; }
            if (ex > H) ex = H;
            s_env[4] = ex;
        }
        if (RS && gt < 32) {
            // the state just stored and published is the reset on the old task: draw the new one into this item's tile
            // buffer (pipelined mode: the pixel warps read the other one), then reset and publish again
            if (__shfl_sync(0xffffffffu, (int)rs_env, 0)) {
                maze_sample_task(c, rs.cfg, rs.seed, a.env_base + e, rs.epoch + e, s_rsws, s_blob);
                __syncwarp();
                uint4 *slot = reinterpret_cast<uint4 *>(const_cast<uint8_t *>(a.blobs) + (size_t)a.env2task[e] * c.blob_bytes);
                for (int i = gt; i < c.blob_bytes / 16; i += 32) slot[i] = reinterpret_cast<const uint4 *>(s_blob)[i];
                // the slot (global) and the tile (shared) were written through the generic proxy; later bulk copies read
                // the slot and overwrite the tile
                asm volatile("fence.proxy.async;" ::: "memory");
                __syncwarp();
                if (gt == 0) {
                    Env s;
                    env_reset(c, s_blob, a.eaten + e, a.n_pad, s);
                    a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
                    a.life[e] = s.life;
                    path_store(c, a, e, s);
                    if (c.kind == MGB_MAZE_CONTINUOUS_3D) {
                        const float2 p2 = make_float2((float)(s.gx * th->cell_size + 0.5 * th->cell_size),
                                                      (float)(s.gy * th->cell_size + 0.5 * th->cell_size));
                        a.cpos[e] = p2; a.cori[e] = 0.0;
                        s_pose[0] = (double)p2.x; s_pose[1] = (double)p2.y; s_pose[2] = 0.0; s_pose[3] = 1.0;   // heading 0
                    }
                    s_env[0] = s.gx; s_env[1] = s.gy; s_env[2] = s.ori; s_env[3] = s.steps;
                    int ex = trunc_i(c.lb_sx + s.life / th->max_life * c.lb_l);
                    if (ex < 0) { ex += H; if (ex < 0) ex = 0; }
                    if (ex > H) ex = H;
                    s_env[4] = ex;
                }
            }
            // the prefetch the step logic deferred: this env's tile again when its reset item follows, else the next item's
            if (gt == 0 && late) {
                const int64_t ne = FIN && s_split[bb] ? e : next_e;
                if (ne >= 0) load_blob(ne, bb ^ 1);
            }
        }
        gsync();
        const int gx = s_env[0], gy = s_env[1], ori = s_env[2], steps = s_env[3];
        const double cell_size = th->cell_size, vision_height = th->agent_height, ceil_height = th->wall_height;
        const bool cont_pose = !FILL && c.kind == MGB_MAZE_CONTINUOUS_3D;
        const double pos_x = cont_pose ? s_pose[0] : gx * cell_size + 0.5 * cell_size;   // get_cell_center, maze_base.py:194-197
        const double pos_y = cont_pose ? s_pose[1] : gy * cell_size + 0.5 * cell_size;
        const double text_to_cell = c.text_size / cell_size;
        (void)text_to_cell;

        // ---- transparent map + row table
        for (int k = gt; k < n * n; k += gn) {
            double v;
            if (c.task_type == MGB_MAZE_SURVIVAL) {
                if (FILL) {   // static superset: every food cell at its full value
                    const int f = reinterpret_cast<const int8_t *>(s_blob + c.off_fidx)[k];
                    v = f >= 0 ? reinterpret_cast<const double *>(s_blob + c.off_fval)[f] : 0.0;
                } else v = food_now(c, s_blob, a.eaten + e, a.n_pad, steps, k);
            } else v = (k == th->goal[0] * n + th->goal[1]) ? 1.0 : 0.0;
            s_transp[k] = v;
        }
        for (int d_v = gt; d_v < V; d_v += gn) {
            RowRec r;
            r.kind = 0; r.distance = 0.0; r.light = 0.0; r.pad = 0;
            if (d_v > V / 2) {                                       // floor rows, ray_caster_utils.py:95-101
                const double v_screen = (d_v + 0.5) * c.pixel_size - c.half_v;
                r.distance = vision_height / v_screen * c.l_focal;
                r.light = v_screen / c.l_focal;
                r.kind = r.distance > c.max_vision ? 0 : 1;
            } else if (d_v < V / 2) {                                // ceiling rows, :129-135
                const double v_screen = c.half_v - (d_v + 0.5) * c.pixel_size;
                r.distance = (ceil_height - vision_height) / v_screen * c.l_focal;
                r.light = v_screen / c.l_focal;
                r.kind = r.distance > c.max_vision ? 0 : 2;
            }
            s_row[d_v] = r;
        }
        gsync();
        // ---- one ray per column: DDA_2D (ray_caster_utils.py:11-62) + wall span set-up (:156-182)
        const int8_t *walls = reinterpret_cast<const int8_t *>(s_blob + c.off_walls);
        const int8_t *texts = reinterpret_cast<const int8_t *>(s_blob + c.off_texts);
        const float *ct = a.coltab + (size_t)(cont_pose ? 0 : ori) * 3 * H;
        for (int d_h = gt; d_h < H; d_h += gn) {
            ColRec cr;
            cr.cos_hp = (double)ct[d_h];
            if (cont_pose) {     // float64 heading: tables from the float64 sin/cos, stored as float32 (:82-92)
                const double ch = a.coltab_d[d_h], sh = a.coltab_d[H + d_h];
                cr.sin_abs = (double)(float)(sh * s_pose[3] + ch * s_pose[2]);
                cr.cos_abs = (double)(float)(ch * s_pose[3] - sh * s_pose[2]);
            } else {
                cr.cos_abs = (double)ct[H + d_h];
                cr.sin_abs = (double)ct[2 * H + d_h];
            }
            const double cos_ori = cr.cos_abs, sin_ori = cr.sin_abs;
            const int i0 = trunc_i(pos_x / cell_size), j0 = trunc_i(pos_y / cell_size);
            const double delta_dist_x = fabs(cos_ori) < 1.0e-6 ? 1.0e+6 : fabs(cell_size / cos_ori);
            const double delta_dist_y = fabs(sin_ori) < 1.0e-6 ? 1.0e+6 : fabs(cell_size / sin_ori);
            const double d_x = cos_ori > 0 ? ((i0 + 1) * cell_size - pos_x) : (i0 * cell_size - pos_x);
            const double d_y = sin_ori > 0 ? ((j0 + 1) * cell_size - pos_y) : (j0 * cell_size - pos_y);
            double side_x = fabs(cos_ori) < 1.0e-6 ? 1.0e+6 : d_x / cos_ori;
            double side_y = fabs(sin_ori) < 1.0e-6 ? 1.0e+6 : d_y / sin_ori;
            const int delta_i = cos_ori > 0 ? 1 : -1, delta_j = sin_ori > 0 ? 1 : -1;
            int hit_i = i0, hit_j = j0, hit_side = 0, nh = 0;
            double hit_dist = 0.0;
            HitRec *hits = s_hit + (size_t)d_h * c.max_hits;
            // a transparent crossing at distance d paints the span of a wall standing there (:191-198)
            const int8_t *fidx_map = reinterpret_cast<const int8_t *>(s_blob + c.off_fidx);
            auto record_hit = [&](double d, double strength, int cell) {
                if (nh >= c.max_hits) return;
                const double ratio = d * cr.cos_hp / c.l_focal;
                const double tv = (ceil_height - vision_height) / ratio, bv = vision_height / ratio;
                const int s0 = trunc_i((c.half_v - tv) / c.pixel_size), s1 = trunc_i((c.half_v + bv) / c.pixel_size);
                HitRec hr;
                hr.tf = strength * 0.50 + 0.10;
                hr.v_s = (int16_t)(s0 < 0 ? 0 : s0);
                hr.v_e = (int16_t)(s1 > V ? V : s1);
                hr.fid = c.task_type == MGB_MAZE_SURVIVAL ? (int)fidx_map[cell] : 0;
                hits[nh++] = hr;
            };
            if (s_transp[hit_i * n + hit_j] > 0.01)                   // start cell, :25-29
                record_hit(side_x < side_y ? side_x : side_y, s_transp[hit_i * n + hit_j], hit_i * n + hit_j);
            while (hit_dist < c.max_vision) {
                if (side_x < side_y) {
                    hit_i += delta_i;
                    side_y -= side_x;
                    hit_dist += side_x;
                    if (hit_i < 0 || hit_i >= n) {
                        if (hit_j < 0 || hit_j >= n) { hit_dist = 1.0e+6; break; }
                    } else if (hit_j >= 0 && hit_j < n) {
                        const double tv = s_transp[hit_i * n + hit_j];
                        if (tv > 0.01) record_hit(hit_dist, tv, hit_i * n + hit_j);
                        if (walls[hit_i * n + hit_j] > 0) { hit_side = 0; break; }
                    }
                    side_x = delta_dist_x;
                } else {
                    hit_j += delta_j;
                    side_x -= side_y;
                    hit_dist += side_y;
                    if (hit_i < 0 || hit_i >= n) {
                        if (hit_j < 0 || hit_j >= n) { hit_dist = 1.0e+6; break; }
                    } else if (hit_j >= 0 && hit_j < n) {
                        const double tv = s_transp[hit_i * n + hit_j];
                        if (tv > 0.01) record_hit(hit_dist, tv, hit_i * n + hit_j);
                        if (walls[hit_i * n + hit_j] > 0) { hit_side = 1; break; }
                    }
                    side_y = delta_dist_y;
                }
            }
            cr.wall = hit_dist > c.max_vision ? 0 : 1;               // :162-163 (skips overlays too)
            cr.n_hits = 0; cr.v_s = 0; cr.v_e = 0; cr.ti = 0; cr.text_id = 0;
            cr.light = 0.0; cr.oma = 0.0; cr.ratio = 1.0; cr.pad = 0;
            if (cr.wall) {
                const double alpha = fmin(1.0, fmax(2.0 * hit_dist / c.max_vision - 1.0, 0.0));
                const int ci = hit_i < 0 ? 0 : (hit_i >= n ? n - 1 : hit_i);
                const int cj = hit_j < 0 ? 0 : (hit_j >= n ? n - 1 : hit_j);
                cr.text_id = texts[ci * n + cj];
                const double hit_pt_x = hit_dist * cos_ori + pos_x;
                const double hit_pt_y = hit_dist * sin_ori + pos_y;
                double local_h;
                if (hit_side == 0) {
                    local_h = hit_pt_y / cell_size; local_h -= floor(local_h);
                    cr.light = fabs(cos_ori);
                } else {
                    local_h = hit_pt_x / cell_size; local_h -= floor(local_h);
                    cr.light = fabs(sin_ori);
                }
                double d_i = local_h / c.text_size;
                d_i -= floor(d_i);
                cr.ti = (int16_t)trunc_i(ts * d_i);
                cr.oma = 1.0 - alpha;
                cr.ratio = hit_dist * cr.cos_hp / c.l_focal;
                const double top_v = (ceil_height - vision_height) / cr.ratio, bot_v = vision_height / cr.ratio;
                int v_s = trunc_i((c.half_v - top_v) / c.pixel_size), v_e = trunc_i((c.half_v + bot_v) / c.pixel_size);
                cr.v_s = (int16_t)(v_s < 0 ? 0 : v_s);
                cr.v_e = (int16_t)(v_e > V ? V : v_e);
                cr.n_hits = (int16_t)nh;
            }
            s_col[d_h] = cr;
            if (FILL) {
                a.c_colhits[(size_t)slot_of(e) * H + d_h] = (uint8_t)cr.n_hits;
                HitRec *gh = reinterpret_cast<HitRec *>(a.c_hits) + ((size_t)slot_of(e) * H + d_h) * c.max_hits;
                for (int k = 0; k < cr.n_hits; ++k) gh[k] = hits[k];
            }
        }
    };
    // ---- pixels of env e from record set b (direct renderer).  dyn: warps pull column runs from a shared counter (the
    // geometry warps join late), else run = warp, warp + n_warps, ...
    auto pixels = [&](int64_t e, int b, int bb, bool dyn) {
        uint8_t *s_blob = (bb ? s_blob2[1] : s_blob2[0]);
        double *s_transp = (b ? s_transp2[1] : s_transp2[0]);
        ColRec *s_col = (b ? s_col2[1] : s_col2[0]);
        RowRec *s_row = (b ? s_row2[1] : s_row2[0]);
        HitRec *s_hit = (b ? s_hit2[1] : s_hit2[0]);
        int *s_env = (b ? s_env2[1] : s_env2[0]);
        double *s_pose = (b ? s_pose2[1] : s_pose2[0]);
        const TaskHdr *th = blob_hdr(s_blob);
        const int gx = s_env[0], gy = s_env[1], ori = s_env[2], steps = s_env[3];
        const double cell_size = th->cell_size, vision_height = th->agent_height, ceil_height = th->wall_height;
        const bool cont_pose = !FILL && c.kind == MGB_MAZE_CONTINUOUS_3D;
        const double pos_x = cont_pose ? s_pose[0] : gx * cell_size + 0.5 * cell_size;   // get_cell_center, maze_base.py:194-197
        const double pos_y = cont_pose ? s_pose[1] : gy * cell_size + 0.5 * cell_size;
        const double text_to_cell = c.text_size / cell_size;

        const int8_t *walls = reinterpret_cast<const int8_t *>(s_blob + c.off_walls);
        const int8_t *texts = reinterpret_cast<const int8_t *>(s_blob + c.off_texts);
        const float *ct = a.coltab + (size_t)(cont_pose ? 0 : ori) * 3 * H;
        (void)walls; (void)steps; (void)ct; (void)ceil_height; (void)text_to_cell; (void)s_transp; (void)s_hit; (void)s_col; (void)s_env;   // the two pixel paths share one preamble
        if (!tex_ready) { mgb_mbar_wait(&s_bar[0], 0); tex_ready = true; }
        // ---- pixels.  Each WARP owns runs of whole screen columns (c.run_px / V of them, 768 B of output): the column
        // record is warp-uniform (one broadcast read, held in registers), lanes take rows d_v = lane, lane + 32, ...,
        // write into the warp's private staging slot, and lane 0 issues ONE bulk (TMA) store per run; the slot is
        // double-buffered.  No block-wide barrier inside an env: a warp with cheap pixels (walls) simply moves on.
        const int total_px = H * V;
        const int lb_sx = trunc_i(c.lb_sx), lb_ex = s_env[4];
        const int lb_sy = trunc_i(c.lb_sy);
        int lb_ey = trunc_i(c.lb_sy + c.lb_w);
        if (lb_ey > V) lb_ey = V;
        const bool has_bar = c.task_type == MGB_MAZE_SURVIVAL;
        uint8_t *gobs = FIN ? *reinterpret_cast<uint8_t *const *>(s_env + 6)   // FIN: the record set's destination
                            : reinterpret_cast<uint8_t *>(a.obs) + (size_t)(a.final_obs ? a.fin_env[e] : e) * total_px * px_bytes;
        const int lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
        const double inv_cell = th->inv_cell, inv_t2c = th->inv_t2c;
        const bool cell_p2 = th->cell_pow2 != 0, t2c_p2 = th->t2c_pow2 != 0, text_p2 = c.text_pow2 != 0;
        const double *efft = (c.n_cls > 0 && th->cls >= 0) ? a.efftab + (size_t)th->cls * total_px : nullptr;
        const double *fogt = efft ? a.fogtab + (size_t)th->cls * total_px : nullptr;
        const double fog_from = 0.4999 * c.max_vision;
        const double dts = (double)ts;
        // Exact integer texel / cell indices.  With cell_size = 2^a, text_size = 2^b (a >= b) and ts = 2^m, every scaling in
        //   texel = trunc(ts * frac((cell/text) * frac(x / cell)))   (floor, ray_caster_utils.py:106-112)
        //   texel = trunc(ts * frac(x / text))                        (ceiling, :140-144),   cell = trunc(x / cell)
        // is by a power of two and every frac() is exact, so for x >= 0 all three equal integer functions of
        // t = trunc(x * ts / text): texel = t mod ts, cell = t >> log2(ts * cell / text).  One multiply and one conversion per
        // axis instead of three multiplies, two floors, two subtractions and two conversions; pixels with a negative
        // coordinate (the reference truncates those toward zero) and tasks with other sizes take the original expressions.
        const bool fast_ix = cell_p2 && t2c_p2 && text_p2 && (ts & (ts - 1)) == 0 && cell_size >= c.text_size;
        const double tex_scale = dts * c.inv_text;
        int cell_shift = 0;
        { int ex = 0; frexp(tex_scale * cell_size, &ex); cell_shift = ex - 1; }
        const int ts_mask = ts - 1;
        const double ix_lim = 1073741824.0 / tex_scale;                        // t < 2^30

        // floor / ceiling pixel (ray_caster_utils.py:94-153) at effective distance `eff`.  Returns true when a transparent
        // cell tinted it (`mark`).  Floor and ceiling rows share ONE instruction stream on the integer-index path (selects
        // for texture id, fog weight and tint threshold): a warp pass that holds both kinds does not run two code paths.
        auto fc_px = [&](const RowRec &rr, double eff, double fog, const ColRec &cr, int rgb[3]) -> bool {
            bool mark = false;
            if (rr.kind == 0) return false;
            const double hit_x = eff * cr.cos_abs + pos_x;
            const double hit_y = eff * cr.sin_abs + pos_y;
            const bool fastpx = fast_ix && hit_x >= 0.0 && hit_y >= 0.0 && hit_x < ix_lim && hit_y < ix_lim;
            if (fastpx) {
                const int tx = trunc_i(hit_x * tex_scale), ty = trunc_i(hit_y * tex_scale);
                const int i = tx >> cell_shift, j = ty >> cell_shift;
                const int tu = tx & ts_mask, tv_ = ty & ts_mask;
                const bool inside = (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n;
                const bool is_floor = rr.kind == 1;
                const int cell = inside ? i * n + j : 0;
                const int text_id = is_floor ? (int)texts[cell] : c.n_tex;
                // floor: 1 - alpha * light (:118), ceiling: 1 - alpha (:149); alpha * 1.0 == alpha exactly
                const double oma = 1.0 - fog * (is_floor ? rr.light : 1.0);
                shade(rgb, rr.light, oma, s_tex[(text_id * ts + tu) * ts + tv_]);
                if (is_floor && !inside) { rgb[0] = 0; rgb[1] = 0; rgb[2] = 0; }   // the floor is drawn inside the maze only (:104)
                const double tv = inside ? s_transp[cell] : 0.0;
                if (tv > (is_floor ? 0.01 : 0.0)) { blend(rgb, tv * 0.50 + 0.10); mark = true; }      // :119-123, :150-153
                return mark;
            }
            const double ci = cell_p2 ? hit_x * inv_cell : hit_x / cell_size;
            const double cj = cell_p2 ? hit_y * inv_cell : hit_y / cell_size;
            const int i = trunc_i(ci), j = trunc_i(cj);
            const bool inside = (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n;
            if (rr.kind == 1) {                                               // floor, :103-126
                if (inside) {
                    const int text_id = texts[i * n + j];
                    double d_i = ci - floor(ci), d_j = cj - floor(cj);
                    d_i = t2c_p2 ? d_i * inv_t2c : d_i / text_to_cell;
                    d_j = t2c_p2 ? d_j * inv_t2c : d_j / text_to_cell;
                    d_i -= floor(d_i); d_j -= floor(d_j);
                    d_i *= dts; d_j *= dts;
                    shade(rgb, rr.light, 1.0 - fog * rr.light, s_tex[(text_id * ts + trunc_i(d_i)) * ts + trunc_i(d_j)]);
                    const double tv = s_transp[i * n + j];
                    if (tv > 0.01) { blend(rgb, tv * 0.50 + 0.10); mark = true; }
                }
            } else {                                                          // ceiling, :137-153
                const double fi = text_p2 ? hit_x * c.inv_text : hit_x / c.text_size;
                const double fj = text_p2 ? hit_y * c.inv_text : hit_y / c.text_size;
                double d_i = fi - floor(fi), d_j = fj - floor(fj);
                d_i *= dts; d_j *= dts;
                shade(rgb, rr.light, 1.0 - fog, s_tex[(c.n_tex * ts + trunc_i(d_i)) * ts + trunc_i(d_j)]);
                if (inside) {
                    const double tv = s_transp[i * n + j];
                    if (tv > 0) { blend(rgb, tv * 0.50 + 0.10); mark = true; }
                }
            }
            return mark;
        };
        // effective distance of pixel (d_h, d_v): tabulated per height class, else the division itself (:97, :131)
        auto eff_of = [&](const double *effc, int d_v, const ColRec &cr) -> double {
            return effc ? __ldg(effc + d_v) : s_row[d_v].distance / cr.cos_hp;
        };
        // alpha = clip(2 eff / max_vision - 1, 0, 1): tabulated with eff, else evaluated here.  It is exactly 0 while
        // 2 eff / max_vision < 1; the margin keeps that shortcut independent of the division's rounding
        auto fog_of = [&](const double *fogc, int d_v, double eff) -> double {
            if (fogc) return __ldg(fogc + d_v);
            return eff > fog_from ? fmin(1.0, fmax(2.0 * eff / c.max_vision - 1.0, 0.0)) : 0.0;
        };
        // wall pixel (:184-189)
        auto wall_px = [&](int d_v, const ColRec &cr, int rgb[3]) {
            const double local_v = s_rowc[d_v] * cr.ratio + vision_height;
            double d_j = text_p2 ? local_v * c.inv_text : local_v / c.text_size;
            d_j -= floor(d_j);
            shade(rgb, cr.light, cr.oma, s_tex[(cr.text_id * ts + cr.ti) * ts + trunc_i(dts * d_j)]);
        };
        const bool out_u8 = c.obs_dtype == MGB_OBS_U8;
        auto store_px = [&](uint8_t *buf, int p, const int rgb[3]) {
            if (out_u8) {
                buf[p * 3 + 0] = (uint8_t)(rgb[0] > 255 ? 255 : rgb[0]);
                buf[p * 3 + 1] = (uint8_t)(rgb[1] > 255 ? 255 : rgb[1]);
                buf[p * 3 + 2] = (uint8_t)(rgb[2] > 255 ? 255 : rgb[2]);
            } else {
                int32_t *o = reinterpret_cast<int32_t *>(buf) + p * 3;
                o[0] = MGB_OBS_WORD(c, rgb[0]); o[1] = MGB_OBS_WORD(c, rgb[1]); o[2] = MGB_OBS_WORD(c, rgb[2]);
            }
        };

        const int cols_per_run = c.run_px / V > 0 ? c.run_px / V : 1;
        const int n_runs = (H + cols_per_run - 1) / cols_per_run;
        auto next_run = [&](int prev) {
            if (!dyn) return prev < 0 ? warp : prev + n_warps;
            int r = 0;
            if (lane == 0) r = atomicAdd(&s_runctr[b], 1);
            return __shfl_sync(0xffffffffu, r, 0);
        };
        for (int run = next_run(-1); run < n_runs; run = next_run(run)) {
            uint8_t *buf = s_out + ((size_t)warp * n_slots + (n_slots == 2 ? run_parity : 0)) * run_bytes;
            const int h0 = run * cols_per_run;
            const int ncol = H - h0 < cols_per_run ? H - h0 : cols_per_run;
            // the bulk store that last used this slot (two runs ago) must have finished reading it
            if (lane == 0) { if (n_slots == 2) mgb_bulk_wait_read<1>(); else mgb_bulk_wait_read<0>(); }
            __syncwarp();
            for (int cc = 0; cc < ncol; ++cc) {
                const int d_h = h0 + cc;
                const ColRec cr = s_col[d_h];                              // warp-uniform
                const bool bar_col = has_bar && d_h >= lb_sx && d_h < lb_ex;
                const double *effc = efft ? efft + (size_t)d_h * V : nullptr;
                const double *fogc = efft ? fogt + (size_t)d_h * V : nullptr;
                if (cr.n_hits == 0) {
                    // Column without transparent crossings: every pixel is EITHER wall OR floor/ceiling.  The two kinds are
                    // walked separately -- the wall span [ws, we), then the remaining rows as one compacted index range --
                    // so that a warp pass runs one code path with (almost) all lanes instead of both paths half empty.
                    int ws = 0, we = 0;
                    if (cr.wall) {
                        ws = cr.v_s < 0 ? 0 : (cr.v_s > V ? V : cr.v_s);
                        we = cr.v_e < ws ? ws : (cr.v_e > V ? V : cr.v_e);
                    }
                    const int span = we - ws, rest = V - span;
                    // the floor/ceiling rows' distances come from L2: ask for the first two passes' worth now, use them after
                    // the wall passes
                    double eff_a = 0.0, eff_b = 0.0, fog_a = 0.0, fog_b = 0.0;
                    {
                        const int ka = lane, kb = lane + 32;
                        if (ka < rest) {
                            const int d_v = ka < ws ? ka : ka + span;
                            eff_a = eff_of(effc, d_v, cr); fog_a = fog_of(fogc, d_v, eff_a);
                        }
                        if (kb < rest) {
                            const int d_v = kb < ws ? kb : kb + span;
                            eff_b = eff_of(effc, d_v, cr); fog_b = fog_of(fogc, d_v, eff_b);
                        }
                    }
                    for (int d_v = ws + lane; d_v < we; d_v += 32) {
                        int rgb[3];
                        wall_px(d_v, cr, rgb);
                        if (bar_col && d_v >= lb_sy && d_v < lb_ey) { rgb[0] = 255; rgb[1] = 0; rgb[2] = 0; }
                        store_px(buf, cc * V + d_v, rgb);
                    }
                    for (int k = lane; k < rest; k += 32) {
                        const int d_v = k < ws ? k : k + span;
                        int rgb[3] = {0, 0, 0};
                        const double eff = k < 32 ? eff_a : (k < 64 ? eff_b : eff_of(effc, d_v, cr));
                        const double fog = k < 32 ? fog_a : (k < 64 ? fog_b : fog_of(fogc, d_v, eff));
                        fc_px(s_row[d_v], eff, fog, cr, rgb);
                        if (bar_col && d_v >= lb_sy && d_v < lb_ey) { rgb[0] = 255; rgb[1] = 0; rgb[2] = 0; }
                        store_px(buf, cc * V + d_v, rgb);
                    }
                    continue;
                }
                const HitRec *hits = s_hit + (size_t)d_h * c.max_hits;
                for (int d_v = lane; d_v < V; d_v += 32) {
                    int rgb[3] = {0, 0, 0};
                    bool mark = false;
                    const bool in_wall = cr.wall && d_v >= cr.v_s && d_v < cr.v_e;
                    const double eff = eff_of(effc, d_v, cr);
                    mark = fc_px(s_row[d_v], eff, fog_of(fogc, d_v, eff), cr, rgb);   // also under a wall: `mark` decides about the overlays below
                    if (in_wall) wall_px(d_v, cr, rgb);
                    if (!mark) {                                              // transparent overlays, :191-205
                        for (int k = 0; k < cr.n_hits; ++k)
                            if (d_v >= hits[k].v_s && d_v < hits[k].v_e) blend(rgb, hits[k].tf);
                    }
                    if (bar_col && d_v >= lb_sy && d_v < lb_ey) {             // life bar, maze_discrete_3d.py:118-126
                        rgb[0] = 255; rgb[1] = 0; rgb[2] = 0;
                    }
                    store_px(buf, cc * V + d_v, rgb);
                }
            }
            uint8_t *dst = gobs + (size_t)h0 * V * px_bytes;
            const uint32_t bytes = (uint32_t)(ncol * V) * (uint32_t)px_bytes;
            if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
                mgb_fence_proxy_async();
                __syncwarp();
                if (lane == 0) {
                    mgb_bulk_store(dst, buf, bytes);
                    mgb_bulk_commit();
                }
            } else {
                __syncwarp();
                for (uint32_t i = lane; i < bytes; i += 32) dst[i] = buf[i];
            }
            run_parity ^= 1;
        }
    };
    // ---- FILL: static layers of pose e (record set 0)
    auto fill_pixels = [&](int64_t e, int bb) {
        const int b = 0;
        uint8_t *s_blob = (bb ? s_blob2[1] : s_blob2[0]);
        double *s_transp = (b ? s_transp2[1] : s_transp2[0]);
        ColRec *s_col = (b ? s_col2[1] : s_col2[0]);
        RowRec *s_row = (b ? s_row2[1] : s_row2[0]);
        HitRec *s_hit = (b ? s_hit2[1] : s_hit2[0]);
        int *s_env = (b ? s_env2[1] : s_env2[0]);
        double *s_pose = (b ? s_pose2[1] : s_pose2[0]);
        const TaskHdr *th = blob_hdr(s_blob);
        const int gx = s_env[0], gy = s_env[1], ori = s_env[2], steps = s_env[3];
        const double cell_size = th->cell_size, vision_height = th->agent_height, ceil_height = th->wall_height;
        const bool cont_pose = !FILL && c.kind == MGB_MAZE_CONTINUOUS_3D;
        const double pos_x = cont_pose ? s_pose[0] : gx * cell_size + 0.5 * cell_size;   // get_cell_center, maze_base.py:194-197
        const double pos_y = cont_pose ? s_pose[1] : gy * cell_size + 0.5 * cell_size;
        const double text_to_cell = c.text_size / cell_size;

        const int8_t *walls = reinterpret_cast<const int8_t *>(s_blob + c.off_walls);
        const int8_t *texts = reinterpret_cast<const int8_t *>(s_blob + c.off_texts);
        const float *ct = a.coltab + (size_t)(cont_pose ? 0 : ori) * 3 * H;
        (void)walls; (void)steps; (void)ct; (void)ceil_height; (void)text_to_cell; (void)s_transp; (void)s_hit; (void)s_col; (void)s_env;   // the two pixel paths share one preamble
            // ---- static layers of this pose: colour before any transparency (wall colour wins inside the wall span),
            // the food slot of the floor / ceiling cell under every pixel, one word + one byte per pixel, coalesced
            const int total_px = H * V;
            const double inv_cell = th->inv_cell, inv_t2c = th->inv_t2c;
            const bool cell_p2 = th->cell_pow2 != 0, t2c_p2 = th->t2c_pow2 != 0, text_p2 = c.text_pow2 != 0;
            const double *efft = (c.n_cls > 0 && th->cls >= 0) ? a.efftab + (size_t)th->cls * total_px : nullptr;
            const double fog_from = 0.4999 * c.max_vision;
            const double dts = (double)ts;
            const int8_t *fidx = reinterpret_cast<const int8_t *>(s_blob + c.off_fidx);
            const int goal_cell = th->goal[0] * n + th->goal[1];
            const size_t slot = (size_t)slot_of(e);
            uint32_t *gpx = a.c_px + slot * total_px;
            uint8_t *gfid = a.c_fid + slot * total_px;
            for (int q = tid; q < total_px; q += blockDim.x) {
                const int d_h = q / V, d_v = q - d_h * V;
                const ColRec &cr = s_col[d_h];
                const RowRec &rr = s_row[d_v];
                int rgb[3] = {0, 0, 0};
                int fid = 0xFF;
                const bool in_wall = cr.wall && d_v >= cr.v_s && d_v < cr.v_e;
                if (rr.kind != 0 && (!in_wall || cr.n_hits > 0)) {
                    const double eff = efft ? __ldg(efft + q) : rr.distance / cr.cos_hp;
                    double fog = 0.0;
                    if (eff > fog_from) fog = fmin(1.0, fmax(2.0 * eff / c.max_vision - 1.0, 0.0));
                    const double hit_x = eff * cr.cos_abs + pos_x;
                    const double hit_y = eff * cr.sin_abs + pos_y;
                    const double ci = cell_p2 ? hit_x * inv_cell : hit_x / cell_size;
                    const double cj = cell_p2 ? hit_y * inv_cell : hit_y / cell_size;
                    const int i = trunc_i(ci), j = trunc_i(cj);
                    const bool inside = (unsigned)i < (unsigned)n && (unsigned)j < (unsigned)n;
                    if (inside) {
                        if (c.task_type == MGB_MAZE_SURVIVAL) { const int f = fidx[i * n + j]; if (f >= 0) fid = f; }
                        else if (i * n + j == goal_cell) fid = 0;
                    }
                    if (rr.kind == 1) {
                        if (inside) {
                            double d_i = ci - floor(ci), d_j = cj - floor(cj);
                            const int text_id = texts[i * n + j];
                            d_i = t2c_p2 ? d_i * inv_t2c : d_i / text_to_cell;
                            d_j = t2c_p2 ? d_j * inv_t2c : d_j / text_to_cell;
                            d_i -= floor(d_i); d_j -= floor(d_j);
                            d_i *= dts; d_j *= dts;
                            shade(rgb, rr.light, 1.0 - fog * rr.light,
                                  s_tex[(text_id * ts + trunc_i(d_i)) * ts + trunc_i(d_j)]);
                        } else fid = 0xFF;
                    } else {
                        const double fi = text_p2 ? hit_x * c.inv_text : hit_x / c.text_size;
                        const double fj = text_p2 ? hit_y * c.inv_text : hit_y / c.text_size;
                        double d_i = fi - floor(fi), d_j = fj - floor(fj);
                        d_i *= dts; d_j *= dts;
                        shade(rgb, rr.light, 1.0 - fog, s_tex[(c.n_tex * ts + trunc_i(d_i)) * ts + trunc_i(d_j)]);
                    }
                }
                if (in_wall) {
                    const double local_v = (c.half_v - (d_v + 0.5) * c.pixel_size) * cr.ratio + vision_height;
                    double d_j = text_p2 ? local_v * c.inv_text : local_v / c.text_size;
                    d_j -= floor(d_j);
                    shade(rgb, cr.light, cr.oma, s_tex[(cr.text_id * ts + cr.ti) * ts + trunc_i(dts * d_j)]);
                }
                gpx[q] = (uint32_t)rgb[0] | ((uint32_t)rgb[1] << 10) | ((uint32_t)rgb[2] << 20) | (in_wall ? (1u << 30) : 0u);
                gfid[q] = (uint8_t)fid;
                uint8_t *g8 = a.c_rgb8 + (slot * total_px + q) * 3;
                g8[0] = (uint8_t)(rgb[0] > 255 ? 255 : rgb[0]);
                g8[1] = (uint8_t)(rgb[1] > 255 ? 255 : rgb[1]);
                g8[2] = (uint8_t)(rgb[2] > 255 ? 255 : rgb[2]);
            }
    };
    // ONE loop for both orders (one call site per phase keeps the kernel's code size down):
    //   sequential (FILL, or no room for two record sets): geometry(e) by the whole CTA, barrier, pixels(e), barrier;
    //   pipelined: the first kGeoThreads threads prepare env e + 1 (record set b ^ 1) and then join the other warps, which
    //   have been painting env e (record set b) since the last barrier; the first trip only prepares.
    const bool pipe = !FILL && c.pipe;
    const int64_t stride = gridDim.x;
    int b = 0, bb = 0;
    if (!pipe && tid == 0 && (int64_t)blockIdx.x < n_items) load_blob(blockIdx.x, 0);
    if (!ROLL) {
        for (int64_t e_pix = pipe ? (int64_t)blockIdx.x - stride : (int64_t)blockIdx.x; e_pix < n_items; e_pix += stride) {
            const int64_t e_geo = pipe ? e_pix + stride : e_pix;
            if (e_geo < n_items && (!pipe || tid < kGeoThreads)) {
                // sequential: the other tile buffer was last read before the barrier that closed the previous env: prefetch into it
                geometry(e_geo, 0, pipe ? b ^ 1 : 0, pipe ? b ^ 1 : bb, tid, pipe ? kGeoThreads : (int)blockDim.x, pipe, pipe,
                         (!pipe && e_geo + stride < n_items) ? e_geo + stride : -1);
            }
            if (!pipe) {
                if (!tex_ready) { mgb_mbar_wait(&s_bar[0], 0); tex_ready = true; }
                __syncthreads();
            }
            if (e_pix >= 0) {
                if (FILL) fill_pixels(e_pix, bb);
                else pixels(e_pix, pipe ? b : 0, pipe ? b : bb, pipe);
            }
            __syncthreads();   // the record set / tile just painted from is rewritten next
            b ^= 1; bb ^= 1;   // pipelined: the set prepared in this trip is painted in the next one
        }
    } else if (FIN) {
        // the same trips over items (env, t) and, after an item whose env finished, (env, t, reset).  The pixels of an item
        // go where its record set says; whether the item just prepared is followed by its reset item is read after the
        // trip's closing barrier from the slot of this trip's tile buffer, so that every thread takes the same next item.
        int64_t e_geo = blockIdx.x;
        int t_geo = 0;
        bool pix = false;              // pipelined: the record set prepared in the previous trip is painted in this one
        while (e_geo < a.n || (pipe && pix)) {
            const bool geo = e_geo < a.n;
            const bool last_t = t_geo + 1 == a.T;
            const int64_t e_next = last_t ? e_geo + stride : e_geo;     // the next item unless e_geo finishes here
            const int gslot = pipe ? b ^ 1 : bb;                        // tile buffer of this trip's geometry
            if (geo && (!pipe || tid < kGeoThreads)) {
                geometry(e_geo, t_geo, pipe ? b ^ 1 : 0, gslot, tid, pipe ? kGeoThreads : (int)blockDim.x, pipe, pipe,
                         (!pipe && e_next < a.n) ? e_next : -1);
            }
            if (!pipe) {
                if (!tex_ready) { mgb_mbar_wait(&s_bar[0], 0); tex_ready = true; }
                __syncthreads();
            }
            if (pipe ? pix : geo) pixels(0, pipe ? b : 0, pipe ? b : bb, pipe);
            __syncthreads();
            b ^= 1; bb ^= 1;
            pix = geo;
            if (geo) {
                if (!geo_reset && s_split[gslot]) geo_reset = true;
                else { geo_reset = false; e_geo = e_next; t_geo = last_t ? 0 : t_geo + 1; }
            }
        }
    } else {
        // the same trips over items (env, t): geometry of item (e_geo, t_geo), pixels of item (e_pix, t_pix) into frame
        // t_pix * n + e_pix -- the same item (sequential) or the one before it (pipelined; none on the first trip).  Every
        // item reloads its env's tile, so the tile buffers alternate exactly as above.
        int64_t e_geo = blockIdx.x, e_pix = pipe ? -1 : e_geo;
        int t_geo = 0, t_pix = 0;
        while (e_pix < a.n) {
            const bool last_t = t_geo + 1 == a.T;
            const int64_t e_next = last_t ? e_geo + stride : e_geo;
            const int t_next = last_t ? 0 : t_geo + 1;
            if (e_geo < a.n && (!pipe || tid < kGeoThreads)) {
                geometry(e_geo, t_geo, pipe ? b ^ 1 : 0, pipe ? b ^ 1 : bb, tid, pipe ? kGeoThreads : (int)blockDim.x, pipe,
                         pipe, (!pipe && e_next < a.n) ? e_next : -1);
            }
            if (!pipe) {
                if (!tex_ready) { mgb_mbar_wait(&s_bar[0], 0); tex_ready = true; }
                __syncthreads();
            }
            if (e_pix >= 0) pixels((int64_t)t_pix * a.n + e_pix, pipe ? b : 0, pipe ? b : bb, pipe);
            __syncthreads();
            b ^= 1; bb ^= 1;
            e_pix = pipe ? e_geo : e_next; t_pix = pipe ? t_geo : t_next;
            e_geo = e_next; t_geo = t_next;
        }
    }
    if (!tex_ready && tid == 0) mgb_mbar_wait(&s_bar[0], 0);   // never leave a TMA load in flight
    if ((tid & 31) == 0) mgb_bulk_wait_read<0>();   // smem must outlive the copies; the kernel boundary flushes the writes
}

// What the compose step needs from an env after its step logic: pose slot, life bar, food presence, and the 8-bit
// signature of the foods that can show in this pose but are currently missing.
__device__ __forceinline__ EnvDyn make_dyn(const MazeConst &c, const MazeArgs &a, const uint8_t *blob, int task, const Env &s,
                                           const int32_t *eaten)
{
    const TaskHdr *th = blob_hdr(blob);
    EnvDyn d;
    const size_t pose = (size_t)task * c.n * c.n * 4 + (s.gx * c.n + s.gy) * 4 + s.ori;
    uint64_t fm[2];
    int vb = -1;
    bool have_vb = false;
    if (a.pose_rec) {                  // one record: nothing below waits for a second round trip
        const int4 *r = reinterpret_cast<const int4 *>(reinterpret_cast<const PoseRec *>(a.pose_rec) + pose);
        const int4 r0 = __ldg(r), r1 = __ldg(r + 1);
        d.slot = r0.x; vb = r0.y; have_vb = true;
        fm[0] = ((uint64_t)(uint32_t)r0.w << 32) | (uint32_t)r0.z;
        fm[1] = ((uint64_t)(uint32_t)r1.y << 32) | (uint32_t)r1.x;
    } else {
        d.slot = a.pose_index[pose];
    }
    d.task = task; d.pad = 0;
    d.present[0] = d.present[1] = 0;
    if (c.task_type == MGB_MAZE_SURVIVAL) {
        const int32_t *fint = reinterpret_cast<const int32_t *>(blob + c.off_fint);
        // batches of 8 foods: the 16 loads of a batch are issued together (one memory latency per batch, not per food)
        const int n_food = th->n_food;
        for (int f0 = 0; f0 < n_food; f0 += 8) {
            int ea[8], fi[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int f = f0 + k < n_food ? f0 + k : n_food - 1;
                ea[k] = eaten[f * a.n_pad];
                fi[k] = fint[f];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int f = f0 + k;
                if (f < n_food && ((ea[k] == kNever) || (s.steps >= ea[k] + fi[k]))) d.present[f >> 6] |= 1ull << (f & 63);
            }
        }
        int ex = trunc_i(c.lb_sx + s.life / th->max_life * c.lb_l);      // maze_discrete_3d.py:118-126
        if (ex < 0) { ex += c.res_h; if (ex < 0) ex = 0; }
        if (ex > c.res_h) ex = c.res_h;
        d.bar_end = ex;
    } else {
        d.present[0] = 1ull;             // the goal cell is pseudo food slot 0, always present (maze_base.py:59-60)
        d.bar_end = 0;
    }
    // 8-bit signature of the foods that can show in this pose but are currently missing; 0 -> the whole frame is the
    // baked "all present" frame + life bar
    if (!a.pose_rec) { fm[0] = a.c_fmask[(size_t)d.slot * 2]; fm[1] = a.c_fmask[(size_t)d.slot * 2 + 1]; }
    uint64_t miss = ((~d.present[0]) & fm[0]) | ((~d.present[1]) & fm[1]);      // fold 128 slots to (f & 7)
    d.vframe = -1; d.pad2 = 0;
    if (miss && (have_vb || a.c_vbase)) {
        if (!have_vb) vb = a.c_vbase[d.slot];
        if (vb >= 0) {
            // variant index = presence bits of the pose's foods, compacted in ascending slot order (all visible -> the
            // c_rgb8 frame, handled by miss == 0 above)
            int v = 0, bit = 0;
#pragma unroll
            for (int w = 0; w < 2; ++w) {
                uint64_t m = fm[w];
                while (m) {
                    const int f = __ffsll((long long)m) - 1;
                    m &= m - 1;
                    v |= (int)((d.present[w] >> f) & 1ull) << bit;
                    ++bit;
                }
            }
            d.vframe = vb + v;
            miss = 0;                    // the variant frame is final
        }
    }
    miss |= miss >> 32; miss |= miss >> 16; miss |= miss >> 8;
    d.pad = (int32_t)(miss & 0xFFu);
    return d;
}

// a finished env's terminal state joins the list pass of mgb_maze_step (before env_reset): the pose cache keeps its EnvDyn,
// the direct renderer everything geometry() reads
__device__ __forceinline__ void push_terminal(const MazeConst &c, const MazeArgs &a, int64_t e, int task, const uint8_t *blob,
                                              const Env &s, const int32_t *eaten)
{
    if (!a.fin_dyn) { push_terminal_state(c, a, e, s, eaten, make_float2(0.0f, 0.0f), 0.0); return; }
    const int i = atomicAdd(a.fin_count, 1);
    a.fin_env[i] = (int32_t)e;
    reinterpret_cast<EnvDyn *>(a.fin_dyn)[i] = make_dyn(c, a, blob, task, s, eaten);
}

// ---------------------------------------------------------------------------------------------------------------
// Pose cache path: step logic (one thread per env) + compose (static pose layers x current food state -> observation)
// ---------------------------------------------------------------------------------------------------------------
// DYN = false: step logic only, ahead of the direct renderer (which then runs with do_step = 0): the per-env logic is a
// chain of dependent L2 round trips that one thread of a 512-thread CTA would otherwise walk once per env, serially.
template <bool DYN>
__global__ void maze3d_logic_kernel(const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const int task = a.env2task[e];
    const uint8_t *blob = a.blobs + (int64_t)task * c.blob_bytes;
    const TaskHdr *th = blob_hdr(blob);
    const int4 ag = a.agent[e];
    Env s = {ag.x, ag.y, ag.z, ag.w, a.life[e]};
    int32_t *eaten = a.eaten + e;
    if (a.do_step) {
        double reward;
        int done;
        maze_logic(c, blob, eaten, a.n_pad, s, a.act[e], reward, done);
        a.rew[e] = reward;
        a.done[e] = (uint8_t)done;
        if (a.truncated) a.truncated[e] = maze_truncated(c, blob, s);
        if (done && a.fin_count) push_terminal(c, a, e, task, blob, s, eaten);
        if (done && a.auto_reset) env_reset(c, blob, eaten, a.n_pad, s);
        a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
        a.life[e] = s.life;
        path_store(c, a, e, s);
    }
    if (DYN) {
        const EnvDyn d = make_dyn(c, a, blob, task, s, eaten);
        reinterpret_cast<EnvDyn *>(a.dyn)[e] = d;
    }
}

// per pose slot, after the FILL render: (1) c_fmask = the food slots that can change this pose's image at all (under a
// pixel or in a crossing record); (2) c_gsig = one byte per 4-pixel group, OR of 1 << (f & 7) over the food slots f that
// can tint a pixel of the group (floor/ceiling cell under it, or a crossing span over it).  0 = never tinted.  An env
// whose missing foods have the 8-bit signature S needs the float64 path only for groups with (gsig & S) != 0.  Block b
// serves pose slot a.fill_slot[b]; int32 screens (a.c_px_all set) also start its all-present colours as the static ones.
__global__ void __launch_bounds__(256) maze3d_sig_kernel(const __grid_constant__ MazeConst c,
                                                         const __grid_constant__ MazeArgs a)
{
    const int64_t slot = a.fill_slot[blockIdx.x];
    const int V = c.res_v, total_px = c.res_h * V;
    if (a.c_px_all) {
        const uint4 *src = reinterpret_cast<const uint4 *>(a.c_px + (size_t)slot * total_px);
        uint4 *dst = reinterpret_cast<uint4 *>(a.c_px_all + (size_t)slot * total_px);
        for (int i = threadIdx.x; i < total_px / 4; i += blockDim.x) dst[i] = src[i];
    }
    const uint8_t *gfid = a.c_fid + (size_t)slot * total_px;
    const uint8_t *colhits = a.c_colhits + (size_t)slot * c.res_h;
    const HitRec *ghits = reinterpret_cast<const HitRec *>(a.c_hits) + (size_t)slot * c.res_h * c.max_hits;
    uint8_t *gsig = a.c_gsig + (size_t)slot * (total_px / 4);
    uint64_t m0 = 0, m1 = 0;
    auto note = [&](int f, uint32_t &sig) {
        if (f < 0 || f >= 128) return;
        sig |= 1u << (f & 7);
        if (f < 64) m0 |= 1ull << f; else m1 |= 1ull << (f - 64);
    };
    for (int g = threadIdx.x; g < total_px / 4; g += blockDim.x) {
        uint32_t sig = 0;
        for (int k = 0; k < 4; ++k) {
            const int q = 4 * g + k, d_h = q / V, d_v = q - d_h * V;
            const int f = gfid[q];
            if (f != 0xFF) note(f, sig);
            const HitRec *hh = ghits + (size_t)d_h * c.max_hits;
            for (int j = 0; j < colhits[d_h]; ++j)
                if (d_v >= hh[j].v_s && d_v < hh[j].v_e) note(hh[j].fid, sig);
        }
        gsig[g] = (uint8_t)sig;
    }
    for (int o = 16; o > 0; o >>= 1) { m0 |= __shfl_xor_sync(0xffffffffu, m0, o); m1 |= __shfl_xor_sync(0xffffffffu, m1, o); }
    __shared__ uint64_t s_m[256 / 32][2];
    if ((threadIdx.x & 31) == 0) { s_m[threadIdx.x >> 5][0] = m0; s_m[threadIdx.x >> 5][1] = m1; }
    __syncthreads();
    if (threadIdx.x == 0) {                  // the whole mask is written: a rebuilt slot keeps nothing of its previous pose
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) { m0 |= s_m[w][0]; m1 |= s_m[w][1]; }
        a.c_fmask[slot * 2] = m0;
        a.c_fmask[slot * 2 + 1] = m1;
    }
}

// Item i of a region kernel (see MazeArgs::region): the pose slot (pose bake) or the variant frame (a.bake_desc set) it
// stands for, -1 when the task has no such pose or frame
__device__ __forceinline__ int64_t region_item(const MazeArgs &a, int64_t i)
{
    const int64_t k = i / a.region_ext, j = i - k * a.region_ext;
    const int64_t t = a.region[k], r = t * a.region_ext + j;
    if (a.bake_desc) return j < a.task_frames[t] ? r : -1;
    return a.poses[r].x >= 0 ? r : -1;
}

// Variant frames of the region's tasks, planned on the device from c_fmask (one warp per task, block = a.region entry): a
// pose whose image depends on k foods, 1 <= k <= bits, gets the 2^k - 1 frames vbase .. vbase + 2^k - 2 (the all-visible
// one is c_rgb8[slot]), in ascending pose-slot order from the task's first frame t V.  bits is the largest <= a.var_bits
// whose frames fit the task's V frames, so a task of the table ensure_pose_cache sized V by takes a.var_bits itself.
__global__ void __launch_bounds__(32) maze3d_plan_kernel(const __grid_constant__ MazeArgs a, int32_t *vbase, BakeDesc *desc,
                                                         int32_t *task_frames)
{
    const int64_t t = a.region[blockIdx.x], S = a.pose_stride, V = a.var_stride;
    const int lane = threadIdx.x;
    auto foods = [&](int64_t j, uint64_t fm[2]) -> int {
        fm[0] = fm[1] = 0;
        if (j >= S || a.poses[t * S + j].x < 0) return 0;
        fm[0] = a.c_fmask[(t * S + j) * 2]; fm[1] = a.c_fmask[(t * S + j) * 2 + 1];
        return __popcll(fm[0]) + __popcll(fm[1]);
    };
    int64_t need[kVariantBitsMax + 1];
#pragma unroll
    for (int b = 0; b <= kVariantBitsMax; ++b) need[b] = 0;
    for (int64_t j = lane; j < S; j += 32) {
        uint64_t fm[2];
        const int k = foods(j, fm);
#pragma unroll
        for (int b = 1; b <= kVariantBitsMax; ++b)
            if (k >= 1 && k <= b) need[b] += ((int64_t)1 << k) - 1;
    }
    int bits = 0;
    int64_t frames = 0;
#pragma unroll
    for (int b = 1; b <= kVariantBitsMax; ++b) {
        int64_t s = need[b];
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (b <= a.var_bits && s <= V) { bits = b; frames = s; }     // need[] grows with b
    }
    int64_t run = t * V;
    for (int64_t j0 = 0; j0 < S; j0 += 32) {
        const int64_t j = j0 + lane;
        uint64_t fm[2];
        const int k = foods(j, fm);
        const int own = (k >= 1 && k <= bits) ? (1 << k) - 1 : 0;
        int incl = own;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        const int64_t base = run + incl - own;
        if (j < S) vbase[t * S + j] = own ? (int32_t)base : -1;
        for (int v = 0; v < own; ++v) {
            BakeDesc bd;
            bd.slot = (int32_t)(t * S + j); bd.pad = 0;
            bd.present[0] = ~fm[0]; bd.present[1] = ~fm[1];            // foods this pose never shows: irrelevant
            int bit = 0;
            for (int w = 0; w < 2; ++w) {
                uint64_t m = fm[w];
                while (m) {
                    const uint64_t low = m & (~m + 1);
                    m &= m - 1;
                    if ((v >> bit) & 1) bd.present[w] |= low;
                    ++bit;
                }
            }
            desc[base + v] = bd;
        }
        run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) task_frames[t] = (int32_t)frames;
}

// variant frames start as copies of the pose's STATIC frame (what the FILL render left in c_rgb8, before any tint is baked);
// block = region item over the tasks' variant frames
__global__ void __launch_bounds__(256) maze3d_varinit_kernel(const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a)
{
    const int64_t f = region_item(a, blockIdx.x);
    if (f < 0) return;
    const size_t frame16 = (size_t)c.res_h * c.res_v * 3 / 16;
    const BakeDesc bd = reinterpret_cast<const BakeDesc *>(a.bake_desc)[f];
    const uint4 *src = reinterpret_cast<const uint4 *>(a.c_rgb8) + (size_t)bd.slot * frame16;
    uint4 *dst = reinterpret_cast<uint4 *>(a.c_var8) + (size_t)f * frame16;
    for (size_t i = threadIdx.x; i < frame16; i += blockDim.x) dst[i] = src[i];
}

constexpr int kComposeThreads = 256;

// Screen and life-bar constants of a pose-cache frame (the bar's end column is per env: EnvDyn::bar_end)
struct FrameConst {
    int H, V, total_px;
    bool survival;               // SURVIVAL task: food values tint, the life bar is drawn
    int lb_sx, lb_sy, lb_ey;     // life bar: first column, rows [lb_sy, lb_ey)
    int px_bytes;                // bytes of one output pixel: 3 (uint8) or 12 (int32 / float32 words)
    int v_shift;                 // log2(V) when V is a power of two, else -1
};
__device__ __forceinline__ FrameConst frame_const(const MazeConst &c)
{
    FrameConst f;
    f.H = c.res_h; f.V = c.res_v; f.total_px = f.H * f.V;
    f.survival = c.task_type == MGB_MAZE_SURVIVAL;
    f.lb_sx = trunc_i(c.lb_sx); f.lb_sy = trunc_i(c.lb_sy);
    f.lb_ey = trunc_i(c.lb_sy + c.lb_w);
    if (f.lb_ey > f.V) f.lb_ey = f.V;
    f.px_bytes = c.obs_dtype == MGB_OBS_U8 ? 3 : 12;
    f.v_shift = (f.V & (f.V - 1)) == 0 ? 31 - __clz(f.V) : -1;
    return f;
}

// The cached static layers of one pose and the food values of its task
struct PoseLayers {
    const double *fval;          // food values of the task
    const uint32_t *px;          // packed colour (10 bits per channel) + in-wall flag, per pixel
    const uint8_t *fid;          // food slot under the pixel, 0xFF: none
    const uint8_t *colhits;      // transparent crossings per column
    const HitRec *hits;          // c.max_hits crossing records per column
};
__device__ __forceinline__ PoseLayers pose_layers(const MazeConst &c, const MazeArgs &a, const FrameConst &f, const EnvDyn &d)
{
    const uint8_t *blob = a.blobs + (int64_t)d.task * c.blob_bytes;
    return {reinterpret_cast<const double *>(blob + c.off_fval), a.c_px + (size_t)d.slot * f.total_px,
            a.c_fid + (size_t)d.slot * f.total_px, a.c_colhits + (size_t)d.slot * f.H,
            reinterpret_cast<const HitRec *>(a.c_hits) + (size_t)d.slot * f.H * c.max_hits};
}

template <int N>
struct PixelGroup {
    int rgb[N][3];
};
// N pixels of ONE screen column (pixel q and the N - 1 after it, rows d_v0 ..): cached static colour -> floor/ceiling
// tint -> crossings of the column -> life bar (ray_caster_utils.py:118-205, maze_discrete_3d.py:118-126).  The channel
// values are not clamped; the caller packs them.  Each crossing record of the column is loaded once for the N pixels
// (they share the column), in ascending order, so every pixel sees the blends in the reference's order.  R records are
// loaded per round trip: 4-pixel groups in the 48-register compose kernels spill with more than one in flight.
template <int N, int R>
__device__ __forceinline__ PixelGroup<N> tint_group(const MazeConst &c, const FrameConst &f, const EnvDyn &d, const PoseLayers &L,
                                                    int q, int d_h, int d_v0)
{
    static_assert(N == 1 || N == 4, "a group is one pixel or four");
    PixelGroup<N> g;
    auto &rgb = g.rgb;
    uint32_t w[N], fids;
    if constexpr (N == 4) {
        const uint4 w4 = __ldg(reinterpret_cast<const uint4 *>(L.px + q));
        w[0] = w4.x; w[1] = w4.y; w[2] = w4.z; w[3] = w4.w;
        fids = __ldg(reinterpret_cast<const uint32_t *>(L.fid + q));
    } else {
        w[0] = __ldg(L.px + q);
        fids = __ldg(L.fid + q);
    }
    const int n_hits = L.colhits[d_h];
    bool mark[N];
#pragma unroll
    for (int k = 0; k < N; ++k) {
        const int d_v = d_v0 + k, fd = (int)((fids >> (8 * k)) & 0xFFu);
        rgb[k][0] = (int)(w[k] & 1023u); rgb[k][1] = (int)((w[k] >> 10) & 1023u); rgb[k][2] = (int)((w[k] >> 20) & 1023u);
        const bool in_wall = (w[k] >> 30) & 1u;
        mark[k] = false;
        if (fd != 0xFF && ((d.present[fd >> 6] >> (fd & 63)) & 1ull)) {
            const double tv = f.survival ? __ldg(L.fval + fd) : 1.0;
            if (d_v > c.res_v / 2 ? tv > 0.01 : tv > 0) {    // floor tests > 0.01 (:119), ceiling > 0 (:150)
                if (!in_wall) blend(rgb[k], tv * 0.50 + 0.10);
                mark[k] = true;
            }
        }
    }
    if (n_hits > 0 && !(mark[0] && mark[1 % N] && mark[2 % N] && mark[3 % N])) {    // N = 1: mark[0] four times
        const int4 *hits = reinterpret_cast<const int4 *>(L.hits + (size_t)d_h * c.max_hits);
        for (int j0 = 0; j0 < n_hits; j0 += R) {                      // R records per round trip
            int4 raw[R];
#pragma unroll
            for (int u = 0; u < R; ++u) raw[u] = __ldg(hits + (j0 + u < n_hits ? j0 + u : n_hits - 1));
#pragma unroll
            for (int u = 0; u < R; ++u) {
                if (j0 + u >= n_hits) break;
                const double tf = __hiloint2double(raw[u].y, raw[u].x);
                const int v_s = (int)(int16_t)(raw[u].z & 0xFFFF), v_e = (int)(int16_t)((uint32_t)raw[u].z >> 16), fid = raw[u].w;
                if (!((d.present[fid >> 6] >> (fid & 63)) & 1ull)) continue;
#pragma unroll
                for (int k = 0; k < N; ++k)
                    if (!mark[k] && d_v0 + k >= v_s && d_v0 + k < v_e) blend(rgb[k], tf);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < N; ++k) {
        const int d_v = d_v0 + k;
        if (f.survival && d_h >= f.lb_sx && d_h < d.bar_end && d_v >= f.lb_sy && d_v < f.lb_ey) { rgb[k][0] = 255; rgb[k][1] = 0; rgb[k][2] = 0; }
    }
    return g;
}

// four pixels' channels as 12 uint8 (values above 255 clamp: MGB_OBS_U8)
__device__ __forceinline__ void pack_u8x4(const int rgb[4][3], uint32_t pk[3])
{
    pk[0] = pk[1] = pk[2] = 0u;
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            const int idx = 3 * k + b;
            pk[idx >> 2] |= (uint32_t)(rgb[k][b] > 255 ? 255 : rgb[k][b]) << (8 * (idx & 3));
        }
}

// One compose work item: pixels [q_begin, q_end) of the frame of env state d, into frame e of `obs` (bake mode: pose slot
// e of the cache).  Pixels no missing food can tint are copied from the pose's baked all-present frame; the others take
// the cached static layers through tint_group with the env's 128-bit food presence mask.  Called by all kComposeThreads
// threads of the CTA.  DEFER (rollout kernel: one CTA = one env per step): tinted groups cluster in a few columns, i.e.
// in a few threads; they are queued in s_slow (total_px / 4 entries, *s_nslow = 0 on entry) and shared out evenly once
// the copies are done.
template <bool DEFER>
__device__ __forceinline__ void compose_item(const MazeConst &c, const MazeArgs &a, const FrameConst &f, const EnvDyn &d,
                                             void *obs, int64_t e, int q_begin, int q_end, int *s_slow = nullptr,
                                             int *s_nslow = nullptr)
{
    const int V = f.V, total_px = f.total_px;
    const PoseLayers L = pose_layers(c, a, f, d);
    const int lb_ex = d.bar_end;
    uint8_t *gobs = reinterpret_cast<uint8_t *>(obs) + (size_t)e * total_px * f.px_bytes;
    if (a.bake) gobs = c.obs_dtype == MGB_OBS_U8 ? a.c_rgb8 + (size_t)e * total_px * 3 : nullptr;
    uint32_t *bake_px = a.bake && c.obs_dtype != MGB_OBS_U8 ? a.c_px_all + (size_t)e * total_px : nullptr;
    const uint32_t miss_sig = (uint32_t)d.pad & 0xFFu;

    if ((V & 3) == 0 && (total_px & 127) == 0 && (reinterpret_cast<uintptr_t>(a.bake ? (void *)a.c_rgb8 : (void *)gobs) & 15u) == 0) {
        // G consecutive 4-row groups of one column per thread and iteration (G = 4 when V % 16 == 0, else 1).
        // FAST PATH: no food that could tint the group(s) is missing -> the baked all-present pixels are final, up to the
        // life bar, which is drawn last (maze_discrete_3d.py:118-126) and simply overwrites them: uint8 copies G x 12
        // finished bytes (three 16-byte words when G = 4), int32 unpacks.  Otherwise: 16 B + 4 B in, tint_group.
        const uint8_t *gsig = a.c_gsig + (size_t)d.slot * (total_px / 4);
        const uint8_t *g8 = frame_of(a, d, (size_t)total_px * 3);
        const uint32_t *gall = a.c_px_all + (size_t)d.slot * total_px;
        bool deferred_pass = false;
        auto one_group = [&](int q, int d_h, int d_v0, bool slow) {
            if (a.bake && !slow) return;                     // bake: untinted groups already hold their final value
            if (!slow) {
                const bool bar = f.survival && d_h >= f.lb_sx && d_h < lb_ex && d_v0 + 3 >= f.lb_sy && d_v0 < f.lb_ey;
                if (c.obs_dtype == MGB_OBS_U8) {
                    const uint32_t *src = reinterpret_cast<const uint32_t *>(g8 + (size_t)q * 3);
                    uint32_t *dst = reinterpret_cast<uint32_t *>(gobs + (size_t)q * 3);
                    uint32_t b[3] = {__ldg(src), __ldg(src + 1), __ldg(src + 2)};
                    if (bar) {
                        uint8_t px[12];
                        memcpy(px, b, 12);
                        for (int k = 0; k < 4; ++k)
                            if (d_v0 + k >= f.lb_sy && d_v0 + k < f.lb_ey) { px[3 * k] = 255; px[3 * k + 1] = 0; px[3 * k + 2] = 0; }
                        memcpy(b, px, 12);
                    }
                    dst[0] = b[0]; dst[1] = b[1]; dst[2] = b[2];
                } else {
                    const uint4 w4 = __ldg(reinterpret_cast<const uint4 *>(gall + q));
                    int o[12] = {(int)(w4.x & 1023u), (int)((w4.x >> 10) & 1023u), (int)((w4.x >> 20) & 1023u),
                                 (int)(w4.y & 1023u), (int)((w4.y >> 10) & 1023u), (int)((w4.y >> 20) & 1023u),
                                 (int)(w4.z & 1023u), (int)((w4.z >> 10) & 1023u), (int)((w4.z >> 20) & 1023u),
                                 (int)(w4.w & 1023u), (int)((w4.w >> 10) & 1023u), (int)((w4.w >> 20) & 1023u)};
                    if (bar) {
                        for (int k = 0; k < 4; ++k)
                            if (d_v0 + k >= f.lb_sy && d_v0 + k < f.lb_ey) { o[3 * k] = 255; o[3 * k + 1] = 0; o[3 * k + 2] = 0; }
                    }
                    int4 *dst = reinterpret_cast<int4 *>(gobs + (size_t)q * 12);
                    if (c.obs_dtype == MGB_OBS_F32)
                        for (int k = 0; k < 12; ++k) o[k] = __float_as_int((float)o[k]);
                    dst[0] = make_int4(o[0], o[1], o[2], o[3]);
                    dst[1] = make_int4(o[4], o[5], o[6], o[7]);
                    dst[2] = make_int4(o[8], o[9], o[10], o[11]);
                }
                return;
            }
            if constexpr (DEFER) {
                if (!deferred_pass) { s_slow[atomicAdd(s_nslow, 1)] = q; return; }
            }
            const PixelGroup<4> g = tint_group<4, 1>(c, f, d, L, q, d_h, d_v0);
            const auto &rgb = g.rgb;
            if (c.obs_dtype == MGB_OBS_U8) {
                uint32_t pk[3];
                pack_u8x4(rgb, pk);
                uint32_t *dst = reinterpret_cast<uint32_t *>(gobs + (size_t)q * 3);
                dst[0] = pk[0]; dst[1] = pk[1]; dst[2] = pk[2];
            } else if (bake_px) {
                uint4 pw;
                pw.x = (uint32_t)rgb[0][0] | ((uint32_t)rgb[0][1] << 10) | ((uint32_t)rgb[0][2] << 20);
                pw.y = (uint32_t)rgb[1][0] | ((uint32_t)rgb[1][1] << 10) | ((uint32_t)rgb[1][2] << 20);
                pw.z = (uint32_t)rgb[2][0] | ((uint32_t)rgb[2][1] << 10) | ((uint32_t)rgb[2][2] << 20);
                pw.w = (uint32_t)rgb[3][0] | ((uint32_t)rgb[3][1] << 10) | ((uint32_t)rgb[3][2] << 20);
                *reinterpret_cast<uint4 *>(bake_px + q) = pw;
            } else {
                int out[12];
                for (int k = 0; k < 12; ++k) out[k] = MGB_OBS_WORD(c, rgb[k / 3][k % 3]);
                int4 *dst = reinterpret_cast<int4 *>(gobs + (size_t)q * 12);
                dst[0] = make_int4(out[0], out[1], out[2], out[3]);
                dst[1] = make_int4(out[4], out[5], out[6], out[7]);
                dst[2] = make_int4(out[8], out[9], out[10], out[11]);
            }
        };
        if ((V & 15) == 0 && c.obs_dtype == MGB_OBS_U8) {      // int32: the 4-pixel loop
            const uint32_t miss4 = miss_sig * 0x01010101u;
            for (int q = q_begin + threadIdx.x * 16; q < q_end; q += kComposeThreads * 16) {
                const int d_h = f.v_shift >= 0 ? (q >> f.v_shift) : q / V;
                const int d_v0 = q - d_h * V;
                uint32_t hit = 0;
                if (miss_sig) hit = __ldg(reinterpret_cast<const uint32_t *>(gsig + (q >> 2))) & miss4;
                const bool bar = f.survival && d_h >= f.lb_sx && d_h < lb_ex && d_v0 + 15 >= f.lb_sy && d_v0 < f.lb_ey;
                if (!hit && !bar && !a.bake && c.obs_dtype == MGB_OBS_U8) {
                    const uint4 *src = reinterpret_cast<const uint4 *>(g8 + (size_t)q * 3);
                    uint4 *dst = reinterpret_cast<uint4 *>(gobs + (size_t)q * 3);
                    const uint4 x0 = __ldg(src), x1 = __ldg(src + 1), x2 = __ldg(src + 2);
                    dst[0] = x0; dst[1] = x1; dst[2] = x2;
                    continue;
                }
#pragma unroll 1
                for (int g = 0; g < 4; ++g) one_group(q + 4 * g, d_h, d_v0 + 4 * g, ((hit >> (8 * g)) & 0xFFu) != 0);
            }
        } else {
            for (int q = q_begin + threadIdx.x * 4; q < q_end; q += kComposeThreads * 4) {
                const int d_h = f.v_shift >= 0 ? (q >> f.v_shift) : q / V;
                const int d_v0 = q - d_h * V;
                bool slow = false;
                if (miss_sig) slow = (__ldg(gsig + (q >> 2)) & miss_sig) != 0;
                one_group(q, d_h, d_v0, slow);
            }
        }
        if constexpr (DEFER) {
            __syncthreads();
            deferred_pass = true;
            for (int i = threadIdx.x; i < *s_nslow; i += kComposeThreads) {
                const int q = s_slow[i];
                const int d_h = f.v_shift >= 0 ? (q >> f.v_shift) : q / V;
                one_group(q, d_h, q - d_h * V, true);
            }
        }
    } else {
        for (int q = q_begin + threadIdx.x; q < q_end; q += kComposeThreads) {
            const int d_h = q / V, d_v = q - d_h * V;
            const PixelGroup<1> g = tint_group<1, 4>(c, f, d, L, q, d_h, d_v);
            const auto &rgb = g.rgb;
            if (c.obs_dtype == MGB_OBS_U8) {
                for (int k = 0; k < 3; ++k) gobs[(size_t)q * 3 + k] = (uint8_t)(rgb[0][k] > 255 ? 255 : rgb[0][k]);
            } else {
                int32_t *o = reinterpret_cast<int32_t *>(gobs) + (size_t)q * 3;
                o[0] = MGB_OBS_WORD(c, rgb[0][0]); o[1] = MGB_OBS_WORD(c, rgb[0][1]); o[2] = MGB_OBS_WORD(c, rgb[0][2]);
            }
        }
    }
}

// Work item = (env, image slice), composed by compose_item.
// REGION (pose-cache build, bake mode): items are region items (MazeArgs::region) that skip the poses / frames a task
// does not have; the step's instantiation stays the plain one.
template <bool REGION>
__global__ void __launch_bounds__(kComposeThreads, 5) maze3d_compose_kernel(const __grid_constant__ MazeConst c,
                                                                         const __grid_constant__ MazeArgs a)
{
    // persistent CTAs: work item = (env, one of kParts slices of its image); grid = resident CTA count, so there is
    // no partial last wave (1024 envs as 1024 CTAs ran 1.15 waves = almost twice the time of one)
    const int kParts = a.do_parts;      // 1..4 image slices per env, chosen by the host so that items >> resident CTAs
    const FrameConst f = frame_const(c);
    const int total_px = f.total_px;
    // slice boundaries stay 128-pixel aligned; the slices cover the frame even when it has fewer pixels than slices
    const int part_px = ((total_px + kParts - 1) / kParts + 127) / 128 * 128;
  // list pass of mgb_maze_step (final_obs set): item = (terminal list entry, slice), frame into final_obs[fin_env[entry]]
  const int64_t n_items = (a.final_obs ? (int64_t)*a.fin_count : a.n) * kParts;
  // bake mode (pose-cache build): item = pose slot, every food present, no life bar, tintable groups only
  auto fetch = [&](int64_t idx) -> EnvDyn {
      if (!a.bake) return reinterpret_cast<const EnvDyn *>(a.dyn)[idx];
      EnvDyn b;
      if (REGION) {
          idx = region_item(a, idx);
          if (idx < 0) { b.slot = 0; b.task = 0; return b; }     // skipped by the loop below
      }
      b.slot = (int32_t)idx; b.bar_end = 0; b.present[0] = b.present[1] = ~0ull; b.pad = 0xFF; b.vframe = -1; b.pad2 = 0;
      if (a.bake_desc) {               // variant frames: item = frame, its pose slot and presence mask come from the descriptor
          const BakeDesc bd = reinterpret_cast<const BakeDesc *>(a.bake_desc)[idx];
          b.slot = bd.slot; b.present[0] = bd.present[0]; b.present[1] = bd.present[1];
      }
      b.task = a.poses[b.slot].x;
      return b;
  };
  EnvDyn d_next;
  if ((int64_t)blockIdx.x < n_items) d_next = fetch(blockIdx.x / kParts);
  for (int64_t item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int64_t entry = item / kParts;
    const int part = (int)(item - entry * kParts);
    const int64_t e = REGION ? region_item(a, entry) : (a.final_obs ? (int64_t)a.fin_env[entry] : entry);
    const int q_begin = part * part_px, q_end = (part + 1) * part_px < total_px ? (part + 1) * part_px : total_px;
    // software pipeline: the next item's EnvDyn (-> pose slot -> every address below) is requested now, so the
    // dependent-load bubble at the start of an item overlaps this item's pixels
    const EnvDyn d = d_next;
    if (item + gridDim.x < n_items) d_next = fetch((item + gridDim.x) / kParts);
    if (q_begin >= total_px || (REGION && e < 0)) continue;
    compose_item<false>(c, a, f, d, a.obs, e, q_begin, q_end);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Fused single-step kernel of the pose-cache path (uint8 frames): step logic + observation in ONE launch, the frame moved by
// the TMA engine.  One CTA per env: thread 0 runs the step logic (action, evaluation rule, auto-reset, pose-cache lookup) and
// immediately issues bulk copies (cp.async.bulk + mbarrier, 12 KB chunks) of the pose's baked all-present frame into shared
// memory; as each chunk lands the CTA patches, in shared memory, the few 4-pixel groups a currently missing food can tint
// (tint_group: float64 blend of the cached static layers, as in the compose kernel) and the life bar, and one bulk store
// sends the chunk to `obs`.  The 49 KB of a frame are in flight without passing through registers (the compose kernel's 256
// threads of dependent 16-byte loads were 48 % long-scoreboard stalls), the separate logic launch and its EnvDyn round trip
// through global memory are gone, and four CTAs per SM overlap one env's logic latency with the others' copies.
// Reference: maze_discrete_3d.py:51-81,113-127, maze_base.py:65-95, ray_caster_utils.py:66-209 (via the cached layers).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kStepThreads = 128;
constexpr int kStepChunkPx = 4096;          // pixels per bulk copy: 12 KB of uint8 RGB

constexpr int kStepBatch = 16;              // envs whose step logic one CTA runs side by side before moving their frames
constexpr int kStepSlots = 8;               // 12 KB chunk slots of a CTA's shared-memory ring
constexpr int kStepSlack = 3;               // bulk stores that may still be reading their slot before it is handed back

template <bool REC>          // path recording on (a.path set): without it the kernel neither tests a.path nor stores
__global__ void __launch_bounds__(kStepThreads, 2) maze3d_step_kernel(const __grid_constant__ MazeConst c,
                                                                      const __grid_constant__ MazeArgs a)
{
    // Two CTAs per SM; CTA j owns the envs j, j + G, j + 2G, ... (G = grid size).  Per pass of up to kStepBatch envs:
    //  (1) threads 0..B-1 run the step logic of the B envs SIDE BY SIDE (each is a chain of ~4 dependent L2 round trips:
    //      one chain per frame would cost more than the frame's copy), leaving B EnvDyn records + frame pointers in shared memory;
    //  (2) the B frames stream, 12 KB chunk by chunk, through a ring of kStepSlots shared-memory slots.  Warp 1's lane 0 only
    //      ISSUES bulk loads, up to kStepSlots chunks ahead, as the consumer hands slots back through their `empty`
    //      mbarriers; warp 0 only consumes: waits for chunk u, draws the life bar into it, sends it to `obs` with one bulk
    //      store and -- once the store of chunk u - kStepSlack has left its slot -- releases that slot.  Loads and stores stay
    //      in flight across frame boundaries.  Warps 0, 2, 3 (named barrier 1, 96 threads) tint the rare frames that still need
    //      float64 blends (poses whose image depends on more foods than have variant frames).
    // The frame move is HBM-bound (every frame is read once and written once), so the step costs launch gap + logic + the
    // time HBM needs to move the frames.
    extern __shared__ __align__(128) uint8_t s_ring[];           // kStepSlots x 12 KB
    // frames of a pass: [0, B) the pass's observations; [B, B + terminal count) with final_obs, the terminal frames of the
    // pass's finished envs (their EnvDyn taken before env_reset), moved through the same ring into final_obs
    __shared__ EnvDyn s_dyn[2 * kStepBatch];
    __shared__ const uint8_t *s_src[2 * kStepBatch];             // finished frame each observation starts from
    __shared__ uint8_t *s_dst[2 * kStepBatch];                   // where a terminal frame goes
    __shared__ int s_nterm[2];                                   // terminal frames of the pass; by pass parity, so that
                                                                 // the next pass's count is cleared while this one is read
    __shared__ __align__(8) uint64_t s_bar[kStepSlots];
    __shared__ __align__(8) uint64_t s_empty[kStepSlots];
    __shared__ int s_nslow;
    __shared__ uint16_t s_slow[1024];                            // queued tinted groups of one chunk (group index in the chunk)
    const int n_chunks = (c.res_h * c.res_v + kStepChunkPx - 1) / kStepChunkPx;
    const FrameConst f = frame_const(c);
    const int V = f.V, total_px = f.total_px;
    const uint32_t frame_bytes = (uint32_t)total_px * 3u;
    const int tid = threadIdx.x, lane = tid & 31;
    const bool warp0 = tid < 32;
    if (tid == 0) {
        for (int k = 0; k < kStepSlots; ++k) { mgb_mbar_init(&s_bar[k], 1); mgb_mbar_init(&s_empty[k], 1); }
        mgb_fence_mbar_init();
        s_nslow = 0;
        s_nterm[0] = s_nterm[1] = 0;
    }
    __syncthreads();
    uint32_t g0 = 0;                                             // chunks this CTA has moved in earlier passes (ring position)
    int pass = 0;
    for (int64_t base = blockIdx.x; base < a.n; base += (int64_t)gridDim.x * kStepBatch, ++pass) {
        const int64_t left = (a.n - base + gridDim.x - 1) / gridDim.x;
        const int B = (int)(left < kStepBatch ? left : kStepBatch);
        // ---- (1) step logic of the pass's envs, one thread each (what maze3d_logic_kernel does for the two-kernel path)
        if (tid < B) {
            const int64_t e = base + (int64_t)tid * gridDim.x;
            const int task = a.env2task[e];
            const uint8_t *blob = a.blobs + (int64_t)task * c.blob_bytes;
            const int4 ag = a.agent[e];
            Env s = {ag.x, ag.y, ag.z, ag.w, a.life[e]};
            int32_t *eaten = a.eaten + e;
            if (a.do_step) {
                double reward;
                int done;
                maze_logic(c, blob, eaten, a.n_pad, s, a.act[e], reward, done);
                a.rew[e] = reward;
                a.done[e] = (uint8_t)done;
                if (a.truncated) a.truncated[e] = maze_truncated(c, blob, s);
                if (done && a.final_obs) {                        // the terminal state still has its food stamps
                    const EnvDyn td = make_dyn(c, a, blob, task, s, eaten);
                    const int j = B + atomicAdd(&s_nterm[pass & 1], 1);
                    s_dyn[j] = td;
                    s_src[j] = frame_of(a, td, frame_bytes);
                    s_dst[j] = reinterpret_cast<uint8_t *>(a.final_obs) + (size_t)e * frame_bytes;
                }
                if (done && a.auto_reset) env_reset(c, blob, eaten, a.n_pad, s);
                a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
                a.life[e] = s.life;
                if (REC) path_store(c, a, e, s);
            }
            const EnvDyn dd = make_dyn(c, a, blob, task, s, eaten);
            s_dyn[tid] = dd;
            s_src[tid] = frame_of(a, dd, frame_bytes);
        }
        __syncthreads();
        const int J = a.final_obs ? B + s_nterm[pass & 1] : B;    // frames of this pass
        const int M = J * n_chunks;                               // chunks of this pass
        if (a.final_obs && tid == 0) s_nterm[(pass + 1) & 1] = 0;  // last read in the previous pass, before its closing barrier
        const bool producer = (tid >> 5) == 1;
        const int t96 = tid < 32 ? tid : tid - 32;                 // index inside the consumer group (warps 0, 2, 3)
        if (producer) {
            if (lane == 0) {
                int it = 0, k = 0;
                for (int u = 0; u < M; ++u) {
                    const uint32_t gu = g0 + (uint32_t)u;
                    const int slot = (int)(gu % kStepSlots);
                    const uint32_t use = gu / kStepSlots;           // how often this slot has been filled before
                    if (use > 0) mgb_mbar_wait(&s_empty[slot], (use - 1) & 1u);
                    const uint32_t off = (uint32_t)k * kStepChunkPx * 3u;
                    const uint32_t bytes = frame_bytes - off < kStepChunkPx * 3u ? frame_bytes - off : kStepChunkPx * 3u;
                    mgb_mbar_expect_tx(&s_bar[slot], bytes);
                    mgb_bulk_load(s_ring + (size_t)slot * (kStepChunkPx * 3), s_src[it] + off, bytes, &s_bar[slot]);
                    if (++k == n_chunks) { k = 0; ++it; }
                }
            }
        } else {
        for (int it = 0; it < J; ++it) {
            asm volatile("bar.sync 1, 96;" ::: "memory");          // frame boundary: nobody runs more than a frame ahead of warp 0
            const EnvDyn d = s_dyn[it];
            const uint32_t miss_sig = (uint32_t)d.pad & 0xFFu;     // != 0: some groups need the float64 path (uniform)
            uint8_t *gobs = it < B ? reinterpret_cast<uint8_t *>(a.obs) + (size_t)(base + (int64_t)it * gridDim.x) * frame_bytes
                                   : s_dst[it];
            if (!warp0 && !miss_sig) continue;
            const PoseLayers L = pose_layers(c, a, f, d);
            const uint8_t *gsig = a.c_gsig + (size_t)d.slot * (total_px / 4);
            const uint32_t miss4 = miss_sig * 0x01010101u;
            for (int k = 0; k < n_chunks; ++k) {
                const int u = it * n_chunks + k;
                const uint32_t gu = g0 + (uint32_t)u;
                const int slot = (int)(gu % kStepSlots);
                const uint32_t parity = (gu / kStepSlots) & 1u;
                uint8_t *s_chunk = s_ring + (size_t)slot * (kStepChunkPx * 3);
                const int q0 = k * kStepChunkPx, q1 = q0 + kStepChunkPx < total_px ? q0 + kStepChunkPx : total_px;
                const uint32_t off = (uint32_t)q0 * 3u, bytes = (uint32_t)(q1 - q0) * 3u;
                if (miss_sig) {
                    // whole CTA: queue the chunk's tinted groups (they cluster in a few columns) ...
                    for (int g4 = (q0 >> 4) + t96; g4 < (q1 >> 4); g4 += 96) {
                        uint32_t hit = __ldg(reinterpret_cast<const uint32_t *>(gsig) + g4) & miss4;
                        while (hit) {
                            const int g = (__ffs(hit) - 1) >> 3;
                            hit &= ~(0xFFu << (8 * g));
                            s_slow[atomicAdd(&s_nslow, 1)] = (uint16_t)(((g4 << 2) + g) - (q0 >> 2));
                        }
                    }
                    asm volatile("bar.sync 1, 96;" ::: "memory");
                    const int n_slow = s_nslow;
                    mgb_mbar_wait(&s_bar[slot], parity);
                    // ... and share them out evenly: float64 blends of the cached static layers over the baked pixels
                    for (int i = t96; i < n_slow; i += 96) {
                        const int q = q0 + 4 * (int)s_slow[i];
                        const int d_h = f.v_shift >= 0 ? (q >> f.v_shift) : q / V;
                        const PixelGroup<4> g = tint_group<4, 4>(c, f, d, L, q, d_h, q - d_h * V);
                        uint32_t pk[3];
                        pack_u8x4(g.rgb, pk);
                        uint32_t *dst = reinterpret_cast<uint32_t *>(s_chunk + (size_t)(q - q0) * 3);
                        dst[0] = pk[0]; dst[1] = pk[1]; dst[2] = pk[2];
                    }
                    mgb_fence_proxy_async();
                    asm volatile("bar.sync 1, 96;" ::: "memory");  // tints done before the bar is drawn over them / the store
                    if (tid == 0) s_nslow = 0;
                }
                if (warp0) {
                    if (!miss_sig) mgb_mbar_wait(&s_bar[slot], parity);
                    // life bar columns inside this chunk (drawn last, maze_discrete_3d.py:118-126)
                    const int h0 = q0 / V, h1 = (q1 + V - 1) / V;      // columns [h0, h1) intersect the chunk
                    const int bh0 = f.lb_sx > h0 ? f.lb_sx : h0, bh1 = d.bar_end < h1 ? d.bar_end : h1;
                    if (f.survival && bh0 < bh1 && f.lb_sy < f.lb_ey) {
                        // one lane per column, rows walked in order: no integer division on the warp that feeds the ring
                        for (int d_h = bh0 + lane; d_h < bh1; d_h += 32) {
                            const int qc = d_h * V - q0;                // the column's first pixel, relative to the chunk
                            int v0 = f.lb_sy, v1 = f.lb_ey;             // rows whose pixel lies inside [q0, q1)
                            if (qc + v0 < 0) v0 = -qc;
                            if (qc + v1 > q1 - q0) v1 = q1 - q0 - qc;
                            uint8_t *px = s_chunk + (size_t)(qc + v0) * 3;
                            for (int d_v = v0; d_v < v1; ++d_v, px += 3) { px[0] = 255; px[1] = 0; px[2] = 0; }
                        }
                        mgb_fence_proxy_async();
                    }
                    __syncwarp();
                    if (lane == 0) {
                        mgb_bulk_store(gobs + off, s_chunk, bytes);
                        mgb_bulk_commit();
                        if (u >= kStepSlack) {
                            mgb_bulk_wait_read<kStepSlack>();      // the store of chunk u - 3 has left its slot: hand it back
                            mgb_mbar_arrive(&s_empty[(int)((gu - kStepSlack) % kStepSlots)]);
                        }
                    }
                }
            }
        }
        if (tid == 0) {                                            // the pass's last stores: wait for them, release their slots
            mgb_bulk_wait_read<0>();
            for (int u = (M > kStepSlack ? M - kStepSlack : 0); u < M; ++u)
                mgb_mbar_arrive(&s_empty[(int)((g0 + (uint32_t)u) % kStepSlots)]);
        }
        }
        g0 += (uint32_t)M;
        __syncthreads();                                           // s_dyn is rewritten by the next pass
    }
    if (tid == 0) mgb_bulk_wait_read<0>();       // shared memory must outlive the copies
}

// T MetaMazeDiscrete3D steps in one launch (pose-cache path): one CTA per env; thread 0 runs the step logic and leaves the
// env's EnvDyn in shared memory, then the whole CTA composes frame t straight into obs[t][env].  No logic launch, no
// EnvDyn round trip through global memory, and the logic of one env overlaps the pixels of the others on the SM.
// FIN (final_obs / truncated): thread 0 also stores the truncation byte of every (t, env) and, for an env that
// finished at step t, publishes the EnvDyn of its terminal state in a second slot -- both before env_reset, which clears the
// food stamps the terminal frame still shows.  The CTA then composes that frame into final_obs + (t n + env) frame, a
// barrier later the usual observation: one compose_item per pass, one deferred-tint queue.
// EXP (mgb_maze_rollout_expert): thread 0 takes act[t] when given, else the expert's action (expert_action) on the state
// it holds before step t, and stores that state's mask into x.out [T][n].
template <bool FIN, bool EXP = false>
__global__ void __launch_bounds__(kComposeThreads, 5) maze3d_rollout_kernel(const __grid_constant__ MazeConst c,
                                                                            const __grid_constant__ MazeArgs a,
                                                                            const __grid_constant__ MazeExpertOr<EXP> x)
{
    __shared__ EnvDyn s_dyn;
    __shared__ int s_nslow;
    __shared__ EnvDyn s_tdyn;                           // FIN: the terminal state's EnvDyn ...
    __shared__ int s_term;                              // ... valid when 1 (done and final_obs wanted)
    extern __shared__ int s_slow[];                     // total_px / 4 entries: queued tinted groups of the current frame
    const FrameConst f = frame_const(c);
    const uint2 akey = make_uint2((uint32_t)a.act_seed, (uint32_t)(a.act_seed >> 32));
    for (int64_t env = blockIdx.x; env < a.n; env += gridDim.x) {
        const int task = a.env2task[env];
        const uint8_t *eblob = a.blobs + (int64_t)task * c.blob_bytes;
        int32_t *eaten = a.eaten + env;
        Env s = {0, 0, 0, 0, 0.0};
        if (threadIdx.x == 0) {
            const int4 ag = a.agent[env];
            s.gx = ag.x; s.gy = ag.y; s.ori = ag.z; s.steps = ag.w; s.life = a.life[env];
        }
        const int64_t genv = a.env_base + env;
        for (int t = 0; t < a.T; ++t) {
            if (threadIdx.x == 0) {
                int action;
                if constexpr (EXP) {
                    const uint8_t m = expert_mask(c, x.mask, task, s);
                    if (a.act) action = a.act[(int64_t)t * a.n + env];
                    else {
                        action = expert_action(x, m, genv, a.t_base + (uint32_t)t);
                        if (a.act_out) a.act_out[(int64_t)t * a.n + env] = action;
                    }
                    if (x.out) x.out[(int64_t)t * a.n + env] = m;
                } else if (a.act) action = a.act[(int64_t)t * a.n + env];
                else {
                    const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32),
                                                                 a.t_base + (uint32_t)t, MGB_STREAM_ACTION), akey);
                    action = (int)(r.x >> 30);
                    if (a.act_out) a.act_out[(int64_t)t * a.n + env] = action;
                }
                double reward;
                int done;
                maze_logic(c, eblob, eaten, a.n_pad, s, action, reward, done);
                if (FIN) {
                    if (a.truncated) a.truncated[(int64_t)t * a.n + env] = maze_truncated(c, eblob, s);
                    s_term = done && a.final_obs;
                    if (done && a.final_obs) s_tdyn = make_dyn(c, a, eblob, task, s, eaten);
                }
                if (done && a.auto_reset) env_reset(c, eblob, eaten, a.n_pad, s);
                path_store(c, a, env, s);
                if (a.rew) a.rew[(int64_t)t * a.n + env] = reward;
                if (a.done) a.done[(int64_t)t * a.n + env] = (uint8_t)done;
                s_dyn = make_dyn(c, a, eblob, task, s, eaten);
                s_nslow = 0;
            }
            __syncthreads();
            if (FIN) {
                // pass 0: the terminal frame (finished envs only), pass 1: the observation; both decisions are CTA-uniform
                const bool term = s_term != 0;
                for (int pass = term ? 0 : 1; pass < 2; ++pass) {
                    void *dst = pass == 0 ? a.final_obs : a.obs;
                    if (!dst) continue;
                    if (pass == 1 && term) {                          // the queue of pass 0 has been read by every thread
                        __syncthreads();
                        if (threadIdx.x == 0) s_nslow = 0;
                        __syncthreads();
                    }
                    const EnvDyn d = pass == 0 ? s_tdyn : s_dyn;
                    compose_item<true>(c, a, f, d, dst, (int64_t)t * a.n + env, 0, f.total_px, s_slow, &s_nslow);
                }
            } else if (a.obs) {
                const EnvDyn d = s_dyn;
                compose_item<true>(c, a, f, d, a.obs, (int64_t)t * a.n + env, 0, f.total_px, s_slow, &s_nslow);
            }
            __syncthreads();                                          // s_dyn is rewritten by the next step
        }
        if (threadIdx.x == 0) {
            a.agent[env] = make_int4(s.gx, s.gy, s.ori, s.steps);
            a.life[env] = s.life;
        }
    }
}

// Pose-independent part of the floor/ceiling geometry: eff(d_h, d_v) = distance(d_v) / cos_hp(d_h)
// (ray_caster_utils.py:97-104,131-138) depends only on the screen, the optics and the two heights of a task, so it is
// tabulated once per (agent_height, wall_height) class with the SAME float64 division the renderer would execute.
__global__ void maze_efftab_kernel(const __grid_constant__ MazeConst c, const float *coltab, const double *cls_heights,
                                   int n_cls, double *efftab, double *fogtab)
{
    const int H = c.res_h, V = c.res_v;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (int64_t)n_cls * H * V) return;
    const int k = (int)(idx / ((int64_t)H * V));
    const int q = (int)(idx - (int64_t)k * H * V);
    const int d_h = q / V, d_v = q - d_h * V;
    const double vision_height = cls_heights[2 * k], ceil_height = cls_heights[2 * k + 1];
    double distance = 0.0;
    if (d_v > V / 2) {
        const double v_screen = (d_v + 0.5) * c.pixel_size - c.half_v;
        distance = vision_height / v_screen * c.l_focal;
    } else if (d_v < V / 2) {
        const double v_screen = c.half_v - (d_v + 0.5) * c.pixel_size;
        distance = (ceil_height - vision_height) / v_screen * c.l_focal;
    }
    const double eff = distance / (double)coltab[d_h];     // cos_hp does not depend on the heading: use heading 0
    efftab[idx] = eff;
    // the fog weight of that distance (ray_caster_utils.py:99,133), the expression the renderer evaluates when it has no table
    fogtab[idx] = eff > 0.4999 * c.max_vision ? fmin(1.0, fmax(2.0 * eff / c.max_vision - 1.0, 0.0)) : 0.0;
}

__global__ void maze_state_kernel(MazeArgs a, int32_t *agent_out, double *life_out)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const int4 ag = a.agent[e];
    agent_out[4 * e + 0] = ag.x; agent_out[4 * e + 1] = ag.y; agent_out[4 * e + 2] = ag.z; agent_out[4 * e + 3] = ag.w;
    if (life_out) life_out[e] = a.life[e];
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// handle + C ABI
// ---------------------------------------------------------------------------------------------------------------
struct MazeFinal {                 // the terminal list of mgb_maze_step (MazeArgs::fin_*, 3-D kinds)
    MgbDev<int32_t> count, env, task, eaten;
    MgbDev<EnvDyn> dyn;
    MgbDev<int4> agent;
    MgbDev<double> life, cori;
    MgbDev<float2> cpos;
};

struct MazeTasks {                 // what mgb_maze_set_task sizes by its table; the terminal list too, so that step_ex can be captured
    MgbDev<uint8_t> blobs;
    MgbDev<int32_t> eaten;
    MgbDev<double> efftab, fogtab;
    MazeFinal fin;
};

struct MazePoseCache {             // built by ensure_pose_cache (MazeArgs describes each table)
    MgbDev<int4> poses;
    MgbDev<int32_t> pose_index, c_vbase;
    MgbDev<uint32_t> c_px, c_px_all;
    MgbDev<uint8_t> c_fid, c_colhits, c_rgb8, c_gsig, c_var8;
    MgbDev<uint64_t> c_fmask;
    MgbDev<HitRec> c_hits;
    MgbDev<EnvDyn> dyn;
    MgbDev<BakeDesc> bake_desc;
    MgbDev<int32_t> task_frames;   // [n_tasks] variant frames of each task slot (maze3d_plan_kernel)
    MgbDev<PoseRec> pose_rec;      // built after the variant frames
};

struct MazeStage {                 // one half of the double-buffered staging of mgb_maze_update_tasks
    MgbPinned<uint8_t> host;
    MgbDev<uint8_t> dev;
    size_t bytes = 0;
    MgbEvent copied;               // recorded after the copy from `host`
};

struct mgb_maze {
    int device = 0;
    int64_t n = 0, n_pad = 0, env_base = 0;
    mgb_maze_cfg cfg;
    MazeConst c;
    MgbDev<int4> agent;
    MgbDev<double> life;
    MgbDev<int32_t> env2task;
    MazeTasks tasks;
    MgbDev<uint32_t> tex;
    MgbDev<float> coltab;
    MgbDev<float2> cpos;           // continuous maze pose
    MgbDev<double> cori, coltab_d;
    // pose cache
    int render_pipe = 1;           // MGB_MAZE_RENDER_PIPE=0: direct renderer without the geometry / pixel software pipeline
    int fused_step = 1;            // MGB_MAZE_FUSED_STEP=0: logic kernel + compose kernel instead of maze3d_step_kernel
    size_t step_smem_set = 0, m2d_smem_set = 0;
    int cache_enabled = 1;         // MGB_MAZE_CACHE=0 disables (direct renderer only)
    int tex_max = 255;             // brightest channel value of the loaded textures
    double cache_budget_gb = 24.0; // MGB_MAZE_CACHE_GB
    bool cache_ready = false, cache_dirty = true;
    int64_t n_poses = 0;
    MazePoseCache cache;
    MgbDev<uint32_t> task_epoch;              // [n_pad] how often each env's task has been resampled on the device
    int32_t trial_k = 0;                      // mgb_maze_set_episodes_per_task: episodes per maze (0: not a trial handle)
    MgbDev<uint32_t> task_count;              // trial handle: [n_pad] episodes each env has finished on its current maze
    bool slot_per_env = false;                // env2task is injective: every env owns its task-table slot
    MgbDev<uint8_t> task_flags;               // [n_tasks] scratch of mgb_maze_update_tasks
    std::vector<double> cls_heights;          // eff-table classes of the current task table
    double min_cell = 0.0;                    // smallest cell_size of the table (bounds the crossings a ray can record)
    MazeStage stage[2];
    int stage_next = 0;
    int variant_bits_used = 0;
    bool var_planned = false;      // the last build read c_fmask back and planned variant frames (cache_info reports them)
    double cache_bytes = 0.0;
    int variant_bits = 7;          // MGB_MAZE_VARIANT_BITS: poses that depend on <= this many foods get all 2^k frames (0 = off)
    MgbDev<uint8_t> hit_scratch;
    size_t hit_scratch_bytes = 0;
    // pose list of the cache, slot-strided: task slot t owns the pose slots [t S, t S + S), S = pose_stride (4 x the most
    // free cells of a task); unused slots hold task -1.  var_stride V: variant frames per task slot, fixed by the first build
    std::vector<int4> host_poses;             // [n_tasks * S]
    std::vector<int32_t> host_pose_index;     // [n_tasks][n * n * 4] -> pose slot or -1
    std::vector<int32_t> task_poses;          // [n_tasks] used pose slots of each task
    int pose_stride = 0;
    int64_t var_stride = 0;
    int n_tasks = 0;
    int auto_reset = 0;
    bool has_task = false, has_tex = false;
    size_t smem3d = 0;
    int render_attr_set[16] = {};            // maze3d_kernel<false / true / rollout / rollout with terminal frames>, then the
                                             // two rollouts with resampling (4 + ...), then the expert rollouts (8 + ...):
                                             // shared-memory opt-in raised by this handle
    int compose_ctas_per_sm = 0;       // occupancy of maze3d_compose_kernel (queried once per handle)
    int num_sms = 0;
    int64_t launches = 0;
    uint32_t t_base = 0;
    uint64_t fp_tex = 0;                      // fingerprint of the loaded textures (mgb_maze_fingerprint)
    std::vector<uint64_t> slot_fp;            // fingerprint of every task-table slot as set_task / update_tasks wrote it
    MgbMirrors mir = {};         // mgb_maze_set_mirrors
    MgbMirrorWindow mir_win;     // mgb_maze_set_mirror_window
    MgbDev<char2> path;            // mgb_maze_set_path: [max_steps + 1][n_pad] recorded cells, empty when not recording
    bool expert = false;           // mgb_maze_set_expert: the tables below follow every change of the task table, so
                                   // the rollouts that draw new mazes inside the launch refuse an expert handle
    MgbDev<uint16_t> exp_dist;     // [n_tasks][planes][n][n] (maze_expert_kernel)
    MgbDev<uint8_t> exp_mask;      // [n_tasks][planes][n][n]
};

// The refusal of in-launch resampling on an expert handle: the kernels that draw a new maze into a slot cannot rebuild
// the slot's expert tables, which would then describe the old maze
static const char *const kExpertNoInLaunchResampling =
    "in-launch resampling is not available on an expert handle (its tables would keep the old mazes): call "
    "mgb_maze_resample_tasks between launches instead";

// Rebuild the expert tables of the task slots a table change touched, on st (maze_expert_kernel's items, map, sel, row)
static int build_expert(mgb_maze *h, int64_t count, const int32_t *map, const uint8_t *sel, const int64_t *row,
                        int64_t n_rec, cudaStream_t st)
{
    if (!h->expert) return MGB_OK;
    maze_expert_kernel<<<(unsigned)((count + kExpertWarps - 1) / kExpertWarps), 32 * kExpertWarps, 0, st>>>(
        h->c, h->tasks.blobs.get(), count, map, sel, row, n_rec, h->exp_dist.get(), h->exp_mask.get());
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// entries of one env's path record: an episode ends at steps <= max_steps
static int64_t path_cap(const mgb_maze *h) { return (int64_t)h->c.max_steps + 1; }

static size_t maze3d_smem_bytes(const MazeConst &c, bool fill, bool rs = false)
{
    auto up = [](size_t x, size_t a) { return (x + a - 1) / a * a; };
    size_t off = 0;
    off = up(off + (size_t)(c.n_tex + 1) * c.ts * c.ts * 4, 128);
    const int nbuf = (!fill && c.pipe) ? 2 : 1;
    off = up(off + c.blob_bytes, 128);
    off = up(off + c.blob_bytes, 128);
    for (int b = 0; b < nbuf; ++b) {
        off = up(off + (size_t)c.n * c.n * 8, 128);
        off = up(off + (size_t)c.res_h * sizeof(ColRec), 128);
        off = up(off + (size_t)c.res_v * sizeof(RowRec), 128);
        if (!c.hits_in_global) off = up(off + (size_t)c.res_h * c.max_hits * sizeof(HitRec), 128);
    }
    off = up(off + (size_t)c.res_v * 8, 128);
    const size_t px = c.obs_dtype == MGB_OBS_U8 ? 3 : 12;
    off = up(off + (size_t)(kRenderThreads / 32) * (c.obs_dtype == MGB_OBS_U8 ? 2 : 1) * c.run_px * px, 128);
    off += 32 + 128 + 16;
    if (rs) off += sampler_ws_bytes(c.n);      // maze3d_kernel<.., RS>: one warp's sampler workspace
    return off;
}

// The tables of a pose cache, into args filled before ensure_pose_cache (re)built it
static void bind_pose_cache(const MazePoseCache &pc, MazeArgs &a)
{
    a.poses = pc.poses.get(); a.pose_index = pc.pose_index.get(); a.pose_rec = pc.pose_rec.get(); a.c_px = pc.c_px.get(); a.c_fid = pc.c_fid.get();
    a.c_colhits = pc.c_colhits.get(); a.c_hits = pc.c_hits.get(); a.dyn = pc.dyn.get(); a.c_rgb8 = pc.c_rgb8.get(); a.c_gsig = pc.c_gsig.get();
    a.c_px_all = pc.c_px_all.get(); a.c_fmask = pc.c_fmask.get(); a.c_vbase = pc.c_vbase.get(); a.c_var8 = pc.c_var8.get();
}

// Kernel arguments of the handle's state; every per-call field is zero
static MazeArgs maze_args(const mgb_maze *h)
{
    MazeArgs a;
    memset(&a, 0, sizeof(a));
    a.n = h->n; a.n_pad = h->n_pad; a.env_base = h->env_base;
    a.agent = h->agent.get(); a.life = h->life.get(); a.eaten = h->tasks.eaten.get(); a.env2task = h->env2task.get(); a.blobs = h->tasks.blobs.get();
    a.tex = h->tex.get(); a.coltab = h->coltab.get(); a.efftab = h->tasks.efftab.get(); a.fogtab = h->tasks.fogtab.get(); a.auto_reset = h->auto_reset;
    a.cpos = h->cpos.get(); a.cori = h->cori.get(); a.coltab_d = h->coltab_d.get();
    a.path = h->path.get();
    bind_pose_cache(h->cache, a);
    return a;
}

extern "C" int mgb_maze_create(mgb_maze **out, int64_t n_envs, const mgb_maze_cfg *cfg, int device,
                               int64_t env_index_base)
{
    MGB_REQUIRE(out && cfg, "null argument");
    MGB_REQUIRE(n_envs > 0, "n_envs must be positive");
    MGB_REQUIRE(cfg->kind == MGB_MAZE_2D || cfg->kind == MGB_MAZE_DISCRETE_3D || cfg->kind == MGB_MAZE_CONTINUOUS_3D,
                "invalid kind");
    MGB_REQUIRE(cfg->task_type == MGB_MAZE_SURVIVAL || cfg->task_type == MGB_MAZE_ESCAPE, "invalid task_type");
    MGB_REQUIRE(cfg->n_cells >= 3 && cfg->n_cells <= kMaxN, "n_cells must be in [3, 31]");
    MGB_REQUIRE(cfg->max_steps > 0, "max_steps must be positive");
    if (cfg->kind == MGB_MAZE_2D) MGB_REQUIRE(cfg->view_grid >= 0 && cfg->view_grid <= 8, "view_grid out of range");
    if (cfg->kind != MGB_MAZE_2D) {
        MGB_REQUIRE(cfg->res_h > 0 && cfg->res_h <= 1024 && cfg->res_v > 0 && cfg->res_v <= 1024, "resolution out of range");
        MGB_REQUIRE(cfg->obs_dtype == MGB_OBS_U8 || cfg->obs_dtype == MGB_OBS_I32 || cfg->obs_dtype == MGB_OBS_F32,
                    "invalid obs_dtype");
        MGB_REQUIRE(cfg->max_vision > 0 && cfg->l_focal > 0 && cfg->text_size > 0 && cfg->fov > 0, "invalid optics");
    }
    int ndev = 0;
    MGB_CUDA(cudaGetDeviceCount(&ndev));
    MGB_REQUIRE(device >= 0 && device < ndev, "device index out of range");
    MgbDeviceGuard guard(device);
    std::unique_ptr<mgb_maze> h(new (std::nothrow) mgb_maze());    // deleted with its buffers on every error exit
    MGB_REQUIRE(h, "out of host memory");
    h->device = device; h->n = n_envs; h->n_pad = (n_envs + 127) / 128 * 128; h->env_base = env_index_base;
    h->cfg = *cfg;
    MazeConst &c = h->c;
    memset(&c, 0, sizeof(c));
    c.kind = cfg->kind; c.task_type = cfg->task_type; c.n = cfg->n_cells; c.max_steps = cfg->max_steps;
    c.view_grid = cfg->view_grid; c.res_h = cfg->res_h; c.res_v = cfg->res_v; c.obs_dtype = cfg->obs_dtype;
    c.max_vision = cfg->max_vision; c.l_focal = cfg->l_focal; c.text_size = cfg->text_size;
    {
        int ex = 0;
        c.text_pow2 = (cfg->text_size > 0 && frexp(cfg->text_size, &ex) == 0.5) ? 1 : 0;
        c.inv_text = cfg->text_size > 0 ? 1.0 / cfg->text_size : 0.0;
    }
    cudaDeviceProp prop;
    MGB_CUDA(cudaGetDeviceProperties(&prop, device));
    h->num_sms = prop.multiProcessorCount;
    if (const char *ev = getenv("MGB_MAZE_FUSED_STEP")) h->fused_step = atoi(ev) != 0;
    if (const char *ev = getenv("MGB_MAZE_RENDER_PIPE")) h->render_pipe = atoi(ev) != 0;
    if (const char *ev = getenv("MGB_MAZE_VARIANT_BITS")) {
        h->variant_bits = atoi(ev);
        if (h->variant_bits < 0) h->variant_bits = 0;
        if (h->variant_bits > kVariantBitsMax) h->variant_bits = kVariantBitsMax;
    }
    if (const char *ev = getenv("MGB_MAZE_CACHE")) h->cache_enabled = atoi(ev) != 0;
    if (const char *ev = getenv("MGB_MAZE_CACHE_GB")) h->cache_budget_gb = atof(ev);
    MGB_CUDA(h->agent.alloc(sizeof(int4) * h->n_pad));
    MGB_CUDA(h->life.alloc(sizeof(double) * h->n_pad));
    MGB_CUDA(h->env2task.alloc(sizeof(int32_t) * h->n_pad));
    MGB_CUDA(cudaMemset(h->agent.get(), 0, sizeof(int4) * h->n_pad));
    MGB_CUDA(cudaMemset(h->life.get(), 0, sizeof(double) * h->n_pad));
    if (cfg->kind != MGB_MAZE_2D) {
        // screen geometry and the per-heading column tables, exactly as maze_view computes them
        // (ray_caster_utils.py:68-92): float64 arithmetic, float32 sin/cos of the float32 heading, float32 tables.
        const int H = cfg->res_h, V = cfg->res_v;
        volatile double half_h = tan(cfg->fov / 2) * cfg->l_focal;
        volatile double half_v = half_h * V / H;
        volatile double pixel_size = 2.0 * half_h / H;
        volatile double pixel_factor = pixel_size / cfg->l_focal;
        c.half_h = half_h; c.half_v = half_v; c.pixel_size = pixel_size;
        c.lb_sx = 0.10 * V; c.lb_sy = 0.10 * V; c.lb_w = 0.05 * H; c.lb_l = 0.80 * V;   // maze_discrete_3d.py:42-45
        std::vector<float> tab((size_t)4 * 3 * H);
        std::vector<double> tab_d((size_t)2 * H);      // heading-independent cos_hp / sin_hp in float64
        const float choice[4] = {0.0f, 0.5f, 1.0f, 1.5f};
        for (int k = 0; k < 4; ++k) {
            volatile float ori = choice[k] * (float)3.1415926;          // maze_discrete_3d.py:46
            volatile float s_ori = sinf(ori), c_ori = cosf(ori);
            volatile double tan_hp = (-0.5 - (double)H / 2) * pixel_factor;
            for (int d = 0; d < H; ++d) {
                tan_hp = tan_hp + pixel_factor;
                volatile double t2 = tan_hp * tan_hp;
                volatile double cos_hp = sqrt(1.0 / (1.0 + t2));
                volatile double sin_hp = tan_hp * cos_hp;
                volatile double a1 = sin_hp * (double)c_ori, a2 = cos_hp * (double)s_ori;
                volatile double b1 = cos_hp * (double)c_ori, b2 = sin_hp * (double)s_ori;
                if (k == 0) { tab_d[d] = cos_hp; tab_d[H + d] = sin_hp; }
                tab[((size_t)k * 3 + 0) * H + d] = (float)cos_hp;
                tab[((size_t)k * 3 + 1) * H + d] = (float)(b1 - b2);
                tab[((size_t)k * 3 + 2) * H + d] = (float)(a1 + a2);
            }
        }
        MGB_CUDA(h->coltab.alloc(tab.size() * sizeof(float)));
        MGB_CUDA(cudaMemcpy(h->coltab.get(), tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
        if (cfg->kind == MGB_MAZE_CONTINUOUS_3D) {
            MGB_CUDA(h->coltab_d.alloc(tab_d.size() * sizeof(double)));
            MGB_CUDA(cudaMemcpy(h->coltab_d.get(), tab_d.data(), tab_d.size() * sizeof(double), cudaMemcpyHostToDevice));
            MGB_CUDA(h->cpos.alloc(sizeof(float2) * h->n_pad));
            MGB_CUDA(h->cori.alloc(sizeof(double) * h->n_pad));
            MGB_CUDA(cudaMemset(h->cpos.get(), 0, sizeof(float2) * h->n_pad));
            MGB_CUDA(cudaMemset(h->cori.get(), 0, sizeof(double) * h->n_pad));
        }
    }
    *out = h.release();
    return MGB_OK;
}

extern "C" void mgb_maze_destroy(mgb_maze *h)
{
    if (!h) return;
    MgbDeviceGuard guard(h->device);
    cudaDeviceSynchronize();
    delete h;                  // the members free the handle's buffers while its device is current
}

extern "C" int64_t mgb_maze_obs_bytes_per_env(const mgb_maze *h)
{
    if (!h) return MGB_ERR_ARG;
    if (h->c.kind == MGB_MAZE_2D) { const int w = 2 * h->c.view_grid + 1; return (int64_t)w * w * 4; }
    return (int64_t)h->c.res_h * h->c.res_v * 3 * (h->c.obs_dtype == MGB_OBS_U8 ? 1 : 4);
}

extern "C" int64_t mgb_maze_launch_count(const mgb_maze *h) { return h ? h->launches : MGB_ERR_ARG; }

extern "C" int mgb_maze_set_episodes_per_task(mgb_maze *h, int32_t k)
{
    MGB_REQUIRE(h, "null handle");
    MGB_REQUIRE(k >= 0, "episodes_per_task must be >= 0 (0: off)");
    MGB_REQUIRE(!h->task_epoch, "call mgb_maze_set_episodes_per_task before mgb_maze_set_task (it fixes the record layout)");
    MgbDeviceGuard guard(h->device);
    MgbDev<uint32_t> count;
    if (k > 0) {
        MGB_CUDA(count.alloc(sizeof(uint32_t) * (size_t)h->n_pad));
        MGB_CUDA(cudaMemset(count.get(), 0, sizeof(uint32_t) * (size_t)h->n_pad));
    }
    h->task_count = std::move(count);
    h->trial_k = k;
    return MGB_OK;
}

extern "C" int mgb_maze_set_expert(mgb_maze *h, int on)
{
    MGB_REQUIRE(h, "null handle");
    MGB_REQUIRE(!h->task_epoch, "call mgb_maze_set_expert before mgb_maze_set_task (the task table then builds the expert's tables)");
    MGB_REQUIRE(!on || h->c.task_type == MGB_MAZE_ESCAPE,
                "the expert is defined for ESCAPE only (SURVIVAL has no single shortest-path target)");
    MGB_REQUIRE(!on || h->c.kind != MGB_MAZE_CONTINUOUS_3D,
                "the expert is defined for the grid mazes only (MetaMazeContinuous3D has continuous actions)");
    h->expert = on != 0;
    return MGB_OK;
}

extern "C" int mgb_maze_task_episodes(mgb_maze *h, int32_t *out_dev, void *stream)
{
    MGB_REQUIRE(h && out_dev, "null argument");
    MGB_REQUIRE(h->trial_k > 0, "not a trial handle (mgb_maze_set_episodes_per_task)");
    MgbDeviceGuard guard(h->device);
    MGB_CUDA(cudaMemcpyAsync(out_dev, h->task_count.get(), sizeof(uint32_t) * (size_t)h->n, cudaMemcpyDeviceToDevice,
                             (cudaStream_t)stream));
    return MGB_OK;
}

extern "C" int mgb_maze_set_options(mgb_maze *h, int auto_reset)
{
    MGB_REQUIRE(h, "null handle");
    h->auto_reset = auto_reset ? 1 : 0;
    return MGB_OK;
}

extern "C" int mgb_maze_cache_info(const mgb_maze *h, int64_t out[16])
{
    MGB_REQUIRE(h && out, "null argument");
    for (int i = 0; i < 16; ++i) out[i] = 0;
    out[0] = h->cache_ready ? h->n_poses : 0;
    if (h->cache_ready && h->var_planned) {
        // update_tasks replans the frames of its tasks on the device: read the counts back (reporting only)
        MgbDeviceGuard guard(h->device);
        MGB_CUDA(cudaDeviceSynchronize());
        std::vector<uint64_t> fm(h->host_poses.size() * 2);
        MGB_CUDA(cudaMemcpy(fm.data(), h->cache.c_fmask.get(), fm.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        for (size_t sl = 0; sl < h->host_poses.size(); ++sl) {
            if (h->host_poses[sl].x < 0) continue;
            const int k = __builtin_popcountll(fm[2 * sl]) + __builtin_popcountll(fm[2 * sl + 1]);
            out[4 + (k < 8 ? k : 8)] += 1;
        }
        if (h->cache.task_frames) {
            std::vector<int32_t> frames((size_t)h->n_tasks);
            MGB_CUDA(cudaMemcpy(frames.data(), h->cache.task_frames.get(), frames.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
            for (int32_t f : frames) out[1] += f;
        }
    }
    out[2] = h->variant_bits_used;
    out[3] = (int64_t)h->cache_bytes;
    out[13] = h->cache_ready ? 1 : 0;
    out[14] = h->c.hits_in_global;      // plan of the last direct-renderer launch: crossing lists in global scratch
    out[15] = h->c.pipe;                // ... and geometry pipelined under the pixels
    return MGB_OK;
}

extern "C" int mgb_maze_set_cache(mgb_maze *h, int enabled)
{
    MGB_REQUIRE(h, "null handle");
    if ((h->cache_enabled != 0) != (enabled != 0)) {
        h->cache_enabled = enabled ? 1 : 0;
        h->cache_dirty = true;            // rebuilt (or dropped) at the next reset / step
    }
    return MGB_OK;
}

namespace {
// entry (steps, e) of every env from its current state: what a step would have stored there
__global__ void maze_path_seed_kernel(const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const int4 ag = a.agent[e];
    const Env s = {ag.x, ag.y, ag.z, ag.w, 0.0};
    path_store(c, a, e, s);
}
}  // namespace

extern "C" int mgb_maze_set_path(mgb_maze *h, int enabled)
{
    MGB_REQUIRE(h, "null handle");
    MgbDeviceGuard guard(h->device);
    if ((bool)h->path == (enabled != 0)) return MGB_OK;
    MGB_CUDA(cudaDeviceSynchronize());
    if (!enabled) { h->path.reset(); return MGB_OK; }
    const size_t bytes = sizeof(char2) * (size_t)path_cap(h) * (size_t)h->n_pad;
    MgbDev<char2> path;
    MGB_CUDA(path.alloc(bytes));
    MGB_CUDA(cudaMemset(path.get(), 0xFF, bytes));          // cells (-1, -1): not recorded
    MazeArgs a = maze_args(h);
    a.path = path.get();                                    // the new buffer, the handle's once it is seeded
    maze_path_seed_kernel<<<(unsigned)((h->n + 255) / 256), 256>>>(h->c, a);
    MGB_CUDA(cudaGetLastError());
    MGB_CUDA(cudaDeviceSynchronize());
    h->launches += 1;
    h->path = std::move(path);
    return MGB_OK;
}

extern "C" int mgb_maze_set_textures(mgb_maze *h, const uint8_t *grounds_host, int32_t n_tex, const uint8_t *ceil_host,
                                     int32_t tex_size)
{
    MGB_REQUIRE(h && grounds_host && ceil_host, "null argument");
    MGB_REQUIRE(h->c.kind != MGB_MAZE_2D, "textures only apply to the 3-D mazes");
    MGB_REQUIRE(n_tex >= 1 && n_tex <= 15, "n_tex must be in [1, 15]");
    MGB_REQUIRE(tex_size >= 1 && tex_size <= 128, "tex_size must be in [1, 128]");
    MgbDeviceGuard guard(h->device);
    MGB_CUDA(cudaDeviceSynchronize());
    const size_t px = (size_t)tex_size * tex_size;
    std::vector<uint32_t> packed((size_t)(n_tex + 1) * px);
    for (size_t i = 0; i < (size_t)n_tex * px; ++i)
        packed[i] = (uint32_t)grounds_host[3 * i] | ((uint32_t)grounds_host[3 * i + 1] << 8) |
                    ((uint32_t)grounds_host[3 * i + 2] << 16);
    for (size_t i = 0; i < px; ++i)
        packed[(size_t)n_tex * px + i] = (uint32_t)ceil_host[3 * i] | ((uint32_t)ceil_host[3 * i + 1] << 8) |
                                         ((uint32_t)ceil_host[3 * i + 2] << 16);
    MgbDev<uint32_t> tex;
    MGB_CUDA(tex.alloc(packed.size() * 4));
    MGB_CUDA(cudaMemcpy(tex.get(), packed.data(), packed.size() * 4, cudaMemcpyHostToDevice));
    h->tex = std::move(tex);
    h->c.n_tex = n_tex; h->c.ts = tex_size;
    h->fp_tex = mgb_fnv(mgb_fnv(mgb_fnv(MGB_FNV_BASIS, &n_tex, sizeof(n_tex)), &tex_size, sizeof(tex_size)), packed.data(),
                        packed.size() * 4);
    h->tex_max = 0;
    for (size_t i = 0; i < 3 * (size_t)n_tex * px; ++i) h->tex_max = grounds_host[i] > h->tex_max ? grounds_host[i] : h->tex_max;
    for (size_t i = 0; i < 3 * px; ++i) h->tex_max = ceil_host[i] > h->tex_max ? ceil_host[i] : h->tex_max;
    h->has_tex = true;
    h->cache_dirty = true;
    return MGB_OK;
}

// One task of the table as the kernels read it: header, walls, textures, food slot of every cell, food values / intervals.
// allow_new_class: set_task may open a new (agent_height, wall_height) class (it builds the eff tables afterwards); a
// partial update may only join an existing class, otherwise the task's pixels compute eff themselves (cls = -1).
static void fill_task_blob(const MazeConst &c, uint8_t *b, const int8_t *walls, const int8_t *texts, const double *food,
                           const int32_t *interval, const mgb_maze_task_scalars &s, std::vector<double> &cls_heights,
                           bool allow_new_class)
{
    const int nn = c.n * c.n;
    TaskHdr hd;
    memset(&hd, 0, sizeof(hd));
    hd.start[0] = s.start[0]; hd.start[1] = s.start[1]; hd.goal[0] = s.goal[0]; hd.goal[1] = s.goal[1];
    hd.cell_size = s.cell_size; hd.wall_height = s.wall_height; hd.agent_height = s.agent_height;
    hd.initial_life = s.initial_life; hd.max_life = s.max_life; hd.step_reward = s.step_reward;
    hd.goal_reward = s.goal_reward;
    {
        int ex = 0;
        const double t2c = c.text_size / s.cell_size;
        hd.cell_pow2 = frexp(s.cell_size, &ex) == 0.5 ? 1 : 0;
        hd.t2c_pow2 = frexp(t2c, &ex) == 0.5 ? 1 : 0;
        hd.inv_cell = 1.0 / s.cell_size;
        hd.inv_t2c = 1.0 / t2c;
        hd.cls = -1;
        for (size_t k = 0; k < cls_heights.size() / 2; ++k)
            if (cls_heights[2 * k] == s.agent_height && cls_heights[2 * k + 1] == s.wall_height) hd.cls = (int)k;
        if (hd.cls < 0 && allow_new_class && cls_heights.size() / 2 < 8) {
            hd.cls = (int)(cls_heights.size() / 2);
            cls_heights.push_back(s.agent_height);
            cls_heights.push_back(s.wall_height);
        }
    }
    int cnt = 0;
    int8_t *fidx = reinterpret_cast<int8_t *>(b + c.off_fidx);
    double *fval = reinterpret_cast<double *>(b + c.off_fval);
    int32_t *fint = reinterpret_cast<int32_t *>(b + c.off_fint);
    for (int k = 0; k < nn; ++k) {
        b[c.off_walls + k] = (uint8_t)walls[k];
        b[c.off_texts + k] = (uint8_t)texts[k];
        const double fv = food[k];
        if (fv > 0.0) {
            fidx[k] = (int8_t)cnt; fval[cnt] = fv; fint[cnt] = interval[k];
            ++cnt;
        } else fidx[k] = -1;
    }
    hd.n_food = cnt;
    memcpy(b, &hd, sizeof(hd));
}

// Free cells of a task: the agent can never stand inside a wall (maze_discrete_3d.py:63-65); the start cell counts as free
static int task_free_cells(const MazeConst &c, const int8_t *walls, const mgb_maze_task_scalars &s)
{
    int cnt = 0;
    for (int k = 0; k < c.n * c.n; ++k) cnt += (walls[k] == 0 || k == s.start[0] * c.n + s.start[1]) ? 1 : 0;
    return cnt;
}

// Pose-cache rows of task slot t: every free cell x 4 headings in cell order at pose slots t S + j (rows[j]); the task's
// other S - 4 x free slots are unused (task -1).  index: the task's [n * n * 4] pose_index row.  Returns the pose count.
static int task_pose_rows(const MazeConst &c, int S, int t, const int8_t *walls, const mgb_maze_task_scalars &s, int4 *rows,
                          int32_t *index)
{
    const int n = c.n, nn = n * n;
    int j = 0;
    for (int k = 0; k < nn; ++k) {
        const bool free = walls[k] == 0 || k == s.start[0] * n + s.start[1];
        for (int o = 0; o < 4; ++o) {
            index[k * 4 + o] = free ? (int32_t)((int64_t)t * S + j) : -1;
            if (free) rows[j++] = make_int4(t, k / n, k % n, o);
        }
    }
    for (int u = j; u < S; ++u) rows[u] = make_int4(-1, 0, 0, 0);
    return j;
}

extern "C" int mgb_maze_set_task(mgb_maze *h, int32_t n_tasks, const int8_t *walls_host, const int8_t *texts_host,
                                 const double *food_rewards_host, const int32_t *food_interval_host,
                                 const mgb_maze_task_scalars *scalars_host, const int32_t *env2task_host)
{
    MgbRange nvtx_range("mgb_maze_set_task");
    MGB_REQUIRE(h && walls_host && texts_host && food_rewards_host && food_interval_host && scalars_host &&
                    env2task_host, "null argument");
    MGB_REQUIRE(n_tasks > 0, "n_tasks must be positive");
    MgbDeviceGuard guard(h->device);
    MGB_CUDA(cudaDeviceSynchronize());
    // Everything the table decides is computed into locals and checked first: a refused call leaves the handle as it was
    MazeConst c = h->c;
    const int n = c.n, nn = n * n;
    // food slots: every cell with a positive reward (the ceiling tint of ray_caster_utils.py:150 tests "> 0")
    int f_max = 0;
    for (int t = 0; t < n_tasks; ++t) {
        int cnt = 0;
        for (int k = 0; k < nn; ++k) cnt += food_rewards_host[(size_t)t * nn + k] > 0.0 ? 1 : 0;
        f_max = cnt > f_max ? cnt : f_max;
        const mgb_maze_task_scalars &s = scalars_host[t];
        MGB_REQUIRE(s.start[0] >= 0 && s.start[0] < n && s.start[1] >= 0 && s.start[1] < n, "start outside the maze");
        MGB_REQUIRE(s.goal[0] >= 0 && s.goal[0] < n && s.goal[1] >= 0 && s.goal[1] < n, "goal outside the maze");
        // maze_base.py:36
        MGB_REQUIRE(s.agent_height < s.wall_height && s.agent_height > 0, "the agent height must be > 0 and < wall height");
        MGB_REQUIRE(s.cell_size > 0, "cell_size must be positive");
    }
    MGB_REQUIRE(f_max <= 127, "at most 127 food cells per task are supported");
    for (int e = 0; e < h->n; ++e) MGB_REQUIRE(env2task_host[e] >= 0 && env2task_host[e] < n_tasks, "env2task out of range");
    bool slot_per_env = true;
    {
        std::vector<uint8_t> used((size_t)n_tasks, 0);
        for (int e = 0; e < h->n; ++e) {
            if (used[env2task_host[e]]) { slot_per_env = false; break; }
            used[env2task_host[e]] = 1;
        }
    }
    c.f_max = f_max;
    // A ray is followed for max_vision at most, i.e. through <= 2 * max_vision / cell_size + 2 cells (one per DDA step
    // plus the start cell), and it moves monotonically in i and j, so it enters at most 2 n - 1 cells of the grid: both
    // bound the transparent crossings a column records (ray_caster_utils.py:24-61), and the reference blends every one.
    double min_cell = scalars_host[0].cell_size;
    for (int t = 1; t < n_tasks; ++t) min_cell = scalars_host[t].cell_size < min_cell ? scalars_host[t].cell_size : min_cell;
    const int geo = (int)ceil(2.0 * c.max_vision / min_cell) + 3;
    int mh = f_max < geo ? f_max : geo;
    mh = mh < 2 * n - 1 ? mh : 2 * n - 1;
    if (mh < 1) mh = 1;
    if (c.task_type == MGB_MAZE_ESCAPE) mh = 2;
    c.max_hits = mh > kMaxHitsCap ? kMaxHitsCap : mh;
    // a warp run = whole columns, about 768 B of output (u8: 256 px, i32: 64 px), never less than one column
    c.run_px = c.obs_dtype == MGB_OBS_U8 ? 256 : 64;
    if (c.kind != MGB_MAZE_2D) {
        if (c.run_px < c.res_v) c.run_px = c.res_v;
        c.run_px = c.run_px / c.res_v * c.res_v;
    }
    // blob layout
    size_t off = sizeof(TaskHdr);
    c.off_walls = (int)off; off += nn;
    c.off_texts = (int)off; off += nn;
    c.off_fidx = (int)off;  off += nn;
    off = (off + 7) / 8 * 8;
    c.off_fval = (int)off;  off += (size_t)(f_max > 0 ? f_max : 1) * 8;
    c.off_fint = (int)off;  off += (size_t)(f_max > 0 ? f_max : 1) * 4;
    c.blob_bytes = (int)((off + 15) / 16 * 16);
    std::vector<uint8_t> blobs((size_t)n_tasks * c.blob_bytes, 0);
    std::vector<double> cls_heights;     // distinct (agent_height, wall_height) pairs, at most 8 get an eff table
    for (int t = 0; t < n_tasks; ++t)
        fill_task_blob(c, blobs.data() + (size_t)t * c.blob_bytes, walls_host + (size_t)t * nn, texts_host + (size_t)t * nn,
                       food_rewards_host + (size_t)t * nn, food_interval_host + (size_t)t * nn, scalars_host[t], cls_heights,
                       true);
    if (c.kind != MGB_MAZE_2D) {
        for (int t = 0; t < n_tasks; ++t)
            for (int k = 0; k < nn; ++k) {
                const int id = texts_host[(size_t)t * nn + k];
                MGB_REQUIRE(id >= 0 && (!h->has_tex || id < c.n_tex), "cell_texts refers to a texture that is not loaded");
            }
    }
    // The per-env resample counts, zero from here on and kept by a later set_task.  They are allocated here, where the
    // call is synchronous anyway, for every table: restore writes them in either record mode, and neither it nor
    // resample_tasks may allocate or touch the legacy stream (both are stream-ordered and can be captured).
    MgbDev<uint32_t> epoch;
    if (!h->task_epoch) {
        MGB_CUDA(epoch.alloc(sizeof(uint32_t) * (size_t)h->n_pad));
        MGB_CUDA(cudaMemset(epoch.get(), 0, sizeof(uint32_t) * (size_t)h->n_pad));
    }
    // The old table goes before the new one is allocated (HBM never holds both); until the new one is complete every
    // step refuses with "Must call set_task" instead of reading a half-built table.
    h->has_task = false; h->tasks = MazeTasks();
    h->exp_dist.reset(); h->exp_mask.reset();
    const size_t eaten_bytes = sizeof(int32_t) * (size_t)(f_max > 0 ? f_max : 1) * h->n_pad;
    MazeTasks tasks;
    MGB_CUDA(tasks.blobs.alloc(blobs.size()));
    MGB_CUDA(cudaMemcpy(tasks.blobs.get(), blobs.data(), blobs.size(), cudaMemcpyHostToDevice));
    MGB_CUDA(tasks.eaten.alloc(eaten_bytes));
    MazeFinal &fin = tasks.fin;
    if (c.kind != MGB_MAZE_2D) {
        MGB_CUDA(fin.count.alloc(sizeof(int32_t)));
        MGB_CUDA(fin.env.alloc(sizeof(int32_t) * h->n));
        MGB_CUDA(fin.task.alloc(sizeof(int32_t) * h->n));
        MGB_CUDA(fin.eaten.alloc(eaten_bytes));
        MGB_CUDA(fin.dyn.alloc(sizeof(EnvDyn) * h->n));
        MGB_CUDA(fin.agent.alloc(sizeof(int4) * h->n));
        MGB_CUDA(fin.life.alloc(sizeof(double) * h->n));
        if (c.kind == MGB_MAZE_CONTINUOUS_3D) {
            MGB_CUDA(fin.cpos.alloc(sizeof(float2) * h->n));
            MGB_CUDA(fin.cori.alloc(sizeof(double) * h->n));
        }
    }
    MGB_CUDA(cudaMemcpy(h->env2task.get(), env2task_host, sizeof(int32_t) * h->n, cudaMemcpyHostToDevice));
    c.n_cls = 0;
    if (c.kind != MGB_MAZE_2D && !cls_heights.empty()) {
        const int n_cls = (int)(cls_heights.size() / 2);
        const size_t cells = (size_t)n_cls * c.res_h * c.res_v;
        MgbDev<double> d_heights;
        MGB_CUDA(tasks.efftab.alloc(cells * sizeof(double)));
        MGB_CUDA(tasks.fogtab.alloc(cells * sizeof(double)));
        MGB_CUDA(d_heights.alloc(cls_heights.size() * sizeof(double)));
        MGB_CUDA(cudaMemcpy(d_heights.get(), cls_heights.data(), cls_heights.size() * sizeof(double), cudaMemcpyHostToDevice));
        maze_efftab_kernel<<<(unsigned)((cells + 255) / 256), 256>>>(c, h->coltab.get(), d_heights.get(), n_cls, tasks.efftab.get(), tasks.fogtab.get());
        MGB_CUDA(cudaDeviceSynchronize());
        c.n_cls = n_cls;
        h->launches += 1;
    }
    h->c = c;
    h->tasks = std::move(tasks);
    if (epoch) h->task_epoch = std::move(epoch);
    h->cls_heights = std::move(cls_heights);
    h->min_cell = min_cell; h->slot_per_env = slot_per_env;
    h->slot_fp.assign((size_t)n_tasks, 0);
    for (int t = 0; t < n_tasks; ++t)
        h->slot_fp[t] = mgb_fnv(MGB_FNV_BASIS, blobs.data() + (size_t)t * c.blob_bytes, (size_t)c.blob_bytes);
    h->n_tasks = n_tasks;
    if (h->expert) {
        const size_t states = (size_t)n_tasks * expert_planes(c.kind) * nn;
        MGB_CUDA(h->exp_dist.alloc(states * sizeof(uint16_t)));
        MGB_CUDA(h->exp_mask.alloc(states));
        const int rc = build_expert(h, n_tasks, nullptr, nullptr, nullptr, 0, nullptr);
        if (rc) return rc;
    }
    h->has_task = true;
    h->task_flags.reset();
    // pose list of the cache: every free cell x 4 headings of every task, S = 4 x the most free cells of a task per task
    // slot, so that update_tasks can rebuild one task's poses in place
    h->host_poses.clear();
    h->host_pose_index.assign((size_t)n_tasks * nn * 4, -1);
    h->task_poses.assign((size_t)n_tasks, 0);
    h->pose_stride = 0;
    h->cache_dirty = true;
    h->cache_ready = false;
    if (c.kind == MGB_MAZE_DISCRETE_3D) {
        int most = 0;
        for (int t = 0; t < n_tasks; ++t) {
            const int f = task_free_cells(c, walls_host + (size_t)t * nn, scalars_host[t]);
            most = f > most ? f : most;
        }
        h->pose_stride = 4 * most;
        h->host_poses.resize((size_t)n_tasks * h->pose_stride);
        for (int t = 0; t < n_tasks; ++t)
            h->task_poses[t] = task_pose_rows(c, h->pose_stride, t, walls_host + (size_t)t * nn, scalars_host[t],
                                              h->host_poses.data() + (size_t)t * h->pose_stride,
                                              h->host_pose_index.data() + (size_t)t * nn * 4);
    }
    // set_task leaves the env in "need reset" state (maze_env.py:44-50): initialise it so a stray step is harmless
    MazeArgs a = maze_args(h);
    if (h->trial_k) MGB_CUDA(cudaMemset(h->task_count.get(), 0, sizeof(uint32_t) * (size_t)h->n_pad));   // every env has a new maze
    maze_reset_kernel<<<(unsigned)((h->n + 255) / 256), 256>>>(h->c, a, nullptr);
    MGB_CUDA(cudaDeviceSynchronize());
    h->launches += 1;
    return MGB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Device-side task sampler (SURVEY.md 8f row 3): per-episode task resampling without the host.  Measured motivation
// (bench.py --workload maze3d, task_churn): 1024 envs finish ~26 000 episodes/s on the direct renderer, the host samplers
// deliver 700 (reference random streams) to 4 200 (numpy RandomState) tasks/s.  This kernel draws a fresh maze per finished
// env -- one thread per env, Philox keyed by (seed, global env index, resample count) -- from the same distribution family
// as MazeTaskSampler(rng=...) (metagym_b200/metamaze.py; the reference's maze_task.py:41-190 draws from Python's and
// numpy's global MT19937 streams, which a device cannot replay: parity with the reference is distributional and
// structural: rooms on odd coordinates, border walls, a spanning tree of the room lattice by randomised Kruskal, loops
// knocked out down to crowd_ratio, textures 1..n_texts-1 on walls, start/goal rooms > 0.45 n apart, food values
// np.clip(U * food_reward, 0.1, food_reward) thinned by 0.9 per round until their sum is <= (n-1)^2 food_density, an
// interval where a value is above 1e-3).  The draws themselves are restated exactly in tests/maze_sampler_draws.py, and
// the tests compare every sampled task with that restatement.
// ---------------------------------------------------------------------------------------------------------------
struct PhiloxStream {
    uint2 key;
    uint4 ctr;
    uint4 buf;
    int have;
    __device__ uint32_t next()
    {
        if (have == 0) { buf = mgb_philox4x32_10(ctr, key); ctr.z += 1u; have = 4; }
        const uint32_t v = have == 4 ? buf.x : (have == 3 ? buf.y : (have == 2 ? buf.z : buf.w));
        --have;
        return v;
    }
    __device__ double uniform() { return (double)(next() >> 8) * (1.0 / 16777216.0); }
    __device__ int below(int n) { return (int)(((uint64_t)next() * (uint64_t)n) >> 32); }     // uniform in [0, n)
};
#define MGB_STREAM_SAMPLER 0x300u

constexpr int kSamplerWarps = 4;
// One WARP per env.  Lane 0 carves the maze (randomised Kruskal + loop knock-out are sequential by nature; their working set
// lives in shared memory); textures, food values and the food thinning rounds are counter-based per cell -- Philox keyed by
// (seed; global env, resample count, cell, purpose) -- so the 32 lanes take cells side by side instead of one
// thread walking them serially (the thinning alone is 20 rounds x n^2 draws).
namespace {
// The draw of one env's task by one whole warp (all 32 lanes call it): the resample count *epoch goes up by one and the
// task is written to the blob b (global memory: the env's table slot; shared memory: a tile that the caller copies there).
// ws: the warp's workspace of sampler_ws_bytes(n) bytes, 16-byte aligned.  Lane 0 returns after the other lanes.
__device__ __noinline__ void maze_sample_task(const MazeConst &c, const SamplerCfg &sc, uint64_t seed, int64_t genv,
                                              uint32_t *epoch, uint8_t *ws, uint8_t *b)
{
    const int lane = threadIdx.x & 31;
    const int n = c.n, nn = n * n, m = (n - 1) / 2;
    uint32_t *val = reinterpret_cast<uint32_t *>(ws);               // 24-bit draw behind every cell's food value
    uint16_t *order = reinterpret_cast<uint16_t *>(ws + 4 * nn);
    uint8_t *walls = ws + 6 * nn;                                   // bit 0 wall, bit 1 food alive
    uint8_t *parent = ws + 7 * nn;
    const uint32_t ep = *epoch + 1u;
    __syncwarp();
    if (lane == 0) *epoch = ep;
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const uint32_t hi = (uint32_t)((uint64_t)genv >> 32);
    // per-cell draws: ctr = (env, resample count, cell, purpose)
    auto cell_draw = [&](int k, uint32_t purpose) { return mgb_philox4x32_10(make_uint4((uint32_t)genv, ep, (uint32_t)k, purpose + hi), key); };
    const uint32_t P_TEX = MGB_STREAM_SAMPLER + 0x10u, P_VAL = MGB_STREAM_SAMPLER + 0x20u, P_KEEP = MGB_STREAM_SAMPLER + 0x1000u;
    for (int k = lane; k < nn; k += 32) {
        const int i = k / n, j = k - i * n;
        walls[k] = ((i & 1) && (j & 1)) ? 0 : 1;
    }
    for (int k = lane; k < m * m; k += 32) parent[k] = (uint8_t)k;
    __syncwarp();
    int sx = 1, sy = 1, gx = n - 2, gy = n - 2;
    if (lane == 0) {
        PhiloxStream rng;                                            // the sequential stream of the carving steps
        rng.key = key;
        rng.ctr = make_uint4((uint32_t)genv, ep, 0u, MGB_STREAM_SAMPLER + hi);
        rng.have = 0;
        auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
        // ---- random spanning tree of the room lattice (Kruskal over shuffled edges); edge id = 2 * room + dir
        int ne = 0;
        for (int ra = 0; ra < m; ++ra)
            for (int rb = 0; rb < m; ++rb) {
                if (ra + 1 < m) order[ne++] = (uint16_t)(2 * (ra * m + rb));
                if (rb + 1 < m) order[ne++] = (uint16_t)(2 * (ra * m + rb) + 1);
            }
        for (int k = ne - 1; k > 0; --k) { const int j = rng.below(k + 1); const uint16_t t = order[k]; order[k] = order[j]; order[j] = t; }
        for (int k = 0; k < ne; ++k) {
            const int room = order[k] >> 1, dir = order[k] & 1, ra = room / m, rb = room % m;
            const int other = dir == 0 ? (ra + 1) * m + rb : ra * m + rb + 1;
            const int x = find(room), y = find(other);
            if (x != y) {
                parent[x] = (uint8_t)y;
                if (dir == 0) walls[(2 * ra + 2) * n + 2 * rb + 1] = 0; else walls[(2 * ra + 1) * n + 2 * rb + 2] = 0;
            }
        }
        // ---- loops: knock interior walls out (in random order, only next to a free cell) down to crowd_ratio
        if (sc.allow_loops) {
            int standing = 0, nc = 0;
            for (int i = 1; i < n - 1; ++i)
                for (int j = 1; j < n - 1; ++j)
                    if (walls[i * n + j]) { ++standing; order[nc++] = (uint16_t)(i * n + j); }
            const double budget = (double)((n - 2) * (n - 2)) * sc.crowd_ratio;
            for (int k = nc - 1; k > 0; --k) { const int j = rng.below(k + 1); const uint16_t t = order[k]; order[k] = order[j]; order[j] = t; }
            for (int k = 0; k < nc && (double)standing > budget; ++k) {
                const int cell = order[k];
                if (!walls[cell - n] || !walls[cell + n] || !walls[cell - 1] || !walls[cell + 1]) { walls[cell] = 0; --standing; }
            }
        }
        // ---- start / goal (maze_task.py:153-160: rooms, goal far enough from the start)
        sx = rng.below(m) * 2 + 1; sy = rng.below(m) * 2 + 1;
        for (int t = 0; t < m * m; ++t) {
            const int ex = rng.below(m) * 2 + 1, ey = rng.below(m) * 2 + 1;
            const double dx = ex - sx, dy = ey - sy;
            if (sqrt(dx * dx + dy * dy) > 0.45 * n) { gx = ex; gy = ey; break; }
        }
    }
    __syncwarp();
    // ---- textures + food values, one cell per lane and pass
    auto value_of = [&](uint32_t u24) {      // np.clip(food_reward * U, 0.10, food_reward): below 0.10, food_reward wins
        const double v = (double)u24 * (1.0 / 16777216.0) * sc.food_reward;
        const double lo = v < 0.10 ? 0.10 : v;
        return lo > sc.food_reward ? sc.food_reward : lo;
    };
    double total = 0.0;
    int alive = 0;
    for (int k = lane; k < nn; k += 32) {
        const uint4 r = cell_draw(k, P_TEX);
        const int tx = 1 + (int)(((uint64_t)r.x * (uint64_t)(sc.n_texts - 1)) >> 32);      // randint(1, n_texts)
        const bool wall = walls[k] & 1;
        b[c.off_walls + k] = wall ? 1 : 0;
        b[c.off_texts + k] = wall ? (uint8_t)tx : 0;
        const uint32_t u24 = cell_draw(k, P_VAL).x >> 8;
        val[k] = u24;
        if (!wall) { walls[k] |= 2; total += value_of(u24); ++alive; }
    }
    auto warp_sum = [&](double &t, int &cnt) {                        // fixed butterfly: the same sum on every lane
        for (int o = 16; o > 0; o >>= 1) { t += __shfl_xor_sync(0xffffffffu, t, o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
    };
    warp_sum(total, alive);
    // ---- thinning: food *= (rand < 0.90) per round until the total value and the slot count fit (maze_task.py:176-180)
    const double expected = (double)((n - 1) * (n - 1)) * sc.food_density;
    for (uint32_t round = 0; total > expected || alive > c.f_max; ++round) {
        total = 0.0; alive = 0;
        for (int k = lane; k < nn; k += 32) {
            if (!(walls[k] & 2)) continue;
            const uint4 r = cell_draw(k, P_KEEP + (round >> 2));
            const uint32_t x = (round & 3u) == 0 ? r.x : ((round & 3u) == 1 ? r.y : ((round & 3u) == 2 ? r.z : r.w));
            if ((double)(x >> 8) * (1.0 / 16777216.0) < 0.90) { total += value_of(val[k]); ++alive; }
            else walls[k] &= ~2;
        }
        warp_sum(total, alive);
    }
    __syncwarp();
    int8_t *fidx = reinterpret_cast<int8_t *>(b + c.off_fidx);
    double *fval = reinterpret_cast<double *>(b + c.off_fval);
    int32_t *fint = reinterpret_cast<int32_t *>(b + c.off_fint);
    if (lane != 0) return;
    {
        int cnt = 0;
        for (int k = 0; k < nn; ++k) {                                 // food slots numbered in cell order
            if (walls[k] & 2) {
                const double v = value_of(val[k]);
                fidx[k] = (int8_t)cnt; fval[cnt] = v; fint[cnt] = v > 1.0e-3 ? sc.food_interval : 0;   // maze_task.py:174
                ++cnt;
            } else fidx[k] = -1;
        }
        // the slots past n_food and the header hold zeros, as fill_task_blob writes them: a sampled blob is byte for
        // byte the blob of the same task given to set_task / update_tasks
        for (int f = cnt; f < c.f_max; ++f) { fval[f] = 0.0; fint[f] = 0; }
        TaskHdr hd = {};
        hd.start[0] = sx; hd.start[1] = sy; hd.goal[0] = gx; hd.goal[1] = gy;
        hd.cell_size = sc.cell_size; hd.wall_height = sc.wall_height; hd.agent_height = sc.agent_height;
        hd.initial_life = sc.initial_life; hd.max_life = sc.max_life; hd.step_reward = sc.step_reward;
        hd.goal_reward = sc.goal_reward;
        hd.n_food = cnt; hd.cls = sc.cls;
        int ex = 0;
        const double t2c = c.text_size / sc.cell_size;
        hd.cell_pow2 = frexp(sc.cell_size, &ex) == 0.5 ? 1 : 0;
        hd.t2c_pow2 = frexp(t2c, &ex) == 0.5 ? 1 : 0;
        hd.inv_cell = 1.0 / sc.cell_size;
        hd.inv_t2c = 1.0 / t2c;
        *reinterpret_cast<TaskHdr *>(b) = hd;
    }
}
}  // namespace

__global__ void __launch_bounds__(32 * kSamplerWarps) maze_sample_tasks_kernel(const __grid_constant__ MazeConst c,
                                                                              const __grid_constant__ MazeArgs a,
                                                                              uint8_t *blobs, const uint8_t *mask, uint32_t *epoch,
                                                                              const __grid_constant__ SamplerCfg sc, uint64_t seed,
                                                                              uint32_t *count)
{
    __shared__ __align__(16) uint8_t s_ws[kSamplerWarps][kSamplerWsMax];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t e = (int64_t)blockIdx.x * kSamplerWarps + w;
    if (e >= a.n) return;                                          // warp-uniform exits: no block-wide barrier below
    if (mask && !mask[e]) return;
    uint8_t *b = blobs + (size_t)a.env2task[e] * c.blob_bytes;
    maze_sample_task(c, sc, seed, a.env_base + e, epoch + e, s_ws[w], b);
    if (lane != 0) return;
    if (count) count[e] = 0;                                       // trial handle: no episode finished on the new maze yet
    // ---- the env starts an episode on its new task (set_task + reset of that env, maze_env.py:44-57)
    Env s;
    env_reset(c, b, a.eaten + e, a.n_pad, s);
    a.agent[e] = make_int4(s.gx, s.gy, s.ori, s.steps);
    a.life[e] = s.life;
    path_store(c, a, e, s);
    if (c.kind == MGB_MAZE_CONTINUOUS_3D) {
        a.cpos[e] = make_float2((float)(s.gx * sc.cell_size + 0.5 * sc.cell_size), (float)(s.gy * sc.cell_size + 0.5 * sc.cell_size));
        a.cori[e] = 0.0;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Partial, stream-ordered task replacement (per-episode task resampling, SURVEY.md 8f row 3 / maze_base.py:19-38)
// ---------------------------------------------------------------------------------------------------------------
// staging layout: [count] int32 table slots | pad to 16 | [count] blobs | with pose lists (discrete 3-D): [count][S] int4
// pose rows | [count][n * n * 4] int32 pose_index rows | [n_fill] int32 pose slots of the replaced tasks.  poses: the
// cache's tables to scatter the rows into (nullptr: no cache built)
__global__ void maze_scatter_tasks_kernel(const __grid_constant__ MazeConst c, uint8_t *blobs, const uint8_t *stage, int count,
                                          uint8_t *task_flags, int4 *poses, int32_t *pose_index, int S)
{
    const int32_t *slots = reinterpret_cast<const int32_t *>(stage);
    const uint8_t *blob0 = stage + (((size_t)count * 4 + 15) / 16) * 16;
    const uint4 *src = reinterpret_cast<const uint4 *>(blob0) + (size_t)blockIdx.x * (c.blob_bytes / 16);
    const int64_t t = slots[blockIdx.x];
    uint4 *dst = reinterpret_cast<uint4 *>(blobs + (size_t)t * c.blob_bytes);
    for (int i = threadIdx.x; i < c.blob_bytes / 16; i += blockDim.x) dst[i] = src[i];
    if (poses) {
        const int per = c.n * c.n * 4;
        const int4 *prow = reinterpret_cast<const int4 *>(blob0 + (size_t)count * c.blob_bytes);
        const int32_t *irow = reinterpret_cast<const int32_t *>(prow + (size_t)count * S) + (size_t)blockIdx.x * per;
        prow += (size_t)blockIdx.x * S;
        for (int i = threadIdx.x; i < S; i += blockDim.x) poses[t * S + i] = prow[i];
        for (int i = threadIdx.x; i < per; i += blockDim.x) pose_index[t * per + i] = irow[i];
    }
    if (threadIdx.x == 0) task_flags[t] = 1;
}
__global__ void maze_clear_flags_kernel(uint8_t *task_flags, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) task_flags[i] = 0;
}

// Trial handles: the envs whose table slot mgb_maze_update_tasks just replaced have finished no episode on their new maze
__global__ void maze_zero_counts_kernel(int64_t n, const int32_t *env2task, const uint8_t *task_flags, uint32_t *count)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n && task_flags[env2task[e]]) count[e] = 0;
}

// Trial handles, after a step (T = 1) or a rollout without resampling: every done of done [T][n] is one more episode
// finished on the env's maze.  The kernels that write done stay as every other handle runs them.
__global__ void maze_count_done_kernel(int64_t n, int T, const uint8_t *__restrict__ done, uint32_t *count)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    uint32_t k = 0;
    for (int t = 0; t < T; ++t) k += done[(int64_t)t * n + e] != 0;
    if (k) count[e] += k;
}

// Lay the host pose lists out at the larger stride S (a handle on the direct renderer took a task with more free cells
// than the table's largest; a cache enabled later is built at the new stride)
static void relayout_poses(mgb_maze *h, int S)
{
    const int old = h->pose_stride;
    std::vector<int4> rows((size_t)h->n_tasks * S, make_int4(-1, 0, 0, 0));
    for (int t = 0; t < h->n_tasks; ++t)
        for (int j = 0; j < h->task_poses[t]; ++j) rows[(size_t)t * S + j] = h->host_poses[(size_t)t * old + j];
    for (int32_t &v : h->host_pose_index)
        if (v >= 0) v = (int32_t)((int64_t)(v / old) * S + v % old);
    h->host_poses = std::move(rows);
    h->pose_stride = S;
}

static int render_region(mgb_maze *h, const MazeArgs &a, int K, int64_t n_fill, cudaStream_t st);
static int bake_region(mgb_maze *h, MazePoseCache &pc, MazeArgs a, int K, cudaStream_t st);
static bool pose_cache_serves(const mgb_maze *h);

extern "C" int mgb_maze_update_tasks(mgb_maze *h, int32_t count, const int32_t *task_slots_host, const int8_t *walls_host,
                                     const int8_t *texts_host, const double *food_rewards_host,
                                     const int32_t *food_interval_host, const mgb_maze_task_scalars *scalars_host,
                                     void *stream)
{
    MgbRange nvtx_range("mgb_maze_update_tasks");
    MGB_REQUIRE(h && task_slots_host && walls_host && texts_host && food_rewards_host && food_interval_host && scalars_host,
                "null argument");
    MGB_REQUIRE(count > 0, "count must be positive");
    MGB_REQUIRE(h->has_task, "call mgb_maze_set_task first (it sizes the task table)");
    MgbDeviceGuard guard(h->device);
    MazeConst &c = h->c;
    const int n = c.n, nn = n * n;
    // discrete 3-D tables keep the cache's pose lists; a handle that serves (or will serve) them from the pose cache
    // rebuilds the replaced tasks' region in place, which needs every task within the table's S / 4 free cells
    const bool poses_kept = c.kind == MGB_MAZE_DISCRETE_3D && !h->host_poses.empty();
    const bool cached = pose_cache_serves(h);
    int most = 0;
    int64_t n_fill = 0;
    for (int t = 0; t < count; ++t) {
        MGB_REQUIRE(task_slots_host[t] >= 0 && task_slots_host[t] < h->n_tasks, "task slot out of range");
        int cnt = 0;
        for (int k = 0; k < nn; ++k) {
            cnt += food_rewards_host[(size_t)t * nn + k] > 0.0 ? 1 : 0;
            const int id = texts_host[(size_t)t * nn + k];
            MGB_REQUIRE(c.kind == MGB_MAZE_2D || (id >= 0 && (!h->has_tex || id < c.n_tex)), "cell_texts refers to a texture that is not loaded");
        }
        MGB_REQUIRE(cnt <= c.f_max, "a replacement task may not have more food cells than the largest task of set_task");
        const mgb_maze_task_scalars &s = scalars_host[t];
        MGB_REQUIRE(s.start[0] >= 0 && s.start[0] < n && s.start[1] >= 0 && s.start[1] < n, "start outside the maze");
        MGB_REQUIRE(s.goal[0] >= 0 && s.goal[0] < n && s.goal[1] >= 0 && s.goal[1] < n, "goal outside the maze");
        MGB_REQUIRE(s.agent_height < s.wall_height && s.agent_height > 0, "the agent height must be > 0 and < wall height");
        MGB_REQUIRE(s.cell_size >= h->min_cell, "a replacement task may not have smaller cells than the table's smallest");
        if (poses_kept) {
            const int f = task_free_cells(c, walls_host + (size_t)t * nn, s);
            MGB_REQUIRE(!cached || 4 * f <= h->pose_stride,
                        "a replacement task may not have more free cells than the largest task of set_task (pose cache)");
            most = f > most ? f : most;
            n_fill += 4 * f;
        }
    }
    if (cached) {
        std::vector<uint8_t> seen((size_t)h->n_tasks, 0);
        for (int t = 0; t < count; ++t) {
            MGB_REQUIRE(!seen[task_slots_host[t]], "a task slot may be replaced only once per call (pose cache)");
            seen[task_slots_host[t]] = 1;
        }
    }
    if (poses_kept && 4 * most > h->pose_stride) relayout_poses(h, 4 * most);
    const int S = h->pose_stride, per = nn * 4;
    const bool rebuild = cached && h->cache_ready && !h->cache_dirty;   // before the first build the build covers the change
    // pinned staging, double-buffered: the host waits only for the COPY of the call before last, never for the device
    MazeStage &s = h->stage[h->stage_next];
    const size_t head = (((size_t)count * 4 + 15) / 16) * 16, rows_off = head + (size_t)count * c.blob_bytes;
    const size_t index_off = rows_off + (poses_kept ? (size_t)count * S * sizeof(int4) : 0);
    const size_t fill_off = index_off + (poses_kept ? (size_t)count * per * sizeof(int32_t) : 0);
    const size_t need = fill_off + (size_t)n_fill * sizeof(int32_t);
    if (!s.copied) MGB_CUDA(s.copied.create(cudaEventDisableTiming));
    else MGB_CUDA(cudaEventSynchronize(s.copied.get()));
    if (need > s.bytes) {
        const size_t cap = need * 2;
        MgbPinned<uint8_t> host;
        MgbDev<uint8_t> dev;
        MGB_CUDA(host.alloc(cap));
        MGB_CUDA(dev.alloc(cap));
        s.host = std::move(host); s.dev = std::move(dev); s.bytes = cap;
    }
    if (!h->task_flags) {
        MgbDev<uint8_t> flags;
        MGB_CUDA(flags.alloc((size_t)h->n_tasks));
        MGB_CUDA(cudaMemset(flags.get(), 0, (size_t)h->n_tasks));
        h->task_flags = std::move(flags);
    }
    uint8_t *hs = s.host.get();
    memset(hs, 0, need);
    memcpy(hs, task_slots_host, (size_t)count * 4);
    for (int t = 0; t < count; ++t)
        fill_task_blob(c, hs + head + (size_t)t * c.blob_bytes, walls_host + (size_t)t * nn, texts_host + (size_t)t * nn,
                       food_rewards_host + (size_t)t * nn, food_interval_host + (size_t)t * nn, scalars_host[t], h->cls_heights,
                       false);
    int4 *rows = reinterpret_cast<int4 *>(hs + rows_off);
    int32_t *index = reinterpret_cast<int32_t *>(hs + index_off), *fill = reinterpret_cast<int32_t *>(hs + fill_off);
    std::vector<int32_t> task_n((size_t)count, 0);
    if (poses_kept) {
        int64_t k = 0;
        for (int t = 0; t < count; ++t) {
            const int64_t slot = task_slots_host[t];
            task_n[t] = task_pose_rows(c, S, (int)slot, walls_host + (size_t)t * nn, scalars_host[t], rows + (size_t)t * S,
                                        index + (size_t)t * per);
            for (int j = 0; j < task_n[t]; ++j) fill[k++] = (int32_t)(slot * S + j);
        }
    }
    cudaStream_t st = (cudaStream_t)stream;
    MGB_CUDA(cudaMemcpyAsync(s.dev.get(), hs, need, cudaMemcpyHostToDevice, st));
    MGB_CUDA(cudaEventRecord(s.copied.get(), st));
    h->stage_next ^= 1;
    maze_scatter_tasks_kernel<<<(unsigned)count, 128, 0, st>>>(c, h->tasks.blobs.get(), s.dev.get(), count, h->task_flags.get(),
                                                               rebuild ? h->cache.poses.get() : nullptr,
                                                               rebuild ? h->cache.pose_index.get() : nullptr, S);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    if (rebuild) {
        MazeArgs ar = maze_args(h);
        ar.region = reinterpret_cast<const int32_t *>(s.dev.get());
        ar.fill_slot = reinterpret_cast<const int32_t *>(s.dev.get() + fill_off);
        int rc = render_region(h, ar, count, n_fill, st);
        if (rc) return rc;
        rc = bake_region(h, h->cache, ar, count, st);
        if (rc) return rc;
    }
    MazeArgs a = maze_args(h);
    maze_reset_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, st>>>(c, a, h->task_flags.get());
    if (h->trial_k) {
        maze_zero_counts_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, st>>>(h->n, h->env2task.get(), h->task_flags.get(),
                                                                               h->task_count.get());
        h->launches += 1;
    }
    if (const int rc = build_expert(h, h->n_tasks, nullptr, h->task_flags.get(), nullptr, 0, st)) return rc;
    maze_clear_flags_kernel<<<(unsigned)((h->n_tasks + 255) / 256), 256, 0, st>>>(h->task_flags.get(), h->n_tasks);
    MGB_CUDA(cudaGetLastError());
    h->launches += 2;
    // the slots' fingerprints and pose lists change once their new blobs are on their way
    for (int t = 0; t < count; ++t) {
        const int64_t slot = task_slots_host[t];
        h->slot_fp[slot] = mgb_fnv(MGB_FNV_BASIS, hs + head + (size_t)t * c.blob_bytes, (size_t)c.blob_bytes);
        if (!poses_kept) continue;
        memcpy(h->host_poses.data() + slot * S, rows + (size_t)t * S, (size_t)S * sizeof(int4));
        memcpy(h->host_pose_index.data() + slot * per, index + (size_t)t * per, (size_t)per * sizeof(int32_t));
        h->n_poses += task_n[t] - h->task_poses[slot];
        h->task_poses[slot] = task_n[t];
    }
    return MGB_OK;
}

// What MGB_REQUIRE does, for a refusal made on behalf of the function `fn`
static int maze_refuse(const char *fn, const char *msg)
{
    mgb_set_error("%s: %s", fn, msg);
    return MGB_ERR_ARG;
}

// What device resampling needs of the handle and of the sampler cfg (mgb_maze_resample_tasks, mgb_maze_rollout):
// the refusal, or nullptr with sc derived from cfg
static const char *sampler_cfg(const mgb_maze *h, const mgb_maze_sampler_cfg *cfg, SamplerCfg &sc)
{
    if (!h->has_task) return "call mgb_maze_set_task first (it sizes the task table)";
    if (!h->slot_per_env)
        return "device resampling needs one task-table slot per env (mgb_maze_set_task with n_tasks >= n_envs and an injective "
               "env2task)";
    const MazeConst &c = h->c;
    if (pose_cache_serves(h))
        return "device resampling needs the direct renderer: create the env with the pose cache off (cache=False)";
    if (!(c.n % 2 == 1 && c.n > 6)) return "Cell Numbers can only be odd, minimum 7 (maze_task.py:57-58)";
    if (!(cfg->step_reward < 0)) return "step_reward must be < 0 (maze_task.py:59)";
    if (!(cfg->agent_height < cfg->wall_height && cfg->agent_height > 0)) return "the agent height must be > 0 and < wall height";
    if (!(cfg->cell_size >= h->min_cell)) return "resampled tasks may not have smaller cells than the table's smallest";
    if (!(cfg->n_texts >= 2 && (c.kind == MGB_MAZE_2D || !h->has_tex || cfg->n_texts <= c.n_tex))) return "n_texts out of range";
    if (!(cfg->food_reward > 0 && cfg->food_density >= 0 && cfg->crowd_ratio >= 0)) return "invalid sampler parameters";
    sc.allow_loops = cfg->allow_loops; sc.n_texts = cfg->n_texts; sc.food_interval = cfg->food_interval;
    sc.cell_size = cfg->cell_size; sc.wall_height = cfg->wall_height; sc.agent_height = cfg->agent_height;
    sc.step_reward = cfg->step_reward;
    sc.goal_reward = cfg->goal_reward > 0 ? cfg->goal_reward : -sqrt((double)c.n) * c.n * cfg->step_reward;   // maze_task.py:163-166
    sc.food_reward = cfg->food_reward; sc.initial_life = cfg->initial_life; sc.max_life = cfg->max_life;
    sc.food_density = cfg->food_density; sc.crowd_ratio = cfg->crowd_ratio;
    sc.cls = -1;
    for (size_t k = 0; k < h->cls_heights.size() / 2; ++k)
        if (h->cls_heights[2 * k] == cfg->agent_height && h->cls_heights[2 * k + 1] == cfg->wall_height) sc.cls = (int)k;
    return nullptr;
}

extern "C" int mgb_maze_resample_tasks(mgb_maze *h, const uint8_t *mask_dev, const mgb_maze_sampler_cfg *cfg, uint64_t seed,
                                       void *stream)
{
    MgbRange nvtx_range("mgb_maze_resample_tasks");
    MGB_REQUIRE(h && cfg, "null argument");
    SamplerCfg sc;
    if (const char *why = sampler_cfg(h, cfg, sc)) return maze_refuse(__func__, why);
    MgbDeviceGuard guard(h->device);
    const MazeConst &c = h->c;
    MazeArgs a = maze_args(h);
    maze_sample_tasks_kernel<<<(unsigned)((h->n + kSamplerWarps - 1) / kSamplerWarps), 32 * kSamplerWarps, 0, (cudaStream_t)stream>>>(c, a, h->tasks.blobs.get(), mask_dev, h->task_epoch.get(),
                                                                                        sc, seed, h->task_count.get());
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return build_expert(h, h->n, h->env2task.get(), mask_dev, nullptr, 0, (cudaStream_t)stream);
}

extern "C" int mgb_maze_get_tasks(mgb_maze *h, int32_t count, const int32_t *task_slots_host, int8_t *walls_host,
                                  int8_t *texts_host, double *food_rewards_host, int32_t *food_interval_host,
                                  mgb_maze_task_scalars *scalars_host)
{
    MGB_REQUIRE(h && task_slots_host && walls_host && texts_host && food_rewards_host && food_interval_host && scalars_host,
                "null argument");
    MGB_REQUIRE(h->has_task && count > 0, "no task table");
    MgbDeviceGuard guard(h->device);
    MGB_CUDA(cudaDeviceSynchronize());
    const MazeConst &c = h->c;
    const int nn = c.n * c.n;
    std::vector<uint8_t> blob((size_t)c.blob_bytes);
    for (int t = 0; t < count; ++t) {
        MGB_REQUIRE(task_slots_host[t] >= 0 && task_slots_host[t] < h->n_tasks, "task slot out of range");
        MGB_CUDA(cudaMemcpy(blob.data(), h->tasks.blobs.get() + (size_t)task_slots_host[t] * c.blob_bytes, blob.size(), cudaMemcpyDeviceToHost));
        TaskHdr hd;
        memcpy(&hd, blob.data(), sizeof(hd));
        const int8_t *fidx = reinterpret_cast<const int8_t *>(blob.data() + c.off_fidx);
        const double *fval = reinterpret_cast<const double *>(blob.data() + c.off_fval);
        const int32_t *fint = reinterpret_cast<const int32_t *>(blob.data() + c.off_fint);
        for (int k = 0; k < nn; ++k) {
            walls_host[(size_t)t * nn + k] = (int8_t)blob[c.off_walls + k];
            texts_host[(size_t)t * nn + k] = (int8_t)blob[c.off_texts + k];
            const int f = fidx[k];
            food_rewards_host[(size_t)t * nn + k] = f >= 0 ? fval[f] : 0.0;
            food_interval_host[(size_t)t * nn + k] = f >= 0 ? fint[f] : 0;
        }
        mgb_maze_task_scalars &s = scalars_host[t];
        s.start[0] = hd.start[0]; s.start[1] = hd.start[1]; s.goal[0] = hd.goal[0]; s.goal[1] = hd.goal[1];
        s.cell_size = hd.cell_size; s.wall_height = hd.wall_height; s.agent_height = hd.agent_height;
        s.initial_life = hd.initial_life; s.max_life = hd.max_life; s.step_reward = hd.step_reward; s.goal_reward = hd.goal_reward;
    }
    return MGB_OK;
}

static int maze_ready(const mgb_maze *h)
{
    if (!h->has_task) { mgb_set_error("Must call \"set_task\" before reset"); return MGB_ERR_STATE; }   // maze_env.py:49-50
    if (h->c.kind != MGB_MAZE_2D && !h->has_tex) {
        mgb_set_error("3-D maze: call mgb_maze_set_textures first");
        return MGB_ERR_STATE;
    }
    return MGB_OK;
}

// pose_index + c_fmask + c_vbase -> one PoseRec per (task, cell, heading), for the `per` = n * n * 4 entries of each task
// of the region
__global__ void maze_pose_rec_kernel(const __grid_constant__ MazeArgs a, PoseRec *rec, int64_t per, int64_t count)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const int64_t k = i / per, idx = (int64_t)a.region[k] * per + (i - k * per);
    PoseRec r;
    r.slot = a.pose_index[idx]; r.vbase = -1; r.fmask[0] = r.fmask[1] = 0; r.pad = 0;
    if (r.slot >= 0) {
        r.fmask[0] = a.c_fmask[(size_t)r.slot * 2]; r.fmask[1] = a.c_fmask[(size_t)r.slot * 2 + 1];
        if (a.c_vbase) r.vbase = a.c_vbase[r.slot];
    }
    rec[idx] = r;
}

// Raise a kernel's dynamic shared-memory opt-in to everything the device allows next to the kernel's static shared memory.
// The value does not depend on the calling handle, so handles (and host threads) cannot undo each other's setting.
template <class F> static cudaError_t maze_allow_max_dynamic_smem(F *kernel)
{
    cudaFuncAttributes fa;
    cudaError_t e = cudaFuncGetAttributes(&fa, kernel);
    if (e != cudaSuccess) return e;
    int dev = 0, optin = 0;
    if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
    if ((e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) return e;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
}

template <bool FILL, bool ROLL = false, bool FIN = false, bool RS = false, bool EXP = false>
static int launch_render(mgb_maze *h, const MazeArgs &a, unsigned grid, cudaStream_t st, const MazeResample &rs = {},
                         const MazeExpertOr<EXP> &x = {})
{
    MazeConst &c = h->c;
    // shared-memory plan, most wanted first: (direct renderer) two record sets with the crossing lists in shared memory,
    // two record sets with the lists in a global scratch, then one record set (the only plan of the FILL pass)
    size_t sm = 0;
    const int plans[4][2] = {{1, 0}, {1, 1}, {0, 0}, {0, 1}};           // {pipe, hits_in_global}
    for (int k = 0; k < 4; ++k) {
        if (plans[k][0] && (FILL || !h->render_pipe)) continue;
        c.pipe = plans[k][0]; c.hits_in_global = plans[k][1];
        sm = maze3d_smem_bytes(c, FILL, RS);
        if (sm <= 227 * 1024) break;
    }
    if (sm > 227 * 1024) {
        mgb_set_error("3-D maze needs %zu bytes of shared memory per CTA (> 227 KB): reduce textures/resolution", sm);
        return MGB_ERR_ARG;
    }
    MazeArgs a2 = a;
    if (c.hits_in_global) {
        const size_t need = (size_t)grid * (c.pipe ? 2 : 1) * c.res_h * c.max_hits * sizeof(HitRec);
        if (need > h->hit_scratch_bytes) {
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
                mgb_set_error("maze renderer scratch must be allocated before stream capture: call reset() once first");
                return MGB_ERR_STATE;
            }
            MGB_CUDA(cudaStreamSynchronize(st));
            h->hit_scratch_bytes = 0;                   // alloc() frees the smaller scratch first
            MGB_CUDA(h->hit_scratch.alloc(need));
            h->hit_scratch_bytes = need;
        }
        a2.hit_scratch = h->hit_scratch.get();
    }
    // The opt-in limit is a property of the kernel on a device, shared by every handle: each handle raises it once to the
    // device maximum (the same value from every handle and thread, so there is no ordering to get wrong and no global state).
    const int attr = (EXP ? 8 : 0) + (RS ? 4 : 0) + (FIN ? 3 : (ROLL ? 2 : (FILL ? 1 : 0)));
    if (!h->render_attr_set[attr]) {
        MGB_CUDA(maze_allow_max_dynamic_smem(maze3d_kernel<FILL, ROLL, FIN, RS, EXP>));
        h->render_attr_set[attr] = 1;
    }
    h->smem3d = sm;
    maze3d_kernel<FILL, ROLL, FIN, RS, EXP><<<grid, kRenderThreads, sm, st>>>(c, a2, rs, x);
    MGB_CUDA(cudaGetLastError());
    return MGB_OK;
}

// Bytes of the pose cache of the handle's task table (slot-strided: n_tasks x S pose slots), and whether the cache can
// serve it: within the budget, and every lit texel fits the 10 bits per channel c_px packs.  Floor and ceiling texels are
// lit by v_screen / l_focal (ray_caster_utils.py:99,132), up to (half_v - pixel_size / 2) / l_focal; times the brightest
// texel that can pass 1023 on tall screens, and those screens render directly.
static bool pose_cache_fits(const mgb_maze *h, double &bytes)
{
    const MazeConst &c = h->c;
    const size_t slots = h->host_poses.size(), px = (size_t)c.res_h * c.res_v;
    bytes = (double)slots * (px * (c.obs_dtype == MGB_OBS_U8 ? 8.0 : 12.0) + px / 4.0 + 16.0 +
                             c.res_h * (1.0 + (double)c.max_hits * sizeof(HitRec)));
    const bool packs = (c.half_v - 0.5 * c.pixel_size) / c.l_focal * h->tex_max < 1024.0;
    return bytes <= h->cache_budget_gb * 1e9 && packs;
}

// Whether the pose cache draws the handle's frames: a discrete 3-D table, the cache on, and pose_cache_fits.  Everything
// it reads is host state that set_task, set_textures, update_tasks and set_cache keep current, so every call decides the
// same way before and after the first reset() builds the cache.
static bool pose_cache_serves(const mgb_maze *h)
{
    double bytes;
    return h->c.kind == MGB_MAZE_DISCRETE_3D && h->cache_enabled && !h->host_poses.empty() && pose_cache_fits(h, bytes);
}

// screens whose columns are whole 4-pixel groups get signatures, baked all-present frames and (uint8 SURVIVAL) variant frames
static bool cache_bakes(const MazeConst &c)
{
    const size_t px = (size_t)c.res_h * c.res_v;
    return (c.res_v & 3) == 0 && (px & 127) == 0;
}
static bool cache_has_variants(const mgb_maze *h)
{
    const MazeConst &c = h->c;
    return cache_bakes(c) && h->variant_bits > 0 && c.obs_dtype == MGB_OBS_U8 && c.task_type == MGB_MAZE_SURVIVAL &&
           ((size_t)c.res_h * c.res_v * 3) % 16 == 0;
}

// The build of the cache region of K tasks (a.region, a bound to the cache), one path for the whole table and for the tasks
// update_tasks replaced, in two halves around the first build's read-back of c_fmask.  First half: the FILL pass over the
// n_fill pose slots a.fill_slot lists, then their signatures.  Grids come from host-known sizes (K S, K V); region items a
// task does not have exit at once.
static int render_region(mgb_maze *h, const MazeArgs &a, int K, int64_t n_fill, cudaStream_t st)
{
    MazeArgs af = a;
    af.n = n_fill;
    af.do_step = 0;
    // the grid depends on K S, not n_fill: the first build (every task) sizes the renderer's scratch for every later region
    const int64_t span = (int64_t)K * h->pose_stride;
    int rc = launch_render<true>(h, af, (unsigned)(span < h->num_sms ? span : h->num_sms), st);
    if (rc) return rc;
    h->launches += 1;
    if (cache_bakes(h->c)) {
        maze3d_sig_kernel<<<(unsigned)n_fill, 256, 0, st>>>(h->c, af);
        MGB_CUDA(cudaGetLastError());
        h->launches += 1;
    }
    return MGB_OK;
}

// Second half: variant planning (device), the variant frames' static copies, the all-present bake (compose kernel, one
// synthetic env per pose slot, every food present), each variant's tints, then the tasks' PoseRec rows.
static int bake_region(mgb_maze *h, MazePoseCache &pc, MazeArgs a, int K, cudaStream_t st)
{
    const MazeConst &c = h->c;
    const int64_t S = h->pose_stride, V = h->var_stride;
    a.pose_stride = (int)S; a.var_stride = (int)V; a.var_bits = h->variant_bits_used; a.task_frames = pc.task_frames.get();
    if (cache_bakes(c)) {
        if (pc.c_vbase) {
            maze3d_plan_kernel<<<(unsigned)K, 32, 0, st>>>(a, pc.c_vbase.get(), pc.bake_desc.get(), pc.task_frames.get());
            MGB_CUDA(cudaGetLastError());
            MazeArgs av = a;
            av.bake_desc = pc.bake_desc.get(); av.region_ext = (int)V;
            maze3d_varinit_kernel<<<(unsigned)(K * V), 256, 0, st>>>(c, av);      // static colours first ...
            MGB_CUDA(cudaGetLastError());
            h->launches += 2;
        }
        MazeArgs ab = a;
        ab.bake = 1; ab.do_parts = 1; ab.region_ext = (int)S; ab.n = K * S;
        maze3d_compose_kernel<true><<<(unsigned)(K * S), kComposeThreads, 0, st>>>(c, ab);
        MGB_CUDA(cudaGetLastError());
        h->launches += 1;
        if (pc.c_vbase) {                                 // ... then each variant's tints
            ab.region_ext = (int)V; ab.n = K * V;
            ab.c_rgb8 = pc.c_var8.get(); ab.bake_desc = pc.bake_desc.get();
            maze3d_compose_kernel<true><<<(unsigned)(K * V), kComposeThreads, 0, st>>>(c, ab);
            MGB_CUDA(cudaGetLastError());
            h->launches += 1;
        }
    }
    const int64_t per = (int64_t)c.n * c.n * 4, count = K * per;     // merged per-pose records, after c_fmask and c_vbase
    maze_pose_rec_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(a, pc.pose_rec.get(), per, count);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// (Re)build the pose cache when tasks or textures changed: every free cell x 4 headings of every task is rendered once
// into its static layers.  Skipped (direct renderer used instead) when disabled or over the memory budget.
static int ensure_pose_cache(mgb_maze *h, cudaStream_t st)
{
    if (!h->cache_dirty) return MGB_OK;
    h->cache_ready = false;
    MazeConst &c = h->c;
    if (!pose_cache_serves(h)) {          // a decision, not a failure: cache_info then reports no cache
        h->cache_dirty = false;
        h->variant_bits_used = 0; h->var_stride = 0; h->var_planned = false; h->cache_bytes = 0.0;
        return MGB_OK;
    }
    const size_t slots = h->host_poses.size(), px = (size_t)c.res_h * c.res_v;
    double bytes;
    pose_cache_fits(h, bytes);
    // From here on a failure (capture in progress, out of memory) leaves cache_dirty set: the next call retries instead of
    // silently rendering every frame with the slow direct renderer (round-1 advice).
    // cudaMalloc/cudaFree synchronise; a capture in progress cannot build the cache
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs != cudaStreamCaptureStatusNone) {
        mgb_set_error("maze pose cache must be built before stream capture: call reset() once first");
        return MGB_ERR_STATE;
    }
    // the old cache goes before the new one (up to the whole budget) is built in `pc`, the handle's once it is complete
    h->cache = MazePoseCache();
    MazePoseCache pc;
    MGB_CUDA(pc.poses.alloc(slots * sizeof(int4)));
    MGB_CUDA(pc.pose_index.alloc(h->host_pose_index.size() * sizeof(int32_t)));
    MGB_CUDA(pc.c_px.alloc(slots * px * sizeof(uint32_t)));
    MGB_CUDA(pc.c_fid.alloc(slots * px));
    MGB_CUDA(pc.c_colhits.alloc(slots * c.res_h));
    MGB_CUDA(pc.c_hits.alloc(slots * c.res_h * c.max_hits * sizeof(HitRec)));
    MGB_CUDA(pc.dyn.alloc((size_t)h->n_pad * sizeof(EnvDyn)));
    MGB_CUDA(pc.c_rgb8.alloc(slots * px * 3));
    MGB_CUDA(pc.c_gsig.alloc(slots * ((px + 3) / 4)));
    MGB_CUDA(cudaMemsetAsync(pc.c_gsig.get(), 0xFF, slots * ((px + 3) / 4), st));
    MGB_CUDA(pc.c_fmask.alloc(slots * 2 * sizeof(uint64_t)));
    // screens the 4-pixel-group path cannot take keep an all-ones mask, i.e. never use the baked frame; the others get
    // every used slot's mask from the signature kernel
    if (!cache_bakes(c)) MGB_CUDA(cudaMemsetAsync(pc.c_fmask.get(), 0xFF, slots * 2 * sizeof(uint64_t), st));
    if (c.obs_dtype != MGB_OBS_U8) MGB_CUDA(pc.c_px_all.alloc(slots * px * sizeof(uint32_t)));
    MGB_CUDA(pc.task_frames.alloc((size_t)h->n_tasks * sizeof(int32_t)));
    MGB_CUDA(cudaMemsetAsync(pc.task_frames.get(), 0, (size_t)h->n_tasks * sizeof(int32_t), st));
    MGB_CUDA(pc.pose_rec.alloc(h->host_pose_index.size() * sizeof(PoseRec)));
    MGB_CUDA(cudaMemcpy(pc.poses.get(), h->host_poses.data(), slots * sizeof(int4), cudaMemcpyHostToDevice));
    MGB_CUDA(cudaMemcpy(pc.pose_index.get(), h->host_pose_index.data(), h->host_pose_index.size() * sizeof(int32_t),
                        cudaMemcpyHostToDevice));
    // the region of the whole table: every task slot, every used pose slot
    const int K = h->n_tasks;
    const int64_t S = h->pose_stride;
    std::vector<int32_t> region((size_t)K), fill;
    for (int t = 0; t < K; ++t) {
        region[t] = t;
        for (int j = 0; j < h->task_poses[t]; ++j) fill.push_back((int32_t)(t * S + j));
    }
    MgbDev<int32_t> d_region, d_fill;
    MGB_CUDA(d_region.alloc(region.size() * sizeof(int32_t)));
    MGB_CUDA(d_fill.alloc(fill.size() * sizeof(int32_t)));
    MGB_CUDA(cudaMemcpy(d_region.get(), region.data(), region.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    MGB_CUDA(cudaMemcpy(d_fill.get(), fill.data(), fill.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    MazeArgs a = maze_args(h);
    bind_pose_cache(pc, a);
    a.region = d_region.get(); a.fill_slot = d_fill.get();
    int rc = render_region(h, a, K, (int64_t)fill.size(), st);
    if (rc) return rc;
    // ---- variant frames: every pose whose image depends on k <= variant_bits foods gets its other 2^k - 1 finished frames
    // too (the all-visible one is c_rgb8[slot]).  Each task slot gets V frames, V = the most frames a task of this table
    // needs at the largest bits whose n_tasks x V frames fit the budget; the device plans them per task (maze3d_plan_kernel).
    h->variant_bits_used = 0;
    h->var_stride = 0;
    h->var_planned = cache_has_variants(h);
    if (h->var_planned) {
        std::vector<uint64_t> fm(slots * 2);
        MGB_CUDA(cudaStreamSynchronize(st));
        MGB_CUDA(cudaMemcpy(fm.data(), pc.c_fmask.get(), slots * 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        std::vector<int64_t> k_tasks((size_t)K * (kVariantBitsMax + 1), 0);     // [task][k] poses depending on k foods
        for (size_t sl = 0; sl < slots; ++sl) {
            if (h->host_poses[sl].x < 0) continue;
            const int k = __builtin_popcountll(fm[2 * sl]) + __builtin_popcountll(fm[2 * sl + 1]);
            if (k <= kVariantBitsMax) k_tasks[(size_t)(sl / S) * (kVariantBitsMax + 1) + k] += 1;
        }
        int bits = h->variant_bits;
        const double room = h->cache_budget_gb * 1e9 - bytes;
        int64_t V = 0;
        for (; bits > 0; --bits) {                         // largest k whose frames fit the cache budget
            V = 0;
            for (int t = 0; t < K; ++t) {
                int64_t frames = 0;
                for (int k = 1; k <= bits; ++k) frames += k_tasks[(size_t)t * (kVariantBitsMax + 1) + k] * (((int64_t)1 << k) - 1);
                V = frames > V ? frames : V;
            }
            if ((double)K * (double)V * (double)(px * 3) <= room) break;
        }
        h->variant_bits_used = bits;
        if (bits > 0 && V > 0) {
            h->var_stride = V;
            MGB_CUDA(pc.c_vbase.alloc(slots * sizeof(int32_t)));
            MGB_CUDA(pc.c_var8.alloc((size_t)K * V * px * 3));
            MGB_CUDA(pc.bake_desc.alloc((size_t)K * V * sizeof(BakeDesc)));
            a.c_vbase = pc.c_vbase.get(); a.c_var8 = pc.c_var8.get();
        }
    }
    rc = bake_region(h, pc, a, K, st);
    if (rc) return rc;
    MGB_CUDA(cudaStreamSynchronize(st));
    h->cache = std::move(pc);
    h->n_poses = (int64_t)fill.size();
    h->cache_bytes = bytes + (double)K * (double)h->var_stride * (double)(px * 3);
    h->cache_ready = true;
    h->cache_dirty = false;
    return MGB_OK;
}

// Paths other than the fused step keep their terminal states in a list (mgb_maze_step): clear its length, and leave
// a.final_obs to the list pass, which step_ex launches after the step.  `listed`: a list was started.
static int start_terminal_list(mgb_maze *h, MazeArgs &a, bool &listed, cudaStream_t st)
{
    listed = a.fin_count != nullptr;
    a.final_obs = nullptr;
    if (!listed) return MGB_OK;
    MGB_CUDA(cudaMemsetAsync(a.fin_count, 0, sizeof(int32_t), st));
    h->launches += 1;
    return MGB_OK;
}

// Resident CTAs of maze3d_compose_kernel on the handle's device (occupancy queried once per handle)
static int64_t compose_resident_ctas(mgb_maze *h)
{
    int &ctas_per_sm = h->compose_ctas_per_sm;
    if (!ctas_per_sm) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, maze3d_compose_kernel<false>, kComposeThreads, 0) !=
                cudaSuccess || ctas_per_sm < 1) ctas_per_sm = 4;
    }
    return (int64_t)h->num_sms * ctas_per_sm;
}

// Observe (a.do_step = 0) or step then observe every env.  `listed`: the step left its finished envs' terminal states in
// the list for step_ex's list pass.
static int launch_observe(mgb_maze *h, MazeArgs &a, bool &listed, cudaStream_t st)
{
    listed = false;
    const MazeConst &c = h->c;
    if (c.kind == MGB_MAZE_2D) {
        const int W = 2 * c.view_grid + 1;
        const size_t sm = (size_t)k2dThreads * W * W * 4;
        if (sm > 48 * 1024 && sm > h->m2d_smem_set) {      // view_grid >= 5: above the default dynamic shared-memory limit
            MGB_REQUIRE(sm <= 200 * 1024, "view_grid too large for the 2-D observation tile");
            MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_kernel));   // the device maximum: the same value from every handle
            h->m2d_smem_set = sm;
        }
        maze2d_kernel<<<(unsigned)((h->n + k2dThreads - 1) / k2dThreads), k2dThreads, sm, st>>>(c, a);
    } else {
        int rc = ensure_pose_cache(h, st);
        if (rc) return rc;
        if (h->cache_ready) {
            // memoised path: integer step logic, then compose static pose layers with the current food state
            bind_pose_cache(h->cache, a);
            // uint8 frames whose columns are whole 16-pixel runs: ONE fused launch (logic + TMA-moved frame)
            const size_t frame_bytes = (size_t)c.res_h * c.res_v * 3;
            if (h->fused_step && c.obs_dtype == MGB_OBS_U8 && (c.res_v & 15) == 0 && ((size_t)c.res_h * c.res_v) % 128 == 0 &&
                frame_bytes <= (size_t)64 * kStepChunkPx * 3 &&
                ((reinterpret_cast<uintptr_t>(a.obs) | reinterpret_cast<uintptr_t>(a.final_obs)) & 15u) == 0) {
                const size_t ring_bytes = (size_t)kStepSlots * kStepChunkPx * 3;       // 96 KB: two CTAs per SM
                if (h->step_smem_set == 0) {
                    MGB_CUDA(maze_allow_max_dynamic_smem(maze3d_step_kernel<false>));
                    MGB_CUDA(maze_allow_max_dynamic_smem(maze3d_step_kernel<true>));
                    h->step_smem_set = ring_bytes;
                }
                const int64_t grid = (int64_t)h->num_sms * 2;
                // terminal frames in the same launch
                const unsigned ctas = (unsigned)(h->n < grid ? h->n : grid);
                if (a.path) maze3d_step_kernel<true><<<ctas, kStepThreads, ring_bytes, st>>>(c, a);
                else maze3d_step_kernel<false><<<ctas, kStepThreads, ring_bytes, st>>>(c, a);
                MGB_CUDA(cudaGetLastError());
                h->launches += 1;
                return MGB_OK;
            }
            rc = start_terminal_list(h, a, listed, st);
            if (rc) return rc;
            maze3d_logic_kernel<true><<<(unsigned)((h->n + 127) / 128), 128, 0, st>>>(c, a);
            MGB_CUDA(cudaGetLastError());
            int64_t parts = (4 * compose_resident_ctas(h) + h->n - 1) / h->n;   // aim at >= 4 work items per resident CTA
            parts = parts < 1 ? 1 : (parts > 4 ? 4 : parts);
            a.do_parts = (int)parts;
            maze3d_compose_kernel<false><<<(unsigned)(h->n * parts), kComposeThreads, 0, st>>>(c, a);   // one CTA per item
            h->launches += 1;
        } else {
            rc = start_terminal_list(h, a, listed, st);
            if (rc) return rc;
            a.fin_dyn = nullptr;                                    // terminal list: full states for the direct renderer
            if (a.do_step && c.kind == MGB_MAZE_DISCRETE_3D) {     // logic for all envs in parallel, then render only
                maze3d_logic_kernel<false><<<(unsigned)((h->n + 127) / 128), 128, 0, st>>>(c, a);
                MGB_CUDA(cudaGetLastError());
                h->launches += 1;
                a.do_step = 0;
            }
            rc = launch_render<false>(h, a, (unsigned)(h->n < h->num_sms ? h->n : h->num_sms), st);
            if (rc) return rc;
        }
    }
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// One step with the optional outputs of mgb_maze_step (obs, rew, done and the state are exactly what they are without
// them).  2-D: the step kernel writes the terminal windows itself.  Fused 3-D step: the terminal frames are extra frames of
// the same launch.  Other 3-D paths: the step logic appends each finished env's terminal state to a list before resetting
// it, then one more launch renders the list into final_obs: the compose kernel over the terminal EnvDyn records on the pose
// cache, the direct renderer over the terminal states otherwise.  The list pass reads its length on the device; its grid
// is fixed, and its work is one frame per finished env.
static int step_ex(mgb_maze *h, MazeArgs &a, void *final_obs, uint8_t *truncated, cudaStream_t st)
{
    a.truncated = truncated;
    a.final_obs = final_obs;
    const MazeFinal &fin = h->tasks.fin;
    if (final_obs && h->c.kind != MGB_MAZE_2D) {
        a.fin_count = fin.count.get(); a.fin_env = fin.env.get(); a.fin_dyn = fin.dyn.get();
        a.fin_agent = fin.agent.get(); a.fin_life = fin.life.get(); a.fin_eaten = fin.eaten.get(); a.fin_task = fin.task.get();
        a.fin_cpos = fin.cpos.get(); a.fin_cori = fin.cori.get();
    }
    bool listed;
    int rc = launch_observe(h, a, listed, st);
    if (rc || !listed) return rc;
    MazeArgs l = maze_args(h);
    l.obs = final_obs; l.final_obs = final_obs; l.do_step = 0;
    l.path = nullptr;                                           // the list holds terminal copies, not env state
    l.fin_count = fin.count.get(); l.fin_env = fin.env.get();
    if (h->cache_ready) {
        l.dyn = fin.dyn.get();
        l.do_parts = 16;     // a few frames per step: slices spread each over many CTAs, so the pass costs a slice, not a frame
        const int64_t resident = compose_resident_ctas(h);
        maze3d_compose_kernel<false><<<(unsigned)(h->n < resident ? h->n : resident), kComposeThreads, 0, st>>>(h->c, l);
        MGB_CUDA(cudaGetLastError());
    } else {
        l.agent = fin.agent.get(); l.life = fin.life.get(); l.eaten = fin.eaten.get(); l.env2task = fin.task.get();
        l.cpos = fin.cpos.get(); l.cori = fin.cori.get();
        rc = launch_render<false>(h, l, (unsigned)(h->n < h->num_sms ? h->n : h->num_sms), st);
        if (rc) return rc;
    }
    h->launches += 1;
    return MGB_OK;
}

// A trial handle's counts after a launch that wrote done [T][n] without resampling (maze_count_done_kernel)
static int count_done(mgb_maze *h, const uint8_t *done_dev, int32_t T, cudaStream_t st)
{
    if (!h->trial_k) return MGB_OK;
    maze_count_done_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, st>>>(h->n, T, done_dev, h->task_count.get());
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// What a trial handle needs of a step or rollout without resampling: the refusal, or nullptr
static const char *trial_needs_done(const mgb_maze *h, const void *done_dev)
{
    return h->trial_k && !done_dev ? "a trial handle counts episodes from done: done_dev may not be null without resampling"
                                   : nullptr;
}

extern "C" int mgb_maze_reset(mgb_maze *h, const uint8_t *mask_dev, void *obs_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_reset");
    MGB_REQUIRE(h, "null handle");
    int rc = maze_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    MazeArgs a = maze_args(h);
    a.mask = mask_dev;
    maze_reset_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, st>>>(h->c, a, nullptr);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    if (obs_dev) {
        a.obs = obs_dev; a.do_step = 0; a.mask = nullptr;
        bool listed;
        return launch_observe(h, a, listed, st);
    }
    return MGB_OK;
}

// The checks of every rollout entry point, in the order it makes them: the handle, T, the entry point's own checks
// (own() returns the refusal, or nullptr), the optional outputs, then the handle's state.  Refusals are made as `fn`.
template <class Own>
static int check_rollout(const char *fn, const mgb_maze *h, int32_t T, const void *final_obs, const void *truncated, Own own)
{
    if (!h) return maze_refuse(fn, "null handle");
    if (T <= 0) return maze_refuse(fn, "T must be positive");
    if (const char *why = own()) return maze_refuse(fn, why);
    if (final_obs && !h->auto_reset)
        return maze_refuse(fn, "final_obs needs auto_reset on (without it obs already is the terminal frame)");
    if ((final_obs || truncated) && h->mir.count != 0)
        return maze_refuse(fn, "final_obs / truncated are not delivered through output mirrors or multicast (set_mirrors([]) first)");
    return maze_ready(h);
}

// maze2d_rollout_kernel<xm, fin, REC> over the handle's envs (xm: 0 plain, 1 peer mirrors, 2 multicast; fin: XM 0 only);
// with rs (xm 0 only): maze2d_rollout_kernel<0, fin, REC, true>, whose sm includes the sampler workspaces
template <bool REC>
static int launch_2d_rollout(const MazeConst &c, int xm, bool fin, const MazeArgs &a, unsigned blocks, size_t sm,
                             cudaStream_t st, const MazeResample *rs = nullptr)
{
    if (rs) {
        if (sm > 48 * 1024) {
            MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_rollout_kernel<0, false, REC, true>));
            MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_rollout_kernel<0, true, REC, true>));
        }
        if (fin) maze2d_rollout_kernel<0, true, REC, true><<<blocks, k2dThreads, sm, st>>>(c, a, *rs, MgbMlp{}, mgb_critic{}, MazeNoExpert{});
        else maze2d_rollout_kernel<0, false, REC, true><<<blocks, k2dThreads, sm, st>>>(c, a, *rs, MgbMlp{}, mgb_critic{}, MazeNoExpert{});
        MGB_CUDA(cudaGetLastError());
        return MGB_OK;
    }
    if (sm > 48 * 1024) {
        MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_rollout_kernel<0, false, REC>));
        MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_rollout_kernel<1, false, REC>));
        MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_rollout_kernel<2, false, REC>));
        MGB_CUDA(maze_allow_max_dynamic_smem(maze2d_rollout_kernel<0, true, REC>));
    }
    const MazeResample none = {};
    if (xm == 2) maze2d_rollout_kernel<2, false, REC><<<blocks, k2dThreads, sm, st>>>(c, a, none, MgbMlp{}, mgb_critic{}, MazeNoExpert{});
    else if (xm == 1) maze2d_rollout_kernel<1, false, REC><<<blocks, k2dThreads, sm, st>>>(c, a, none, MgbMlp{}, mgb_critic{}, MazeNoExpert{});
    else if (fin) maze2d_rollout_kernel<0, true, REC><<<blocks, k2dThreads, sm, st>>>(c, a, none, MgbMlp{}, mgb_critic{}, MazeNoExpert{});
    else maze2d_rollout_kernel<0, false, REC><<<blocks, k2dThreads, sm, st>>>(c, a, none, MgbMlp{}, mgb_critic{}, MazeNoExpert{});
    MGB_CUDA(cudaGetLastError());
    return MGB_OK;
}

// The engine mgb_maze_rollout runs for the handle: the 2-D rollout kernel for MetaMaze2D; for MetaMazeDiscrete3D without
// resampling the pose cache when ensure_pose_cache leaves it ready (the choice launch_observe makes for a step); the direct
// raycaster otherwise.  It builds the pose cache when one is due, so it runs after every check that does not depend on
// the engine.
enum class RolloutEngine { grid2d, pose_cache, direct };

static int rollout_engine(mgb_maze *h, bool resample, cudaStream_t st, RolloutEngine &eng)
{
    eng = h->c.kind == MGB_MAZE_2D ? RolloutEngine::grid2d : RolloutEngine::direct;
    if (h->c.kind != MGB_MAZE_DISCRETE_3D || resample) return MGB_OK;
    const int rc = ensure_pose_cache(h, st);
    if (rc == MGB_OK && h->cache_ready) eng = RolloutEngine::pose_cache;
    return rc;
}

// Dynamic shared memory of a 2-D rollout CTA in front of a policy's region: two observation tiles and, when resampling,
// one sampler workspace per warp (16-byte multiples), rounded up to 16 bytes
static size_t maze2d_tiles_bytes(const mgb_maze *h, bool resample)
{
    const int W = 2 * h->c.view_grid + 1;
    size_t sm = (size_t)2 * k2dThreads * W * W * 4;
    if (resample) sm += (size_t)(k2dThreads / 32) * sampler_ws_bytes(h->c.n);
    return (sm + 15) / 16 * 16;
}

extern "C" int mgb_maze_rollout(mgb_maze *h, int32_t T, const void *act_dev, uint64_t act_seed, void *act_out_dev,
                                void *obs_dev, double *rew_dev, uint8_t *done_dev, void *final_obs_dev,
                                uint8_t *truncated_dev, const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                                void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout");
    SamplerCfg sc;
    int rc = check_rollout(__func__, h, T, final_obs_dev, truncated_dev, [&]() -> const char * {
        if (h->c.kind != MGB_MAZE_2D && h->mir.count != 0)
            return "output mirrors are not implemented for the 3-D rollouts (set_mirrors([]) first)";
        if (!resample_cfg) return trial_needs_done(h, done_dev);
        if (h->expert) return kExpertNoInLaunchResampling;
        if (!h->auto_reset) return "resampling finished envs needs auto_reset on";
        if (h->mir.count != 0)
            return "output mirrors and multicast are not implemented for the resampling rollout (set_mirrors([]) first)";
        return sampler_cfg(h, resample_cfg, sc);
    });
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    const cudaStream_t st = (cudaStream_t)stream;
    RolloutEngine eng;
    rc = rollout_engine(h, resample_cfg != nullptr, st, eng);
    if (rc) return rc;
    if (eng == RolloutEngine::direct && !(obs_dev && rew_dev && done_dev)) return maze_refuse(__func__, "null argument");
    MazeArgs a = maze_args(h);
    if (h->c.kind == MGB_MAZE_CONTINUOUS_3D) {
        a.act_c = static_cast<const float *>(act_dev); a.act_out_c = static_cast<float *>(act_out_dev);
    } else {
        a.act = static_cast<const int32_t *>(act_dev); a.act_out = static_cast<int32_t *>(act_out_dev);
    }
    a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev; a.do_step = 1;
    a.T = T; a.act_seed = act_seed; a.t_base = h->t_base;
    a.final_obs = final_obs_dev; a.truncated = truncated_dev;
    const bool fin = final_obs_dev || truncated_dev;
    MazeResample r = {};
    if (resample_cfg) {
        r.cfg = sc; r.seed = resample_seed; r.epoch = h->task_epoch.get();
        r.count = h->task_count.get(); r.k = h->trial_k;
    }
    if (eng == RolloutEngine::pose_cache) {
        const int64_t resident = (int64_t)h->num_sms * 5;          // __launch_bounds__(256, 5): 48 registers
        const size_t qbytes = ((size_t)h->c.res_h * h->c.res_v / 4 + 1) * sizeof(int);
        MGB_REQUIRE(qbytes <= 200 * 1024, "screen too large for the fused rollout's group queue");
        const unsigned grid = (unsigned)(h->n < resident ? h->n : resident);
        if (fin) {
            if (qbytes > 40 * 1024)
                MGB_CUDA(maze_allow_max_dynamic_smem(maze3d_rollout_kernel<true>));
            maze3d_rollout_kernel<true><<<grid, kComposeThreads, qbytes, st>>>(h->c, a, MazeNoExpert{});
        } else {
            if (qbytes > 40 * 1024)
                MGB_CUDA(maze_allow_max_dynamic_smem(maze3d_rollout_kernel<false>));
            maze3d_rollout_kernel<false><<<grid, kComposeThreads, qbytes, st>>>(h->c, a, MazeNoExpert{});
        }
        MGB_CUDA(cudaGetLastError());
    } else if (eng == RolloutEngine::direct) {
        const unsigned grid = (unsigned)(h->n < h->num_sms ? h->n : h->num_sms);
        if (fin)
            rc = resample_cfg ? launch_render<false, true, true, true>(h, a, grid, st, r)
                              : launch_render<false, true, true>(h, a, grid, st);
        else
            rc = resample_cfg ? launch_render<false, true, false, true>(h, a, grid, st, r)
                              : launch_render<false, true>(h, a, grid, st);
    } else if (resample_cfg) {
        const size_t sm = maze2d_tiles_bytes(h, true);
        int optin = 0;
        MGB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
        if (sm > (size_t)optin) {
            mgb_set_error("%s: the resampling rollout needs %zu bytes of shared memory per CTA at n = %d and view_grid = %d, "
                          "more than the %d the device allows (use a smaller view_grid)", __func__, sm, h->c.n,
                          h->c.view_grid, optin);
            return MGB_ERR_ARG;
        }
        const unsigned blocks = (unsigned)((h->n + k2dThreads - 1) / k2dThreads);
        rc = h->path ? launch_2d_rollout<true>(h->c, 0, fin, a, blocks, sm, st, &r)
                     : launch_2d_rollout<false>(h->c, 0, fin, a, blocks, sm, st, &r);
    } else {
        if (h->mir.count != 0)
            MGB_REQUIRE(h->mir_win.holds_rollout((uint64_t)T * h->n, obs_dev, (uint64_t)mgb_maze_obs_bytes_per_env(h),
                                                 rew_dev, 8, done_dev, act_out_dev, 4),
                        "mirrors are on but an output lies outside the mirrored arena (set_mirrors([]) first)");
        if (h->mir.count == MGB_MIRROR_MULTICAST) {
            MGB_REQUIRE(h->n % 4 == 0, "multicast outputs need num_envs % 4 == 0");
            MGB_REQUIRE((((uintptr_t)done_dev | (uintptr_t)obs_dev | (uintptr_t)act_out_dev) & 3) == 0 && ((uintptr_t)rew_dev & 7) == 0,
                        "multicast outputs must be 4-byte (rewards: 8-byte) aligned");
        }
        a.mir = h->mir;
        const size_t sm = maze2d_tiles_bytes(h, false);
        const unsigned blocks = (unsigned)((h->n + k2dThreads - 1) / k2dThreads);
        const int xm = h->mir.count == MGB_MIRROR_MULTICAST ? 2 : (h->mir.count > 0 ? 1 : 0);
        rc = h->path ? launch_2d_rollout<true>(h->c, xm, fin, a, blocks, sm, st)
                     : launch_2d_rollout<false>(h->c, xm, fin, a, blocks, sm, st);
    }
    if (rc) return rc;
    h->t_base += (uint32_t)T;
    h->launches += 1;
    return resample_cfg ? MGB_OK : count_done(h, done_dev, T, st);
}

// ---------------------------------------------------------------------------------------------------------------
// ESCAPE expert entry points (include/mgb200.h "Expert")
// ---------------------------------------------------------------------------------------------------------------
// What every expert entry point needs of the handle: the refusal, or nullptr
static const char *expert_refusal(const mgb_maze *h)
{
    if (h->c.task_type != MGB_MAZE_ESCAPE) return "the expert is defined for ESCAPE only (SURVIVAL has no single shortest-path target)";
    if (h->c.kind == MGB_MAZE_CONTINUOUS_3D)
        return "the expert is defined for the grid mazes only (MetaMazeContinuous3D has continuous actions)";
    if (!h->expert) return "not an expert handle (mgb_maze_set_expert before mgb_maze_set_task)";
    if (h->mir.count != 0) return "expert outputs are not delivered through output mirrors or multicast (set_mirrors([]) first)";
    return nullptr;
}

template <bool FIN>
static int launch_2d_expert(mgb_maze *h, const MazeArgs &a, const MazeExpert &x, cudaStream_t st)
{
    const size_t sm = maze2d_tiles_bytes(h, false);
    const unsigned blocks = (unsigned)((h->n + k2dThreads - 1) / k2dThreads);
    const auto kernel = h->path ? maze2d_rollout_kernel<0, FIN, true, false, 0, false, false, true>
                                : maze2d_rollout_kernel<0, FIN, false, false, 0, false, false, true>;
    if (sm > 48 * 1024) MGB_CUDA(maze_allow_max_dynamic_smem(kernel));
    kernel<<<blocks, k2dThreads, sm, st>>>(h->c, a, MazeResample{}, MgbMlp{}, mgb_critic{}, x);
    MGB_CUDA(cudaGetLastError());
    return MGB_OK;
}

extern "C" int mgb_maze_rollout_expert(mgb_maze *h, int32_t T, const int32_t *act_dev, float eps, int32_t mode,
                                       uint64_t seed, int32_t *act_out_dev, uint8_t *expert_out_dev, void *obs_dev,
                                       double *rew_dev, uint8_t *done_dev, void *final_obs_dev, uint8_t *truncated_dev,
                                       void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_expert");
    int rc = check_rollout(__func__, h, T, final_obs_dev, truncated_dev, [&]() -> const char * {
        if (const char *why = expert_refusal(h)) return why;
        if (!(eps >= 0.0f && eps <= 1.0f)) return "eps must be finite and in [0, 1]";
        if (mode != 0 && mode != 1) return "mode must be 0 (sample) or 1 (mean)";
        if (!(obs_dev && rew_dev && done_dev)) return "null argument (obs, rew and done are required)";
        return nullptr;
    });
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    const cudaStream_t st = (cudaStream_t)stream;
    RolloutEngine eng;
    if ((rc = rollout_engine(h, false, st, eng))) return rc;
    MazeArgs a = maze_args(h);
    a.act = act_dev; a.act_out = act_out_dev;
    a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev; a.do_step = 1;
    a.T = T; a.t_base = h->t_base;
    a.final_obs = final_obs_dev; a.truncated = truncated_dev;
    const bool fin = final_obs_dev || truncated_dev;
    MazeExpert x;
    x.mask = h->exp_mask.get(); x.out = expert_out_dev; x.eps = eps; x.mean = mode; x.seed = seed;
    if (eng == RolloutEngine::pose_cache) {
        const int64_t resident = (int64_t)h->num_sms * 5;
        const size_t qbytes = ((size_t)h->c.res_h * h->c.res_v / 4 + 1) * sizeof(int);
        MGB_REQUIRE(qbytes <= 200 * 1024, "screen too large for the fused rollout's group queue");
        const unsigned grid = (unsigned)(h->n < resident ? h->n : resident);
        const auto kernel = fin ? maze3d_rollout_kernel<true, true> : maze3d_rollout_kernel<false, true>;
        if (qbytes > 40 * 1024) MGB_CUDA(maze_allow_max_dynamic_smem(kernel));
        kernel<<<grid, kComposeThreads, qbytes, st>>>(h->c, a, x);
        MGB_CUDA(cudaGetLastError());
    } else if (eng == RolloutEngine::direct) {
        const unsigned grid = (unsigned)(h->n < h->num_sms ? h->n : h->num_sms);
        rc = fin ? launch_render<false, true, true, false, true>(h, a, grid, st, {}, x)
                 : launch_render<false, true, false, false, true>(h, a, grid, st, {}, x);
    } else {
        rc = fin ? launch_2d_expert<true>(h, a, x, st) : launch_2d_expert<false>(h, a, x, st);
    }
    if (rc) return rc;
    h->t_base += (uint32_t)T;
    h->launches += 1;
    return count_done(h, done_dev, T, st);
}

extern "C" int mgb_maze_expert(mgb_maze *h, uint8_t *mask_out_dev, uint16_t *dist_out_dev, void *stream)
{
    if (!h) return maze_refuse(__func__, "null handle");
    if (const char *why = expert_refusal(h)) return maze_refuse(__func__, why);
    if (!mask_out_dev) return maze_refuse(__func__, "null argument (mask_out is required)");
    if (int rc = maze_ready(h)) return rc;
    MgbDeviceGuard guard(h->device);
    maze_expert_state_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        h->c, maze_args(h), h->exp_mask.get(), h->exp_dist.get(), mask_out_dev, dist_out_dev);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

extern "C" int mgb_maze_step_expert(mgb_maze *h, const int32_t *act_dev, void *obs_dev, double *rew_dev, uint8_t *done_dev,
                                    void *final_obs_dev, uint8_t *truncated_dev, uint8_t *expert_out_dev, void *stream)
{
    if (!h) return maze_refuse(__func__, "null handle");
    if (const char *why = expert_refusal(h)) return maze_refuse(__func__, why);
    if (!expert_out_dev) return maze_refuse(__func__, "null argument (expert_out is required)");
    int rc = mgb_maze_step(h, act_dev, obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev, stream);
    return rc ? rc : mgb_maze_expert(h, expert_out_dev, nullptr, stream);
}

extern "C" int mgb_maze_expert_table(mgb_maze *h, int32_t slot0, int32_t count, uint8_t *mask_out_dev,
                                     uint16_t *dist_out_dev, void *stream)
{
    if (!h) return maze_refuse(__func__, "null handle");
    if (const char *why = expert_refusal(h)) return maze_refuse(__func__, why);
    if (!mask_out_dev) return maze_refuse(__func__, "null argument (mask_out is required)");
    if (int rc = maze_ready(h)) return rc;
    if (!(slot0 >= 0 && count > 0 && (int64_t)slot0 + count <= h->n_tasks))
        return maze_refuse(__func__, "slots [slot0, slot0 + count) must lie in the task table");
    MgbDeviceGuard guard(h->device);
    const size_t per = (size_t)expert_planes(h->c.kind) * h->c.n * h->c.n;
    const cudaStream_t st = (cudaStream_t)stream;
    MGB_CUDA(cudaMemcpyAsync(mask_out_dev, h->exp_mask.get() + slot0 * per, count * per, cudaMemcpyDeviceToDevice, st));
    if (dist_out_dev)
        MGB_CUDA(cudaMemcpyAsync(dist_out_dev, h->exp_dist.get() + slot0 * per, count * per * sizeof(uint16_t),
                                 cudaMemcpyDeviceToDevice, st));
    return MGB_OK;
}

// maze2d_rollout_kernel<0, fin, REC, RS, POL>, sm bytes of dynamic shared memory; refused (as `fn`) when the CTA would
// need more shared memory than the device allows
// (with a critic: maze2d_rollout_kernel<0, true, REC, RS, POL, true>; with ev, mgb_maze_evaluate:
// maze2d_rollout_kernel<0, false, REC, RS, POL, false, true>)
template <bool REC, bool RS, int POL>
static int launch_2d_policy(const char *fn, const mgb_maze *h, bool fin, const MazeArgs &a, const MazeResample &r,
                            const MgbPolicyPlan<POL> &m, unsigned blocks, size_t sm, cudaStream_t st,
                            const mgb_critic *critic, const MgbEval *ev = nullptr)
{
    // the launch of `kernel`, whose last parameter is `last` (the critic, or the evaluation's outputs)
    const auto launch = [&](auto kernel, const auto &last) -> int {
        int optin = 0;
        MGB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
        cudaFuncAttributes fa;
        MGB_CUDA(cudaFuncGetAttributes(&fa, kernel));
        if (fa.sharedSizeBytes + sm > (size_t)optin) {
            mgb_set_error("%s: the policy rollout needs %zu bytes of shared memory per CTA (windows of "
                          "view_grid %d, %sweights and activations of %d envs), more than the %d the device allows (use a "
                          "smaller view_grid or narrower layers)", fn, fa.sharedSizeBytes + sm, h->c.view_grid,
                          RS ? "sampler workspaces, " : "", k2dThreads, optin);
            return MGB_ERR_ARG;
        }
        MGB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        kernel<<<blocks, k2dThreads, sm, st>>>(h->c, a, r, m, last, MazeNoExpert{});
        MGB_CUDA(cudaGetLastError());
        return MGB_OK;
    };
    if (ev) return launch(maze2d_rollout_kernel<0, false, REC, RS, POL, false, true>, *ev);
    const auto kernel = critic ? maze2d_rollout_kernel<0, true, REC, RS, POL, true>
                        : fin  ? maze2d_rollout_kernel<0, true, REC, RS, POL>
                               : maze2d_rollout_kernel<0, false, REC, RS, POL>;
    return launch(kernel, critic ? *critic : mgb_critic{});
}

// A policy rollout of kind POL (mgb_maze_rollout_policy, mgb_maze_rollout_rnn) with the plan `pol`.  The checks, in
// order: the handle, T, the handle kind, then own(observation width) (the entry point plans the policy into pol and
// makes its own checks; it returns the refusal, or nullptr), the population (one member: nothing to refuse), logp_out
// in the mean mode, mirrors, resampling, the
// optional outputs and the handle's state.  The policy's region of dynamic shared memory follows the tiles and the
// sampler workspaces.
// A critic (the *_critic entry points, whose own() plans the value row; null for the others) is checked last.
// With ev (mgb_maze_evaluate, which passes no per-step output) the launch is the EVAL instantiation over the step bound
// T, and a trial handle without resampling has its episodes counted in the launch instead of from done.
template <int POL, class Own>
static int maze_rollout_policy(const char *fn, mgb_maze *h, int32_t T, MgbPolicyPlan<POL> &pol, Own own,
                               int32_t members, int64_t member_stride, uint64_t seed,
                               const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed, int32_t *act_out_dev,
                               float *logp_out_dev, float *obs0_out_dev, float *obs_dev, double *rew_dev,
                               uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev, void *stream,
                               bool val = false, const mgb_critic *critic = nullptr, const MgbEval *ev = nullptr)
{
    MgbMlp &head = mgb_policy_head(pol);
    SamplerCfg sc;
    int rc = check_rollout(fn, h, T, final_obs_dev, truncated_dev, [&]() -> const char * {
        if (h->c.kind != MGB_MAZE_2D)
            return POL == kPolMlp ? "mgb_maze_rollout_policy serves MetaMaze2D (the 3-D envs observe frames)"
                                  : "mgb_maze_rollout_rnn serves MetaMaze2D (the 3-D envs observe frames)";
        const int W = 2 * h->c.view_grid + 1;
        if (const char *why = own(W * W)) return why;
        if (const char *why = mgb_population_plan(head, h->n, members, member_stride, k2dThreads)) return why;
        if (logp_out_dev && head.mode != MGB_POLICY_SAMPLE) return "logp_out needs MGB_POLICY_SAMPLE (the mean mode draws nothing)";
        if (h->mir.count != 0)
            return "policy rollouts are not delivered through output mirrors or multicast (set_mirrors([]) first)";
        if (!resample_cfg) {
            if (const char *why = ev ? nullptr : trial_needs_done(h, done_dev)) return why;
        } else {
            if (h->expert) return kExpertNoInLaunchResampling;                            // as mgb_maze_rollout
            if (!h->auto_reset) return "resampling finished envs needs auto_reset on";     // as mgb_maze_rollout
            if (const char *why = sampler_cfg(h, resample_cfg, sc)) return why;
        }
        return val ? mgb_critic_check(critic, h->auto_reset, rew_dev, done_dev, truncated_dev) : nullptr;
    });
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    const size_t base = maze2d_tiles_bytes(h, resample_cfg != nullptr);
    pol.smem_off = (int)(base / 4);
    head.seed = seed;
    head.logp_out = logp_out_dev;
    head.obs0_out = obs0_out_dev;
    size_t sm = base;
    if constexpr (POL == kPolMlp) sm += mgb_mlp_smem_bytes(pol, k2dThreads);
    else sm += mgb_rnn_smem_bytes(pol, k2dThreads);
    MazeArgs a = maze_args(h);
    a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev; a.do_step = 1;
    a.T = T; a.t_base = h->t_base; a.act_out = act_out_dev;
    a.final_obs = final_obs_dev; a.truncated = truncated_dev;
    MazeResample r = {};
    if (resample_cfg) {
        r.cfg = sc; r.seed = resample_seed; r.epoch = h->task_epoch.get();
        r.count = h->task_count.get(); r.k = h->trial_k;
    } else if (ev && h->trial_k) {
        r.count = h->task_count.get();
    }
    const bool fin = final_obs_dev || truncated_dev;
    const unsigned blocks = (unsigned)((h->n + k2dThreads - 1) / k2dThreads);
    const cudaStream_t st = (cudaStream_t)stream;
    const mgb_critic *cr = val ? critic : nullptr;
    if (resample_cfg)
        rc = h->path ? launch_2d_policy<true, true, POL>(fn, h, fin, a, r, pol, blocks, sm, st, cr, ev)
                     : launch_2d_policy<false, true, POL>(fn, h, fin, a, r, pol, blocks, sm, st, cr, ev);
    else
        rc = h->path ? launch_2d_policy<true, false, POL>(fn, h, fin, a, r, pol, blocks, sm, st, cr, ev)
                     : launch_2d_policy<false, false, POL>(fn, h, fin, a, r, pol, blocks, sm, st, cr, ev);
    if (rc) return rc;
    h->t_base += (uint32_t)T;
    h->launches += 1;
    return resample_cfg || ev ? MGB_OK : count_done(h, done_dev, T, st);
}

// mgb_maze_rollout_policy of `members` policies (one: mgb_maze_rollout_policy), refused as `fn`
static int maze_rollout_mlp(const char *fn, mgb_maze *h, int32_t T, const mgb_policy *pol, int32_t members,
                            int64_t member_stride, uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg,
                            uint64_t resample_seed, int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                            float *obs_dev, double *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                            uint8_t *truncated_dev, void *stream, bool val = false, const mgb_critic *critic = nullptr,
                            const MgbEval *ev = nullptr, bool value_row = false)
{
    MgbMlp m;
    const auto own = [&](int obs_dim) { return mgb_mlp_plan(pol, obs_dim, false, m, val || value_row); };
    return maze_rollout_policy<kPolMlp>(fn, h, T, m, own, members, member_stride, seed, resample_cfg, resample_seed,
                                        act_out_dev, logp_out_dev, obs0_out_dev, obs_dev, rew_dev, done_dev,
                                        final_obs_dev, truncated_dev, stream, val, critic, ev);
}

extern "C" int mgb_maze_rollout_policy(mgb_maze *h, int32_t T, const mgb_policy *pol, uint64_t seed,
                                       const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                                       int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev, float *obs_dev,
                                       double *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                                       void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_policy");
    return maze_rollout_mlp(__func__, h, T, pol, 1, 0, seed, resample_cfg, resample_seed, act_out_dev, logp_out_dev,
                            obs0_out_dev, obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev, stream);
}

extern "C" int mgb_maze_rollout_population(mgb_maze *h, int32_t T, const mgb_policy *pol, int32_t members,
                                           int64_t member_stride, uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg,
                                           uint64_t resample_seed, int32_t *act_out_dev, float *logp_out_dev,
                                           float *obs0_out_dev, float *obs_dev, double *rew_dev, uint8_t *done_dev,
                                           float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_population");
    return maze_rollout_mlp(__func__, h, T, pol, members, member_stride, seed, resample_cfg, resample_seed, act_out_dev,
                            logp_out_dev, obs0_out_dev, obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev, stream);
}

// mgb_maze_rollout_rnn of `members` policies (one: mgb_maze_rollout_rnn), refused as `fn`
static int maze_rollout_rnn(const char *fn, mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                            int64_t member_stride, uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg,
                            uint64_t resample_seed, float *state_dev, float *state0_out_dev, float *hid_out_dev,
                            int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev, float *obs_dev,
                            double *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev,
                            void *stream, bool val = false, const mgb_critic *critic = nullptr,
                            const MgbEval *ev = nullptr, bool value_row = false)
{
    // the same rollout for either cell: kind is std::integral_constant<int, kPolGru or kPolLstm>
    const auto run = [&](auto kind) {
        constexpr int POL = decltype(kind)::value;
        MgbPolicyPlan<POL> p;
        const auto own = [&](int obs_dim) -> const char * {
            if (const char *why = mgb_rnn_plan(pol, obs_dim, p, val || value_row)) return why;
            p.state = state_dev;
            p.state0_out = state0_out_dev;
            p.hid_out = hid_out_dev;
            if (!state_dev) return "null state";
            if ((uintptr_t)state_dev % sizeof(float)) return "state must be 4-byte aligned";
            if (!h->auto_reset) return "the recurrent rollout needs auto_reset on (an episode boundary has no next step without it)";
            return nullptr;
        };
        return maze_rollout_policy<POL>(fn, h, T, p, own, members, member_stride, seed, resample_cfg, resample_seed,
                                        act_out_dev, logp_out_dev, obs0_out_dev, obs_dev, rew_dev, done_dev,
                                        final_obs_dev, truncated_dev, stream, val, critic, ev);
    };
    return pol && pol->cell == MGB_RNN_CELL_LSTM ? run(std::integral_constant<int, kPolLstm>{})
                                                 : run(std::integral_constant<int, kPolGru>{});
}

extern "C" int mgb_maze_rollout_rnn(mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, uint64_t seed,
                                    const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                                    float *state_dev, float *state0_out_dev, float *hid_out_dev,
                                    int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                                    float *obs_dev, double *rew_dev, uint8_t *done_dev,
                                    float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_rnn");
    return maze_rollout_rnn(__func__, h, T, pol, 1, 0, seed, resample_cfg, resample_seed, state_dev, state0_out_dev,
                            hid_out_dev, act_out_dev, logp_out_dev, obs0_out_dev, obs_dev, rew_dev, done_dev,
                            final_obs_dev, truncated_dev, stream);
}

extern "C" int mgb_maze_rollout_rnn_population(mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                                               int64_t member_stride, uint64_t seed,
                                               const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                                               float *state_dev, float *state0_out_dev, float *hid_out_dev,
                                               int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                                               float *obs_dev, double *rew_dev, uint8_t *done_dev,
                                               float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_rnn_population");
    return maze_rollout_rnn(__func__, h, T, pol, members, member_stride, seed, resample_cfg, resample_seed, state_dev,
                            state0_out_dev, hid_out_dev, act_out_dev, logp_out_dev, obs0_out_dev, obs_dev, rew_dev,
                            done_dev, final_obs_dev, truncated_dev, stream);
}

extern "C" int mgb_maze_rollout_critic(mgb_maze *h, int32_t T, const mgb_policy *pol, int32_t members,
                                       int64_t member_stride, uint64_t seed, const mgb_maze_sampler_cfg *resample_cfg,
                                       uint64_t resample_seed, int32_t *act_out_dev, float *logp_out_dev,
                                       float *obs0_out_dev, float *obs_dev, double *rew_dev, uint8_t *done_dev,
                                       float *final_obs_dev, uint8_t *truncated_dev, const mgb_critic *critic,
                                       void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_critic");
    return maze_rollout_mlp(__func__, h, T, pol, members, member_stride, seed, resample_cfg, resample_seed, act_out_dev,
                            logp_out_dev, obs0_out_dev, obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev, stream,
                            true, critic);
}

extern "C" int mgb_maze_rollout_rnn_critic(mgb_maze *h, int32_t T, const mgb_rnn_policy *pol, int32_t members,
                                           int64_t member_stride, uint64_t seed,
                                           const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed,
                                           float *state_dev, float *state0_out_dev, float *hid_out_dev,
                                           int32_t *act_out_dev, float *logp_out_dev, float *obs0_out_dev,
                                           float *obs_dev, double *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                                           uint8_t *truncated_dev, const mgb_critic *critic, void *stream)
{
    MgbRange nvtx_range("mgb_maze_rollout_rnn_critic");
    return maze_rollout_rnn(__func__, h, T, pol, members, member_stride, seed, resample_cfg, resample_seed, state_dev,
                            state0_out_dev, hid_out_dev, act_out_dev, logp_out_dev, obs0_out_dev, obs_dev, rew_dev,
                            done_dev, final_obs_dev, truncated_dev, stream, true, critic);
}

extern "C" int mgb_maze_evaluate(mgb_maze *h, int32_t episodes, const mgb_policy *mlp, const mgb_rnn_policy *rnn,
                                 int32_t value_row, int32_t members, int64_t member_stride, uint64_t seed,
                                 const mgb_maze_sampler_cfg *resample_cfg, uint64_t resample_seed, float *state_dev,
                                 double *return_dev, int32_t *length_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_evaluate");
    int32_t T = 0;
    const char *why = !h ? "null handle"
                      : h->c.kind != MGB_MAZE_2D ? "mgb_maze_evaluate serves MetaMaze2D (the 3-D envs have no policy path)"
                      : mgb_eval_check(episodes, h->c.max_steps, h->auto_reset, mlp, rnn, state_dev, value_row,
                                       return_dev, length_dev, truncated_dev, T);
    if (why) return maze_refuse(__func__, why);
    const MgbEval ev = {return_dev, length_dev, truncated_dev, episodes};
    if (mlp)
        return maze_rollout_mlp(__func__, h, T, mlp, members, member_stride, seed, resample_cfg, resample_seed, nullptr,
                                nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, stream, false, nullptr,
                                &ev, value_row != 0);
    return maze_rollout_rnn(__func__, h, T, rnn, members, member_stride, seed, resample_cfg, resample_seed, state_dev,
                            nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                            stream, false, nullptr, &ev, value_row != 0);
}

extern "C" int mgb_maze_set_mirrors(mgb_maze *h, int count, const int64_t *byte_delta)
{
    MGB_REQUIRE(h, "null handle");
    const char *why = h->mir.set_peers(count, byte_delta);
    MGB_REQUIRE(!why, why);
    return MGB_OK;
}

extern "C" int mgb_maze_set_mirror_window(mgb_maze *h, const void *base, uint64_t bytes)
{
    MGB_REQUIRE(h, "null handle");
    h->mir_win.set(base, bytes);
    return MGB_OK;
}

extern "C" int mgb_maze_set_multicast(mgb_maze *h, int64_t byte_delta)
{
    MGB_REQUIRE(h, "null handle");
    const char *why = h->mir.set_multicast(byte_delta);
    MGB_REQUIRE(!why, why);
    return MGB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// God view: the right-hand panel of the reference window (MazeBase.render_init + render_update, maze_base.py:100-157,
// with the agent marker of maze_2d.py:73-75, maze_discrete_3d.py:83-99 and maze_continuous_3d.py:58-74) for many envs per
// launch.  One CTA (or a few, for small batches) per env: the env's cells and the pixel -> cell tables are staged in shared
// memory, then every thread colours 16 pixels at a time and stores them as three 16-byte words.  The pixel rules (rect by
// pixel centre, disc and Bresenham line on truncated coordinates) are DESIGN.md "God view"; oracle/maze_godview.py states
// them again in numpy.  The trajectory view (MazeBase.render_trajectory, maze_base.py:159-189) is the same kernel in its
// trajectory mode followed by maze_god_path_kernel, which draws the recorded path as width-3 lines
// (tests/trajectory_view.py restates that picture).
// ---------------------------------------------------------------------------------------------------------------
namespace {

constexpr int kGodThreads = 256;
constexpr int kGodPx = 16;                       // pixels per item: 48 bytes, three 16-byte stores
constexpr int kGodMaxView = 4096;
constexpr uint32_t kGodNone = 0xFFFFFFFFu;       // colours are 0x00BBGGRR: the bytes leave in R, G, B order
constexpr uint32_t kGodWhite = 0xFFFFFFu, kGodBlack = 0u, kGodGreen = 0x00FF00u, kGodRed = 0x0000FFu;

struct GodEnv {
    int valid;                   // 0: env index out of range, the frame is written as zeros
    int gx, gy;                  // 2-D: the red agent cell
    int dcx, dcy, dr2;           // 3-D: disc centre and squared radius (dr2 < 0: nothing drawn)
    int lx0, ly0, lx1, ly1;      // 3-D: heading line end points
    int bx0, by0, bx1, by1;      // 3-D: bounding box of disc and line (empty for 2-D)
};

// int() of a screen coordinate; far-off values are clamped so that the integer arithmetic below cannot overflow
__device__ __forceinline__ int god_trunc(double v)
{
    return (int)(v < -1.0e9 ? -1.0e9 : (v > 1.0e9 ? 1.0e9 : v));
}

// Bresenham: the major axis steps by one from the start point; at step i the minor offset is i d_minor / d_major rounded
// half up (a tie moves toward the end point)
__device__ __forceinline__ bool god_on_line(int px, int py, const GodEnv &g)
{
    const int dx = abs(g.lx1 - g.lx0), dy = abs(g.ly1 - g.ly0);
    const int sx = g.lx1 >= g.lx0 ? 1 : -1, sy = g.ly1 >= g.ly0 ? 1 : -1;
    if (dx >= dy) {
        const int i = (px - g.lx0) * sx;
        if (i < 0 || i > dx) return false;
        if (dx == 0) return py == g.ly0;
        return py == g.ly0 + sy * (int)((2LL * i * dy + dx) / (2LL * dx));
    }
    const int i = (py - g.ly0) * sy;
    if (i < 0 || i > dy) return false;
    return px == g.lx0 + sx * (int)((2LL * i * dx + dy) / (2LL * dy));
}

__device__ __forceinline__ void god_push(char2 &v, int cell)
{
    if (v.x < 0) v.x = (char)cell; else if (v.y < 0) v.y = (char)cell;
}

// The agent marker of one env in panel coordinates, typed like the reference computes it: the discrete 3-D env and a
// continuous env at reset hold python floats as position (float64) and the continuous env's position after a step is a
// float32 array, so `agent_pos = pos * pos_conversion` and `agent_pos + view_size` are float32 there; after a step the
// discrete heading is a float32 table entry, so its cos / sin and `ori_size * cos` are float32 too.  Right after a reset
// both 3-D envs have the heading 0.0 that MazeBase.reset leaves.
// heading: cos / sin of the four float32 heading table entries (computed once on the host, mgb_maze_god_view).
__device__ void god_marker(const MazeConst &c, const MazeArgs &a, const TaskHdr *th, int64_t e, int S,
                           const float4 &hcos, const float4 &hsin, GodEnv &g)
{
    const int4 ag = a.agent[e];
    g.gx = ag.x; g.gy = ag.y;
    g.dr2 = -1;
    g.bx0 = g.by0 = 1; g.bx1 = g.by1 = 0;
    if (c.kind == MGB_MAZE_2D) return;
    const double rcs = (double)S / (double)c.n;                   // render_init: view_size / self._n
    const double pc = rcs / th->cell_size;                        // self._pos_conversion
    const double ori_size = 0.60 * pc;
    double cx, cy, ex, ey;
    if (c.kind == MGB_MAZE_CONTINUOUS_3D && ag.w > 0) {
        const float2 p = a.cpos[e];
        const float ax = p.x * (float)pc, ay = p.y * (float)pc;
        const float fcx = ax + (float)S, fcy = (float)S - ay;
        const double o = a.cori[e];
        cx = (double)fcx; cy = (double)fcy;
        ex = cx + ori_size * cos(o);
        ey = cy - ori_size * sin(o);
    } else {
        const double ax = (ag.x * th->cell_size + 0.5 * th->cell_size) * pc;   // get_cell_center, maze_base.py:194-197
        const double ay = (ag.y * th->cell_size + 0.5 * th->cell_size) * pc;
        cx = ax + (double)S; cy = (double)S - ay;
        if (c.kind == MGB_MAZE_DISCRETE_3D && ag.w > 0) {
            const int k = ag.z & 3;
            const float co = k == 0 ? hcos.x : (k == 1 ? hcos.y : (k == 2 ? hcos.z : hcos.w));
            const float si = k == 0 ? hsin.x : (k == 1 ? hsin.y : (k == 2 ? hsin.z : hsin.w));
            ex = cx + (double)((float)ori_size * co);
            ey = cy - (double)((float)ori_size * si);
        } else {                                                   // heading 0.0 after reset (maze_base.py:50)
            ex = cx + ori_size * 1.0;
            ey = cy - ori_size * 0.0;
        }
    }
    const int r = god_trunc(0.15 * pc);
    g.dcx = god_trunc(cx) - S; g.dcy = god_trunc(cy);
    g.dr2 = r >= 1 ? r * r : -1;
    g.lx0 = g.dcx; g.ly0 = g.dcy;
    g.lx1 = god_trunc(ex) - S; g.ly1 = god_trunc(ey);
    const int rr = r >= 1 ? r : 0;
    g.bx0 = min(min(g.lx0, g.lx1), g.dcx - rr); g.bx1 = max(max(g.lx0, g.lx1), g.dcx + rr);
    g.by0 = min(min(g.ly0, g.ly1), g.dcy - rr); g.by1 = max(max(g.ly0, g.ly1), g.dcy + rr);
}

__global__ void __launch_bounds__(kGodThreads) maze_god_view_kernel(const __grid_constant__ MazeConst c,
                                                                    const __grid_constant__ MazeArgs a,
                                                                    const int32_t *__restrict__ envs, int S,
                                                                    const float4 hcos, const float4 hsin,
                                                                    uint8_t *__restrict__ out, int traj)
{
    // traj: the panel of render_trajectory (maze_base.py:159-176) under its path lines: walls and goal, a red agent rect
    // at the current cell for every kind, then the food, all on the panel's own coordinates; no 3-D disc or heading line
    extern __shared__ __align__(16) uint32_t god_smem[];
    __shared__ GodEnv g;
    __shared__ uint4 stage[kGodThreads / 32][3 * 32];              // per warp: 32 items of 48 bytes, stored coalesced
    const int n = c.n, nn = n * n;
    uint32_t *base = god_smem;                                     // [nn] wall / goal colour or kGodNone
    uint32_t *food = god_smem + nn;                                // [nn] food colour or kGodNone
    uint32_t *cell = god_smem + 2 * nn;                            // [nn] final colour of a pixel inside this cell only
    char2 *xg = reinterpret_cast<char2 *>(god_smem + 3 * nn);      // [S] cells whose rect holds the pixel column (_surf_god)
    char2 *xs = xg + S;                                            // [S] the same for rects drawn on the screen (x + view_size)
    char2 *yc = xs + S;                                            // [S] cells whose rect holds the pixel row
    // [S] each: the one cell holding the column (in both xg and xs) / the row, or -1 when a pixel there can lie in none or
    // in two cells' rects (a cell edge within rounding of a pixel centre): such pixels take the general path
    int8_t *colx = reinterpret_cast<int8_t *>(yc + S);
    int8_t *rowy = colx + S;
    const int64_t k = blockIdx.x;
    const int64_t e = envs ? (int64_t)envs[k] : k;
    const bool valid = e >= 0 && e < a.n;
    const uint8_t *blob = valid ? a.blobs + (int64_t)a.env2task[e] * c.blob_bytes : nullptr;
    const TaskHdr *th = valid ? blob_hdr(blob) : nullptr;
    if (threadIdx.x == 0) {
        g.valid = valid;
        if (valid && traj) {
            const int4 ag = a.agent[e];
            g.gx = ag.x; g.gy = ag.y;
            g.dr2 = -1;
            g.bx0 = g.by0 = 1; g.bx1 = g.by1 = 0;
        } else if (valid) {
            god_marker(c, a, th, e, S, hcos, hsin, g);
        }
    }
    if (valid) {
        const int8_t *walls = reinterpret_cast<const int8_t *>(blob + c.off_walls);
        const int4 ag = a.agent[e];
        const int steps = ag.w;
        for (int i = threadIdx.x; i < nn; i += blockDim.x) {      // render_init (walls, ESCAPE goal) and draw_food
            const int x = i / n, y = i - x * n;
            uint32_t b = walls[i] > 0 ? kGodBlack : kGodNone;
            if (c.task_type == MGB_MAZE_ESCAPE && x == th->goal[0] && y == th->goal[1]) b = kGodGreen;
            uint32_t f = kGodNone;
            if (c.task_type == MGB_MAZE_SURVIVAL) {
                const double v = food_now(c, blob, a.eaten + e, a.n_pad, steps, i);
                if (v > 1.0e-2) {
                    const double fv = 255.0 - 255.0 * v;          // int(255 - 255 * food), clamped to a colour
                    const uint32_t q = fv <= 0.0 ? 0u : (fv >= 255.0 ? 255u : (uint32_t)fv);
                    f = q | (255u << 8) | (q << 16);
                }
            }
            base[i] = b; food[i] = f;
            const bool at_agent = x == ag.x && y == ag.y;
            uint32_t v;
            if (traj) {
                v = f != kGodNone ? f : (at_agent ? kGodRed : (b != kGodNone ? b : kGodWhite));
            } else {
                v = f != kGodNone ? f : (b != kGodNone ? b : kGodWhite);
                if (c.kind == MGB_MAZE_2D && at_agent) v = kGodRed;
            }
            cell[i] = v;
        }
        const double rcs = (double)S / (double)n;
        const double soff = traj ? 0.0 : (double)S;                // x offset of the rects drawn on the screen
        for (int p = threadIdx.x; p < S; p += blockDim.x) {
            const double pcen = (double)p + 0.5;
            const int cx0 = (int)(pcen / rcs), cy0 = (int)(((double)S - pcen) / rcs);   // y points up
            char2 vg = make_char2(-1, -1), vs = make_char2(-1, -1), vy = make_char2(-1, -1);
            for (int d = -1; d <= 1; ++d) {
                const int q = cx0 + d, r = cy0 + d;
                if (q >= 0 && q < n) {
                    const double x0 = q * rcs;                     // x * self._render_cell_size
                    if (x0 <= pcen && pcen < x0 + rcs) god_push(vg, q);
                    const double x1 = q * rcs + soff;              // ... + offset[0] (draw_food, the 2-D agent rect)
                    if (x1 <= pcen + soff && pcen + soff < x1 + rcs) god_push(vs, q);
                }
                if (r >= 0 && r < n) {
                    const double y0 = (double)S - (r + 1) * rcs;   // view_size - (y + 1) * self._render_cell_size
                    if (y0 <= pcen && pcen < y0 + rcs) god_push(vy, r);
                }
            }
            xg[p] = vg; xs[p] = vs; yc[p] = vy;
            colx[p] = (vg.x >= 0 && vg.y < 0 && vs.y < 0 && vs.x == vg.x) ? vg.x : (int8_t)-1;
            rowy[p] = (vy.x >= 0 && vy.y < 0) ? vy.x : (int8_t)-1;
        }
    }
    __syncthreads();
    const GodEnv ge = g;
    const bool is2d = c.kind == MGB_MAZE_2D, surv = c.task_type == MGB_MAZE_SURVIVAL;
    // every primitive that can cover the pixel, in the reference's draw order (used where a pixel is not inside one cell)
    auto general = [&](int row, int col) -> uint32_t {
        uint32_t v = kGodWhite;
        const char2 cy = yc[row], cg = xg[col], cs = xs[col];
        const int ys[2] = {cy.x, cy.y}, gs[2] = {cg.x, cg.y}, ss[2] = {cs.x, cs.y};
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                if (gs[i] >= 0 && ys[j] >= 0) {
                    const uint32_t b = base[gs[i] * n + ys[j]];
                    if (b != kGodNone) v = b;
                }
        if (traj && (gs[0] == ge.gx || gs[1] == ge.gx) && (ys[0] == ge.gy || ys[1] == ge.gy)) v = kGodRed;
        if (surv) {
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j)
                    if (ss[i] >= 0 && ys[j] >= 0) {
                        const uint32_t f = food[ss[i] * n + ys[j]];
                        if (f != kGodNone) v = f;
                    }
        }
        if (is2d && !traj && (ss[0] == ge.gx || ss[1] == ge.gx) && (ys[0] == ge.gy || ys[1] == ge.gy)) v = kGodRed;
        return v;
    };
    auto colour = [&](int row, int col, int cy) -> uint32_t {
        if (!ge.valid) return 0u;
        const int cx = colx[col];
        uint32_t v = (cx >= 0 && cy >= 0) ? cell[cx * n + cy] : general(row, col);
        if (col >= ge.bx0 && col <= ge.bx1 && row >= ge.by0 && row <= ge.by1) {    // 3-D agent marker
            const int64_t dx = col - ge.dcx, dy = row - ge.dcy;
            if (dx * dx + dy * dy <= (int64_t)ge.dr2 || god_on_line(col, row, ge)) v = kGodGreen;
        }
        return v;
    };
    const int64_t npx = (int64_t)S * S;
    uint8_t *frame = out + k * npx * 3;
    const int64_t items = (npx + kGodPx - 1) / kGodPx;
    const int64_t full = (reinterpret_cast<uintptr_t>(frame) & 15u) == 0 ? npx / kGodPx : 0;   // items stored as 16-byte words
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kGodThreads / 32;
    // a warp takes 32 consecutive items (1536 contiguous bytes): each lane colours 16 pixels, the warp's words go through
    // shared memory so that each of its three store instructions writes 512 contiguous bytes
    for (int64_t wb = ((int64_t)blockIdx.y * nwarps + warp) * 32; wb < items; wb += (int64_t)gridDim.y * nwarps * 32) {
        const int64_t it = wb + lane;
        if (it >= items) continue;
        const int64_t p0 = it * kGodPx;
        int row = (int)(p0 / S), col = (int)(p0 - (int64_t)row * S);
        uint32_t px[kGodPx];
        int cy = rowy[row];                                        // the row's cell, reloaded only where the row changes
#pragma unroll
        for (int j = 0; j < kGodPx; ++j) {
            px[j] = row < S ? colour(row, col, cy) : 0u;
            if (++col == S) { col = 0; ++row; cy = row < S ? rowy[row] : -1; }
        }
        if (it < full) {
            uint32_t w[12];
#pragma unroll
            for (int i = 0; i < 12; ++i) {
                uint32_t v = 0;
#pragma unroll
                for (int b = 0; b < 4; ++b) v |= ((px[(4 * i + b) / 3] >> (8 * ((4 * i + b) % 3))) & 0xFFu) << (8 * b);
                w[i] = v;
            }
            if (wb + 32 <= full) {                                 // warp-uniform: all 32 items are whole words
                stage[warp][3 * lane] = make_uint4(w[0], w[1], w[2], w[3]);
                stage[warp][3 * lane + 1] = make_uint4(w[4], w[5], w[6], w[7]);
                stage[warp][3 * lane + 2] = make_uint4(w[8], w[9], w[10], w[11]);
                __syncwarp();
                uint4 *dst = reinterpret_cast<uint4 *>(frame + wb * kGodPx * 3);
#pragma unroll
                for (int i = 0; i < 3; ++i) __stcs(dst + i * 32 + lane, stage[warp][i * 32 + lane]);
                __syncwarp();
            } else {
                uint4 *dst = reinterpret_cast<uint4 *>(frame + p0 * 3);
                __stcs(dst, make_uint4(w[0], w[1], w[2], w[3]));
                __stcs(dst + 1, make_uint4(w[4], w[5], w[6], w[7]));
                __stcs(dst + 2, make_uint4(w[8], w[9], w[10], w[11]));
            }
        } else {
            for (int j = 0; j < kGodPx && p0 + j < npx; ++j) {
                uint8_t *d = frame + (p0 + j) * 3;
                d[0] = (uint8_t)px[j]; d[1] = (uint8_t)(px[j] >> 8); d[2] = (uint8_t)(px[j] >> 16);
            }
        }
    }
}

// pygame.draw.line(surface, red, p, q, width=3) between the centres of cells (x0, y0) and (x1, y1): the Bresenham pixels of
// the truncated end points, each widened into a 3-pixel span across the minor axis (along x when |dx| <= |dy|, along y
// otherwise; a zero-length segment is one span).  Pixels outside the panel are dropped.
// Pixels i0, i0 + di, ... of the line: one thread walks a whole segment with (0, 1), a warp's lanes share one with
// (lane, 32), so that the warp's stores of a step lie side by side.
__device__ void god_wide_line(uint8_t *frame, int S, double rcs, int x0c, int y0c, int x1c, int y1c, int i0 = 0, int di = 1)
{
    const int x0 = god_trunc((x0c + 0.5) * rcs), y0 = god_trunc((double)S - (y0c + 0.5) * rcs);
    const int x1 = god_trunc((x1c + 0.5) * rcs), y1 = god_trunc((double)S - (y1c + 0.5) * rcs);
    const int dx = abs(x1 - x0), dy = abs(y1 - y0);
    const int sx = x1 >= x0 ? 1 : -1, sy = y1 >= y0 ? 1 : -1;
    const bool span_x = dx <= dy;
    const int len = dx >= dy ? dx : dy;
    for (int i = i0; i <= len; i += di) {
        int px, py;
        if (dx >= dy) { px = x0 + sx * i; py = dx == 0 ? y0 : y0 + sy * (int)((2LL * i * dy + dx) / (2LL * dx)); }
        else { py = y0 + sy * i; px = x0 + sx * (int)((2LL * i * dx + dy) / (2LL * dy)); }
        for (int k = -1; k <= 1; ++k) {
            const int qx = span_x ? px + k : px, qy = span_x ? py : py + k;
            if (qx < 0 || qx >= S || qy < 0 || qy >= S) continue;
            uint8_t *d = frame + ((int64_t)qy * S + qx) * 3;
            d[0] = 255; d[1] = 0; d[2] = 0;
        }
    }
}

// The path lines of render_trajectory (maze_base.py:178-183) over the panel maze_god_view_kernel<traj> left in `out`: one
// CTA per env.  Every line is the same red, so the picture depends only on the set of distinct segments: segments between
// neighbouring cells (every discrete move) are collected as direction bits per cell in shared memory and drawn once each;
// longer ones (a continuous env crossing more than one cell in a step) are drawn where they are found.  A segment with an
// end that was never recorded ((-1, -1), recording switched on mid-episode) is skipped.
__global__ void __launch_bounds__(kGodThreads) maze_god_path_kernel(const __grid_constant__ MazeConst c,
                                                                    const __grid_constant__ MazeArgs a,
                                                                    const int32_t *__restrict__ envs, int S,
                                                                    uint8_t *__restrict__ out)
{
    __shared__ uint32_t s_dirs[kMaxN * kMaxN];     // bit (dy + 1) * 3 + dx + 1: the segment from the cell to (x + dx, y + dy)
    __shared__ uint16_t s_segs[kMaxN * kMaxN * 9]; // the set bits as cell * 9 + bit, in no particular order
    __shared__ int s_nseg;
    const int64_t k = blockIdx.x;
    const int64_t e = envs ? (int64_t)envs[k] : k;
    if (e < 0 || e >= a.n) return;                 // the frame stays all zero
    const int n = c.n, nn = n * n;
    for (int i = threadIdx.x; i < nn; i += blockDim.x) s_dirs[i] = 0u;
    if (threadIdx.x == 0) s_nseg = 0;
    __syncthreads();
    const int steps = a.agent[e].w;
    const int len = (steps < c.max_steps ? steps : c.max_steps) + 1;
    uint8_t *frame = out + k * (int64_t)S * S * 3;
    const double rcs = (double)S / (double)n;      // render_init: view_size / self._n
    for (int i = threadIdx.x; i + 1 < len; i += blockDim.x) {
        const char2 p = a.path[(int64_t)i * a.n_pad + e], q = a.path[(int64_t)(i + 1) * a.n_pad + e];
        if (p.x < 0 || p.y < 0 || q.x < 0 || q.y < 0) continue;
        const int dx = q.x - p.x, dy = q.y - p.y;
        if (dx >= -1 && dx <= 1 && dy >= -1 && dy <= 1 && p.x < n && p.y < n)
            atomicOr(&s_dirs[p.x * n + p.y], 1u << ((dy + 1) * 3 + dx + 1));
        else
            god_wide_line(frame, S, rcs, p.x, p.y, q.x, q.y);
    }
    __syncthreads();
    for (int cl = threadIdx.x; cl < nn; cl += blockDim.x) {
        uint32_t m = s_dirs[cl];
        if (!m) continue;
        int j = atomicAdd(&s_nseg, __popc(m));
        for (; m; m &= m - 1) s_segs[j++] = (uint16_t)(cl * 9 + __ffs(m) - 1);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nseg = s_nseg;
    for (int j = warp; j < nseg; j += kGodThreads / 32) {         // one warp per segment, lanes along it
        const int cl = s_segs[j] / 9, d = s_segs[j] - cl * 9;
        const int x = cl / n, y = cl - x * n;
        god_wide_line(frame, S, rcs, x, y, x + d % 3 - 1, y + d / 3 - 1, lane, 32);
    }
}

// mgb_maze_path: env envs[k]'s current-episode path -> cells[k][0 .. len), len[k]
__global__ void maze_path_kernel(const __grid_constant__ MazeConst c, const __grid_constant__ MazeArgs a,
                                 const int32_t *__restrict__ envs, int64_t cap, char2 *__restrict__ cells,
                                 int32_t *__restrict__ lens)
{
    const int64_t k = blockIdx.x;
    const int64_t e = envs ? (int64_t)envs[k] : k;
    int len = 0;
    if (e >= 0 && e < a.n) {
        const int steps = a.agent[e].w;
        len = (steps < c.max_steps ? steps : c.max_steps) + 1;
    }
    if (threadIdx.x == 0) lens[k] = len;
    for (int i = threadIdx.x; i < len; i += blockDim.x) cells[k * cap + i] = a.path[(int64_t)i * a.n_pad + e];
}

}  // namespace

extern "C" int mgb_maze_god_view(mgb_maze *h, int32_t count, const int32_t *envs_dev, int32_t view_size, int32_t mode,
                                 uint8_t *out_dev, void *stream)
{
    MGB_REQUIRE(h, "null argument");
    MGB_REQUIRE(mode == MGB_GOD_LIVE || mode == MGB_GOD_TRAJECTORY,
                "mgb_maze_god_view: mode must be MGB_GOD_LIVE or MGB_GOD_TRAJECTORY");
    MGB_REQUIRE(mode != MGB_GOD_TRAJECTORY || h->path,
                "mgb_maze_god_view: MGB_GOD_TRAJECTORY needs path recording (mgb_maze_set_path)");
    MGB_REQUIRE(count >= 0 && count <= INT_MAX / 2, "mgb_maze_god_view: count out of range");
    MGB_REQUIRE(view_size >= 1 && view_size <= kGodMaxView, "mgb_maze_god_view: view_size must be in [1, 4096]");
    MGB_REQUIRE(h->has_task, "mgb_maze_god_view: set a task first");
    if (count == 0) return MGB_OK;
    MGB_REQUIRE(out_dev, "mgb_maze_god_view: null output");
    MGB_REQUIRE(envs_dev || count <= h->n, "mgb_maze_god_view: count exceeds the env count (pass envs_dev)");
    MgbDeviceGuard guard(h->device);
    MazeArgs a = maze_args(h);
    const int64_t items = ((int64_t)view_size * view_size + kGodPx - 1) / kGodPx;
    // enough CTAs to fill the GPU when the batch is small; one CTA per env otherwise
    const int64_t want = (int64_t)(h->num_sms > 0 ? h->num_sms : 132) * 8;
    int64_t split = (want + count - 1) / count;
    const int64_t most = (items + kGodThreads - 1) / kGodThreads;
    split = split < most ? split : most;
    split = split < 65535 ? split : 65535;
    // maze_discrete_3d.py:46: float32 table entries k * 0.5 * PI, and numpy's float32 cos / sin of them.  Computed here so
    // that the kernel needs no device trig table (which would renumber the module's constant-bank entries that the other
    // kernels reference).
    float hc[4], hs[4];
    for (int k = 0; k < 4; ++k) {
        const float o = (float)(0.5 * k) * (float)3.1415926;
        hc[k] = cosf(o); hs[k] = sinf(o);
    }
    const size_t smem = (size_t)3 * h->c.n * h->c.n * 4 + (size_t)3 * view_size * sizeof(char2) + (size_t)2 * view_size;
    maze_god_view_kernel<<<dim3((unsigned)count, (unsigned)split), kGodThreads, smem, (cudaStream_t)stream>>>(
        h->c, a, envs_dev, view_size, make_float4(hc[0], hc[1], hc[2], hc[3]), make_float4(hs[0], hs[1], hs[2], hs[3]),
        out_dev, mode == MGB_GOD_TRAJECTORY);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    if (mode == MGB_GOD_TRAJECTORY) {
        maze_god_path_kernel<<<(unsigned)count, kGodThreads, 0, (cudaStream_t)stream>>>(h->c, a, envs_dev, view_size, out_dev);
        MGB_CUDA(cudaGetLastError());
        h->launches += 1;
    }
    return MGB_OK;
}

extern "C" int mgb_maze_path(mgb_maze *h, int32_t count, const int32_t *envs_dev, int8_t *cells_out, int32_t *len_out,
                             void *stream)
{
    MGB_REQUIRE(h, "null argument");
    MGB_REQUIRE(h->path, "mgb_maze_path: path recording is off (mgb_maze_set_path)");
    MGB_REQUIRE(count >= 0 && count <= INT_MAX / 2, "mgb_maze_path: count out of range");
    if (count == 0) return MGB_OK;
    MGB_REQUIRE(cells_out && len_out, "mgb_maze_path: null output");
    MGB_REQUIRE(envs_dev || count <= h->n, "mgb_maze_path: count exceeds the env count (pass envs_dev)");
    MgbDeviceGuard guard(h->device);
    maze_path_kernel<<<(unsigned)count, 256, 0, (cudaStream_t)stream>>>(h->c, maze_args(h), envs_dev, path_cap(h),
                                                                         reinterpret_cast<char2 *>(cells_out), len_out);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

__global__ void maze_pose_kernel(MazeArgs a, float *pos_out, double *ori_out)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const float2 p = a.cpos[e];
    pos_out[2 * e] = p.x; pos_out[2 * e + 1] = p.y;
    if (ori_out) ori_out[e] = a.cori[e];
}

extern "C" int mgb_maze_pose(mgb_maze *h, float *pos_dev, double *ori_dev, void *stream)
{
    MGB_REQUIRE(h && pos_dev, "null argument");
    MGB_REQUIRE(h->c.kind == MGB_MAZE_CONTINUOUS_3D, "mgb_maze_pose needs a MGB_MAZE_CONTINUOUS_3D handle");
    MgbDeviceGuard guard(h->device);
    MazeArgs a = maze_args(h);
    maze_pose_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, pos_dev, ori_dev);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// act_dev: float [n][2] for a MGB_MAZE_CONTINUOUS_3D handle, int32 [n] otherwise
extern "C" int mgb_maze_step(mgb_maze *h, const void *act_dev, void *obs_dev, double *rew_dev, uint8_t *done_dev,
                             void *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_step");
    MGB_REQUIRE(h && act_dev && obs_dev && rew_dev && done_dev, "null argument");
    int rc = maze_ready(h);
    if (rc) return rc;
    MGB_REQUIRE(!final_obs_dev || h->auto_reset,
                "final_obs needs auto_reset on (without it obs already is the terminal frame)");
    MgbDeviceGuard guard(h->device);
    MazeArgs a = maze_args(h);
    if (h->c.kind == MGB_MAZE_CONTINUOUS_3D) a.act_c = static_cast<const float *>(act_dev);
    else a.act = static_cast<const int32_t *>(act_dev);
    a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev; a.do_step = 1;
    rc = step_ex(h, a, final_obs_dev, truncated_dev, (cudaStream_t)stream);
    return rc ? rc : count_done(h, done_dev, 1, (cudaStream_t)stream);
}

extern "C" int mgb_maze_state(mgb_maze *h, int32_t *agent_dev, double *life_dev, void *stream)
{
    MGB_REQUIRE(h && agent_dev, "null argument");
    MgbDeviceGuard guard(h->device);
    MazeArgs a = maze_args(h);
    maze_state_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, agent_dev, life_dev);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Snapshot / restore records (DESIGN.md "Snapshot, restore and clone").  A record is
//   [0, 16)   agent int4 (gx, gy, ori, steps)
//   [16, 32)  life f64 | resample count u32 | task-table slot i32
//   [32, 48)  continuous position f32 x 2 | heading f64 (zero for the other kinds)
//   [48, ..)  food stamps int32 [f_max], in groups of four (16 bytes each, unused tail zero)
//   [.., +16) trial handles only: the env's episode count u32 | zero padding
//   [tail, ..) the task of the env's slot, blob_bytes, when records carry their tasks
//   [.., ..)  path recording on: the path entries char2 [max_steps + 1], padded to 16 bytes
// ---------------------------------------------------------------------------------------------------------------
namespace {

constexpr int64_t kMazeRecHead = 48;

__global__ void maze_snapshot_kernel(int f_max, const __grid_constant__ MazeArgs a, const uint32_t *__restrict__ epoch,
                                     const uint32_t *__restrict__ count, uint8_t *__restrict__ rec, int64_t rec_bytes)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    uint4 *r = reinterpret_cast<uint4 *>(rec + e * rec_bytes);
    const int4 ag = a.agent[e];
    const double life = a.life[e];
    r[0] = make_uint4((uint32_t)ag.x, (uint32_t)ag.y, (uint32_t)ag.z, (uint32_t)ag.w);
    r[1] = make_uint4((uint32_t)__double2loint(life), (uint32_t)__double2hiint(life), epoch ? epoch[e] : 0u,
                      (uint32_t)a.env2task[e]);
    const float2 p = a.cpos ? a.cpos[e] : make_float2(0.f, 0.f);
    const double o = a.cori ? a.cori[e] : 0.0;
    r[2] = make_uint4(__float_as_uint(p.x), __float_as_uint(p.y), (uint32_t)__double2loint(o), (uint32_t)__double2hiint(o));
    for (int f = 0; f < f_max; f += 4) {
        uint32_t v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = f + j < f_max ? (uint32_t)a.eaten[(int64_t)(f + j) * a.n_pad + e] : 0u;
        r[3 + f / 4] = make_uint4(v[0], v[1], v[2], v[3]);
    }
    if (count) r[3 + (f_max + 3) / 4] = make_uint4(count[e], 0u, 0u, 0u);
}

// env2task_w: null when records carry their tasks (the env keeps its own slot)
__global__ void maze_restore_kernel(int f_max, const __grid_constant__ MazeArgs a, uint32_t *__restrict__ epoch,
                                    uint32_t *__restrict__ count, int32_t *__restrict__ env2task_w, int n_tasks, const uint8_t *__restrict__ rec,
                                    int64_t rec_bytes, int64_t n_rec, const int64_t *__restrict__ row)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const int64_t rw = row[e];
    if (rw < 0 || rw >= n_rec) return;
    const uint4 *s = reinterpret_cast<const uint4 *>(rec + rw * rec_bytes);
    const uint4 h0 = s[0], h1 = s[1], h2 = s[2];
    a.agent[e] = make_int4((int)h0.x, (int)h0.y, (int)h0.z, (int)h0.w);
    a.life[e] = __hiloint2double((int)h1.y, (int)h1.x);
    epoch[e] = h1.z;
    if (env2task_w && (int)h1.w >= 0 && (int)h1.w < n_tasks) env2task_w[e] = (int)h1.w;
    if (a.cpos) {
        a.cpos[e] = make_float2(__uint_as_float(h2.x), __uint_as_float(h2.y));
        a.cori[e] = __hiloint2double((int)h2.w, (int)h2.z);
    }
    for (int f = 0; f < f_max; f += 4) {
        const uint4 u = s[3 + f / 4];
        const uint32_t v[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (f + j < f_max) a.eaten[(int64_t)(f + j) * a.n_pad + e] = (int32_t)v[j];
    }
    if (count) count[e] = s[3 + (f_max + 3) / 4].x;
}

// The task of every env's own slot <-> the tail of its record: one uint4 per thread over all (env, uint4) pairs, so that
// both sides are read and written contiguously.  LOAD: restore (row map as for maze_restore_kernel), else snapshot.
template <bool LOAD>
__global__ void maze_record_tasks_kernel(int64_t n, int blob_bytes, const int32_t *__restrict__ env2task, uint8_t *blobs,
                                         uint8_t *rec, int64_t rec_bytes, int64_t tail, int64_t n_rec,
                                         const int64_t *__restrict__ row)
{
    const int64_t q = blob_bytes / 16, total = n * q;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = i / q, k = i - e * q;
        uint4 *blob = reinterpret_cast<uint4 *>(blobs + (int64_t)env2task[e] * blob_bytes) + k;
        if (LOAD) {
            const int64_t rw = row[e];
            if (rw >= 0 && rw < n_rec) *blob = reinterpret_cast<const uint4 *>(rec + rw * rec_bytes + tail)[k];
        } else {
            reinterpret_cast<uint4 *>(rec + e * rec_bytes + tail)[k] = *blob;
        }
    }
}

// Every env's path entries <-> its record at byte `off`, over all (entry, env) pairs, env fastest (the path is
// step-major).  LOAD: restore (row map as for maze_restore_kernel), else snapshot.
template <bool LOAD>
__global__ void maze_record_path_kernel(int64_t n, int64_t n_pad, int64_t cap, char2 *path, uint8_t *rec, int64_t rec_bytes,
                                        int64_t off, int64_t n_rec, const int64_t *__restrict__ row)
{
    const int64_t total = n * cap;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = i / n, e = i - s * n;
        char2 *p = path + s * n_pad + e;
        if (LOAD) {
            const int64_t rw = row[e];
            if (rw >= 0 && rw < n_rec) *p = reinterpret_cast<const char2 *>(rec + rw * rec_bytes + off)[s];
        } else {
            reinterpret_cast<char2 *>(rec + e * rec_bytes + off)[s] = *p;
        }
    }
}

}  // namespace

// Records carry their env's whole task when the env owns its table slot and the table can change on the device
// (resample_tasks needs the direct renderer).  Otherwise the table is shared, and fingerprinted.
static bool records_carry_tasks(const mgb_maze *h)
{
    return h->slot_per_env && !pose_cache_serves(h);
}

static int64_t record_tail(const mgb_maze *h)
{
    return kMazeRecHead + (int64_t)(h->c.f_max + 3) / 4 * 16 + (h->trial_k ? 16 : 0);
}

// where the path entries start in a record (recording on)
static int64_t record_path_off(const mgb_maze *h)
{
    return record_tail(h) + (records_carry_tasks(h) ? h->c.blob_bytes : 0);
}

static int64_t record_bytes(const mgb_maze *h)
{
    return record_path_off(h) + (h->path ? (path_cap(h) * 2 + 15) / 16 * 16 : 0);
}

// snapshot (LOAD false) or restore the path entries of the records.  A snapshot also zeroes the padding behind each
// record's entries, so that the same state always gives the same record bytes.
static int record_paths(mgb_maze *h, bool load, const uint8_t *rec_dev, int64_t n_rec, const int64_t *row, cudaStream_t st)
{
    if (!h->path) return MGB_OK;
    const int64_t total = h->n * path_cap(h), most = (int64_t)h->num_sms * 16;
    const int64_t grid = (total + 255) / 256 < most ? (total + 255) / 256 : most;
    uint8_t *rec = const_cast<uint8_t *>(rec_dev);
    if (load)
        maze_record_path_kernel<true><<<(unsigned)grid, 256, 0, st>>>(h->n, h->n_pad, path_cap(h), h->path.get(), rec,
                                                                     record_bytes(h), record_path_off(h), n_rec, row);
    else
        maze_record_path_kernel<false><<<(unsigned)grid, 256, 0, st>>>(h->n, h->n_pad, path_cap(h), h->path.get(), rec,
                                                                      record_bytes(h), record_path_off(h), 0, nullptr);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    const int64_t used = path_cap(h) * 2, pad = (used + 15) / 16 * 16 - used;
    if (!load && pad)
        MGB_CUDA(cudaMemset2DAsync(rec + record_path_off(h) + used, (size_t)record_bytes(h), 0, (size_t)pad,
                                   (size_t)h->n, st));
    return MGB_OK;
}

extern "C" int64_t mgb_maze_record_bytes(const mgb_maze *h)
{
    MGB_REQUIRE(h, "null handle");
    MGB_REQUIRE(h->has_task, "call mgb_maze_set_task first (it fixes the record layout)");
    return record_bytes(h);
}

extern "C" int mgb_maze_snapshot(mgb_maze *h, uint8_t *rec_dev, void *stream)
{
    MgbRange nvtx_range("mgb_maze_snapshot");
    MGB_REQUIRE(h && rec_dev, "null argument");
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(rec_dev) & 15u) == 0, "rec_dev must be 16-byte aligned");
    MGB_REQUIRE(h->has_task, "call mgb_maze_set_task first (it fixes the record layout)");
    MgbDeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    const MazeArgs a = maze_args(h);
    const int64_t rb = record_bytes(h);
    maze_snapshot_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, st>>>(h->c.f_max, a, h->task_epoch.get(),
                                                                         h->task_count.get(), rec_dev, rb);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    if (records_carry_tasks(h)) {
        const int64_t total = h->n * (h->c.blob_bytes / 16), cap = (int64_t)h->num_sms * 16;
        const int64_t grid = (total + 255) / 256 < cap ? (total + 255) / 256 : cap;
        maze_record_tasks_kernel<false><<<(unsigned)grid, 256, 0, st>>>(h->n, h->c.blob_bytes, h->env2task.get(), h->tasks.blobs.get(), rec_dev,
                                                                       rb, record_tail(h), 0, nullptr);
        MGB_CUDA(cudaGetLastError());
        h->launches += 1;
    }
    return record_paths(h, false, rec_dev, 0, nullptr, st);
}

extern "C" int mgb_maze_restore(mgb_maze *h, const uint8_t *rec_dev, int64_t n_rec, const int64_t *row_of_env_dev,
                                void *stream)
{
    MgbRange nvtx_range("mgb_maze_restore");
    MGB_REQUIRE(h && rec_dev && row_of_env_dev, "null argument");
    MGB_REQUIRE(n_rec >= 0, "n_rec must not be negative");
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(rec_dev) & 15u) == 0, "rec_dev must be 16-byte aligned");
    int rc = maze_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    // what the first reset() builds, so that a handle restored right after set_task steps (and can be captured) like a
    // reset one
    if (h->c.kind != MGB_MAZE_2D && (rc = ensure_pose_cache(h, st))) return rc;
    const bool carry = records_carry_tasks(h);
    const int64_t rb = record_bytes(h);
    const MazeArgs a = maze_args(h);
    maze_restore_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, st>>>(h->c.f_max, a, h->task_epoch.get(),
                                                                        h->task_count.get(), carry ? nullptr : h->env2task.get(), h->n_tasks, rec_dev,
                                                                        rb, n_rec, row_of_env_dev);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    if (carry) {
        const int64_t total = h->n * (h->c.blob_bytes / 16), cap = (int64_t)h->num_sms * 16;
        const int64_t grid = (total + 255) / 256 < cap ? (total + 255) / 256 : cap;
        maze_record_tasks_kernel<true><<<(unsigned)grid, 256, 0, st>>>(h->n, h->c.blob_bytes, h->env2task.get(), h->tasks.blobs.get(),
                                                                      const_cast<uint8_t *>(rec_dev), rb, record_tail(h),
                                                                      n_rec, row_of_env_dev);
        MGB_CUDA(cudaGetLastError());
        h->launches += 1;
        if ((rc = build_expert(h, h->n, h->env2task.get(), nullptr, row_of_env_dev, n_rec, st))) return rc;
    }
    return record_paths(h, true, rec_dev, n_rec, row_of_env_dev, st);
}

extern "C" int mgb_maze_counters(mgb_maze *h, uint64_t *t_base, int set)
{
    MGB_REQUIRE(h && t_base, "null argument");
    if (set) h->t_base = (uint32_t)*t_base;
    else *t_base = h->t_base;
    return MGB_OK;
}

extern "C" int mgb_maze_fingerprint(const mgb_maze *h, uint64_t *out)
{
    MGB_REQUIRE(h && out, "null argument");
    MGB_REQUIRE(h->has_task, "call mgb_maze_set_task first (it fixes the record layout)");
    const MazeConst &c = h->c;
    const bool carry = records_carry_tasks(h);
    const int64_t rb = record_bytes(h);
    uint64_t f = mgb_fnv(MGB_FNV_BASIS, &h->cfg, sizeof(h->cfg));
    f = mgb_fnv(f, &h->auto_reset, sizeof(h->auto_reset));
    f = mgb_fnv(f, &c.f_max, sizeof(c.f_max));
    f = mgb_fnv(f, &c.blob_bytes, sizeof(c.blob_bytes));
    f = mgb_fnv(f, &c.max_hits, sizeof(c.max_hits));
    f = mgb_fnv(f, &h->min_cell, sizeof(h->min_cell));
    f = mgb_fnv(f, h->cls_heights.data(), h->cls_heights.size() * sizeof(double));
    if (h->path) {                              // path recording and its capacity (a handle without it hashes as before)
        const int64_t cap = path_cap(h);
        f = mgb_fnv(f, "path", 4);
        f = mgb_fnv(f, &cap, sizeof(cap));
    }
    if (h->trial_k) {                           // episodes per maze (a handle without trials hashes as before)
        f = mgb_fnv(f, "trial", 5);
        f = mgb_fnv(f, &h->trial_k, sizeof(h->trial_k));
    }
    out[0] = mgb_fnv(f, &rb, sizeof(rb));
    out[1] = h->fp_tex;
    uint64_t t = 0;
    if (!carry) {
        t = mgb_fnv(MGB_FNV_BASIS, &h->n_tasks, sizeof(h->n_tasks));
        t = mgb_fnv(t, h->slot_fp.data(), h->slot_fp.size() * sizeof(uint64_t));
    }
    out[2] = t;
    out[3] = carry ? 1 : 0;
    return MGB_OK;
}
