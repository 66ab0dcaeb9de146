// Quadrotor hot path for sm_90a.  The float32 arithmetic of one env.step() is written ONCE, templated on a lane type
// (quad_lanes.cuh): T = float runs one env per thread; T = f2 runs TWO envs per thread as two independent scalar
// chains.  The 22-float rigid-body state, the adjugate
// of the rotation matrix and every substep intermediate live in registers for the whole env.step().
//
// Replaces (reference file:line, PaddlePaddle/MetaGym):
//   QuadrotorSim._run_internal / _check_failure / step      metagym/quadrotor/quadrotorsim.py:122-221, 295-304
//   QuadrotorSim.get_state / get_sensor / reset              metagym/quadrotor/quadrotorsim.py:239-293
//   Quadrotor.step / _get_reward / _check_collision / _update_state / _convert_state_to_ndarray
//                                                             metagym/quadrotor/env.py:127-165, 193-281
//
// Data layout in HBM (DESIGN.md "state planes"): per tile of 128 envs, six planes of float4 stored back to back
// (tile t, plane k, env j -> float4 index (t*6 + k)*128 + j).  Every load/store is one coalesced 128-bit access per
// thread (512 B contiguous per warp) AND a tile's whole state is one contiguous 12 KB block, so a CTA touches 3 DRAM
// pages instead of 12 far-apart ones (and the streaming kernel fetches it with one bulk/TMA copy):
//   P0 = p.x p.y p.z v.x | P1 = v.y v.z w.x w.y | P2 = w.z m0 m1 m2 | P3 = m3 R00 R01 R02
//   P4 = R10 R11 R12 R20 | P5 = R21 R22 ct(int) episode(int)
// (p position, v velocity, w body angular velocity, m propeller speeds, R rotation matrix)
// Observations leave through a shared-memory tile and ONE bulk (TMA) store per CTA, so the [n][obs_dim] row-major
// array the gym API wants is written with full 128 B lines even though obs_dim*4 (64 or 76 B) is not a line.
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
#include "quad_lanes.cuh"

namespace {

constexpr int kThreads = 64;   // scalar tile kernel / rollout kernel: envs per CTA
static_assert(kThreads == MGB_QUAD_POLICY_CTA_ENVS, "include/mgb200.h publishes the policy CTA's env count");
constexpr int kMaxObs = 19;

// Constants derived on the host (double arithmetic, rounded once to float32 -- numpy's "weak python scalar" rule).
struct QuadConst {
    float h;         // substep
    float k1phi;     // (phi/ra)*phi
    float k1;        // phi/ra
    float inv_phi;   // 1/phi
    float hjm;       // h/jm
    float hk;        // (h/jm)*(phi/ra)*phi : per-substep relative decay of a rotor's speed
    float mm;
    float ct0, ct1, ct2;
    float vmin, vmax;
    float A[4], B[4];      // py*|p|, px*|p|   (inflow term, quadrotorsim.py:149-151)
    float px[4], py[4], pz[4];
    float Df[3], Dm[3];
    float cg[3];
    float hI[9];           // h * inverse inertia
    float gm;              // -9.8 * mass
    float c_hm;            // h / mass
    float c_h2m;           // 0.5 h^2 / mass
    float fail_r2, fail_v2, fail_w2;
    float dt, healthy, z_off;
    float init_v[3], init_w[3], noise_v, noise_w;
    int nt, task, substeps, obs_dim;
    int rk4_steps;         // 0 = reference substeps; > 0 = classical RK4 steps per env step
    float rk4_h;           // dt / rk4_steps
    float inv_jm, inv_m;   // continuous-time rates used by RK4 (1/Jm, 1/mass)
    float Iinv[9];         // inverse inertia (unscaled)
    int simple;            // propeller z == 0, cg == 0, diagonal inertia, ct2 == 0
};

struct QuadArgs {
    float4 *planes;
    int64_t n_pad;
    int64_t n;
    int64_t env_base;          // global index of local env 0
    const float *act;          // [n][4]  (rollout: [T][n][4] or null)
    float *obs;                // [n][D]
    float *rew;
    uint8_t *done;
    int32_t *fail;
    float *final_obs;
    const float4 *targets;     // [nt][n_tasks] (x, y, z, 0): the handle's time-major copy (mgb_quad_set_targets)
    int n_tasks;
    const int32_t *sat;        // obstacle map: summed-area table of non-zero cells [(rows+1)][(cols+1)], or null (flat)
    int map_rows, map_cols, x_off, y_off;
    const int32_t *env2task;   // [n]
    uint64_t seed;
    int auto_reset;
    int per_cta;               // quad_step_wide_kernel / quad_step2_kernel: envs per CTA (multiple of 4)
    // rollout only
    int T;
    uint64_t act_seed;
    uint32_t t_base;
    float *act_out;
    MgbMirrors mir;            // rollout only: every output is also stored at ptr + mir.delta[i]
    // [n] (rollout: [T][n]) uint8, 1 where done came only from ct == nt (env.py:159-161); null: not produced.  Last, so
    // that the parameter offsets of the fields above do not move.
    uint8_t *truncated;
};

// Register state of Lanes<T>::N envs
template <class T> struct VState {
    T p[3], v[3], om[3], w[4], R[9];
    int ct[Lanes<T>::N], ep[Lanes<T>::N];
};
using QState = VState<float>;

constexpr int kTileEnvs = 128;   // envs per state tile (layout unit, independent of the CTA size)
constexpr int kPlanes = 6;       // float4 planes per env

__device__ __forceinline__ float4 *tile_base(const QuadArgs &a, int64_t e)
{
    return a.planes + (e / kTileEnvs) * (kPlanes * kTileEnvs) + (e % kTileEnvs);
}

__device__ __forceinline__ void unpack_state(const float4 q[kPlanes], QState &s)
{
    s.p[0] = q[0].x; s.p[1] = q[0].y; s.p[2] = q[0].z; s.v[0] = q[0].w;
    s.v[1] = q[1].x; s.v[2] = q[1].y; s.om[0] = q[1].z; s.om[1] = q[1].w;
    s.om[2] = q[2].x; s.w[0] = q[2].y; s.w[1] = q[2].z; s.w[2] = q[2].w;
    s.w[3] = q[3].x; s.R[0] = q[3].y; s.R[1] = q[3].z; s.R[2] = q[3].w;
    s.R[3] = q[4].x; s.R[4] = q[4].y; s.R[5] = q[4].z; s.R[6] = q[4].w;
    s.R[7] = q[5].x; s.R[8] = q[5].y; s.ct[0] = __float_as_int(q[5].z); s.ep[0] = __float_as_int(q[5].w);
}
__device__ __forceinline__ void pack_state(const QState &s, float4 q[kPlanes])
{
    q[0] = make_float4(s.p[0], s.p[1], s.p[2], s.v[0]);
    q[1] = make_float4(s.v[1], s.v[2], s.om[0], s.om[1]);
    q[2] = make_float4(s.om[2], s.w[0], s.w[1], s.w[2]);
    q[3] = make_float4(s.w[3], s.R[0], s.R[1], s.R[2]);
    q[4] = make_float4(s.R[3], s.R[4], s.R[5], s.R[6]);
    q[5] = make_float4(s.R[7], s.R[8], __int_as_float(s.ct[0]), __int_as_float(s.ep[0]));
}

__device__ __forceinline__ void load_state(const QuadArgs &a, int64_t e, QState &s)
{
    const float4 *b = tile_base(a, e);
    float4 q[kPlanes];
#pragma unroll
    for (int k = 0; k < kPlanes; ++k) q[k] = b[k * kTileEnvs];
    unpack_state(q, s);
}

__device__ __forceinline__ void store_state(const QuadArgs &a, int64_t e, const QState &s)
{
    float4 *b = tile_base(a, e);
    float4 q[kPlanes];
    pack_state(s, q);
#pragma unroll
    for (int k = 0; k < kPlanes; ++k) b[k * kTileEnvs] = q[k];
}

// lane h of a packed state <-> scalar state (forward declarations used by the packed load/store)
template <class T> __device__ __forceinline__ void get_lane_state(const VState<T> &s, int h, QState &o);
template <class T> __device__ __forceinline__ void set_lane_state(VState<T> &s, int h, const QState &o);

// packed threads own the envs (e, e+1), e even: two float4 per plane, adjacent in the plane (one 32-byte stretch)
__device__ __forceinline__ void load_state2(const QuadArgs &a, int64_t e, VState<f2> &s)
{
    QState s0, s1;
    load_state(a, e, s0);
    load_state(a, e + 1, s1);            // e + 1 < n_pad: the planes are padded to whole tiles
    set_lane_state(s, 0, s0);
    set_lane_state(s, 1, s1);
}
__device__ __forceinline__ void store_state2(const QuadArgs &a, int64_t e, const VState<f2> &s)
{
    QState s0, s1;
    get_lane_state(s, 0, s0);
    get_lane_state(s, 1, s1);
    store_state(a, e, s0);
    store_state(a, e + 1, s1);
}

// lane h of a packed state <-> scalar state
template <class T> __device__ __forceinline__ void get_lane_state(const VState<T> &s, int h, QState &o)
{
#pragma unroll
    for (int k = 0; k < 3; ++k) { o.p[k] = lane(s.p[k], h); o.v[k] = lane(s.v[k], h); o.om[k] = lane(s.om[k], h); }
#pragma unroll
    for (int k = 0; k < 4; ++k) o.w[k] = lane(s.w[k], h);
#pragma unroll
    for (int k = 0; k < 9; ++k) o.R[k] = lane(s.R[k], h);
    o.ct[0] = s.ct[h];
    o.ep[0] = s.ep[h];
}
template <class T> __device__ __forceinline__ void set_lane_state(VState<T> &s, int h, const QState &o)
{
#pragma unroll
    for (int k = 0; k < 3; ++k) { set_lane(s.p[k], h, o.p[k]); set_lane(s.v[k], h, o.v[k]); set_lane(s.om[k], h, o.om[k]); }
#pragma unroll
    for (int k = 0; k < 4; ++k) set_lane(s.w[k], h, o.w[k]);
#pragma unroll
    for (int k = 0; k < 9; ++k) set_lane(s.R[k], h, o.R[k]);
    s.ct[h] = o.ct[0];
    s.ep[h] = o.ep[0];
}

// ---- explicit float32 building blocks.  This file is compiled with -fmad=false and every fused multiply-add is
// written out, so the arithmetic of an env does not depend on which kernel variant (scalar / packed / streaming /
// rollout) or which inlining context the compiler happened to see: results are bit-identical for any batch size,
// sharding or lane type.
template <class T> __device__ __forceinline__ T dot3(T a0, T b0, T a1, T b1, T a2, T b2)
{
    return vfma(a2, b2, vfma(a1, b1, vmul(a0, b0)));
}
template <class T> __device__ __forceinline__ T det2(T a, T b, T c, T d) { return vfma(a, b, vneg(vmul(c, d))); }   // ab - cd
template <class T> __device__ __forceinline__ T sq3(const T v[3]) { return dot3(v[0], v[0], v[1], v[1], v[2], v[2]); }

// ---- fast float32 primitives.  The reference's own float32 noise (SURVEY.md 8c: 1.3e-7 relative per step against a
// float64 restatement) is larger than the error of any of these, and each replaces a 10-60 instruction IEEE sequence.
// atan2 with a degree-7 minimax polynomial in a^2 on [0,1] (max abs error 7.5e-8 rad evaluated in float32, fitted for
// this file) instead of libdevice's ~65-instruction atan2f.  atan2(+-0, x>0) = +-0 like numpy.
template <class T> __device__ __forceinline__ T fast_atan2(T y, T x)
{
    const T ax = vabs(x), ay = vabs(y);
    const T mx = vmax(ax, ay), mn = vmin(ax, ay);
    const T rc = vrcp_approx(mx);
    T a = vmul(mn, rc);
    a = vfma(vfma(vneg(a), mx, mn), rc, a);                  // one correction step of the quotient
#pragma unroll
    for (int h = 0; h < Lanes<T>::N; ++h) set_lane(a, h, lane(mx, h) > 0.f ? lane(a, h) : 0.f);
    const T q = vmul(a, a);
    T r = bc<T>(0.0026222404558211565f);
    r = vfma(r, q, bc<T>(-0.015132519416511059f));
    r = vfma(r, q, bc<T>(0.04112182930111885f));
    r = vfma(r, q, bc<T>(-0.07366703450679779f));
    r = vfma(r, q, bc<T>(0.10573931038379669f));
    r = vfma(r, q, bc<T>(-0.1418597549200058f));
    r = vfma(r, q, bc<T>(0.1999039649963379f));
    r = vfma(r, q, bc<T>(-0.33332985639572144f));
    r = vfma(vmul(r, q), a, a);
    const T r1 = vsub(1.57079632679489662f, r);
    const T r2a = vsub(3.14159265358979324f, r), r2b = vsub(3.14159265358979324f, r1);
    T out;
#pragma unroll
    for (int h = 0; h < Lanes<T>::N; ++h) {
        // the sign bit, not x < 0: atan2(+-0, -0) = +-pi like np.arctan2 (gimbal lock, an inverted vehicle)
        const bool swap = lane(ay, h) > lane(ax, h), neg = signbit(lane(x, h));
        const float v = swap ? (neg ? lane(r2b, h) : lane(r1, h)) : (neg ? lane(r2a, h) : lane(r, h));
        set_lane(out, h, copysignf(v, lane(y, h)));
    }
    return out;
}

// adjugate of R (unscaled inverse) and 1/det; R^-1 = adj * id.  R drifts away from orthogonality (the reference never
// re-orthonormalises, quadrotorsim.py:193-202), so this is a genuine inverse, not a transpose.  det = 1 +- a few 1e-3.
template <class T> __device__ __forceinline__ void adjugate(const T R[9], T adj[9], T &id)
{
    adj[0] = det2(R[4], R[8], R[5], R[7]);
    adj[3] = det2(R[5], R[6], R[3], R[8]);
    adj[6] = det2(R[3], R[7], R[4], R[6]);
    const T det = dot3(R[0], adj[0], R[1], adj[3], R[2], adj[6]);
    adj[1] = det2(R[2], R[7], R[1], R[8]);
    adj[2] = det2(R[1], R[5], R[2], R[4]);
    adj[4] = det2(R[0], R[8], R[2], R[6]);
    adj[5] = det2(R[2], R[3], R[0], R[5]);
    adj[7] = det2(R[1], R[6], R[0], R[7]);
    adj[8] = det2(R[0], R[4], R[1], R[3]);
    id = vrcp(det);
}

// One call of _run_internal (quadrotorsim.py:122-208) on register state.  Algebra used (exact in real arithmetic):
//   me_i  = (phi/ra)(V_i - phi w_i) = kV_i - k1phi w_i                                   :136-138
//   w_i' = w_i + (h/jm)(me_i - Mm) = w_i + (cw_i - hk w_i),  hk = (h/jm) k1phi, cw_i = (h/jm)(kV_i - Mm)   :141-145
//   yaw reaction -me0+me1-me2+me3 = Kz - k1phi((w1-w0)+(w3-w2)),  Kz = (kV1-kV0)+(kV3-kV2)               :164
// so the per-rotor work is 2 ops for the speed, 2 for the inflow, 3 for the thrust, 2 for the torque arm.
template <bool SIMPLE, class T>
__device__ __forceinline__ void substep(const QuadConst &c, VState<T> &s, const T cw[4], T Kz, T adj[9], T &id, T &vsq,
                                        T &osq)
{
    // body-frame velocity R^-1 v (:147-148), shared by the four rotors and the drag term
    const T bvx = vmul(dot3(adj[0], s.v[0], adj[1], s.v[1], adj[2], s.v[2]), id);
    const T bvy = vmul(dot3(adj[3], s.v[0], adj[4], s.v[1], adj[5], s.v[2]), id);
    const T bvz = vmul(dot3(adj[6], s.v[0], adj[7], s.v[1], adj[8], s.v[2]), id);
    const T nvn = vneg(vsqrt(vsq)), non = vneg(vsqrt(osq));
    const T tz = vfma(-c.k1phi, vadd(vsub(s.w[1], s.w[0]), vsub(s.w[3], s.w[2])), Kz);
    T th[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const T v1 = vfma(s.om[0], c.A[i], vfma(vneg(s.om[1]), c.B[i], bvz));      // inflow, :146-151
        // increment first, then ONE rounding at the magnitude of w -- the reference's rounding structure (:144-145).  Near
        // its fixed point a rotor's float32 speed stagnates within +-ulp/2 of increment; any other association
        // (w*(1-hk)+cw, (w+cw)-hk*w) stagnates elsewhere and biases thrust by ~1e-5.
        const T wm = vadd(s.w[i], vfma(-c.hk, s.w[i], cw[i]));
        th[i] = vmul(wm, vfma(c.ct0, wm, vmul(c.ct1, v1)));                        // :154-156
        if (!SIMPLE) th[i] = vfma(vmul(c.ct2, v1), vabs(v1), th[i]);
        s.w[i] = wm;
    }
    const T fz = vadd(vadd(th[0], th[1]), vadd(th[2], th[3]));
    // -(0,0,th) x p_i summed over the rotors, :160-162
    const T tx = vfma(th[0], c.py[0], vfma(th[1], c.py[1], vfma(th[2], c.py[2], vmul(th[3], c.py[3]))));
    const T ty = vneg(vfma(th[0], c.px[0], vfma(th[1], c.px[1], vfma(th[2], c.px[2], vmul(th[3], c.px[3])))));

    // force: thrust + gravity (R^-1 g m) + drag (-|v| Df R^-1 v), :166-180
    const T idgm = vmul(id, c.gm);
    const T Fx = vfma(vmul(nvn, c.Df[0]), bvx, vmul(adj[2], idgm));
    const T Fy = vfma(vmul(nvn, c.Df[1]), bvy, vmul(adj[5], idgm));
    const T Fz = vfma(vmul(nvn, c.Df[2]), bvz, vfma(adj[8], idgm, fz));
    T Tx = vfma(vmul(non, c.Dm[0]), s.om[0], tx);
    T Ty = vfma(vmul(non, c.Dm[1]), s.om[1], ty);
    T Tz = vfma(vmul(non, c.Dm[2]), s.om[2], tz);
    if (!SIMPLE) {  // gravity torque -(f_grav x cg), :177-178
        const T gx = vmul(adj[2], idgm), gy = vmul(adj[5], idgm), gz = vmul(adj[8], idgm);
        Tx = vsub(Tx, det2(gy, bc<T>(c.cg[2]), gz, bc<T>(c.cg[1])));
        Ty = vsub(Ty, det2(gz, bc<T>(c.cg[0]), gx, bc<T>(c.cg[2])));
        Tz = vsub(Tz, det2(gx, bc<T>(c.cg[1]), gy, bc<T>(c.cg[0])));
    }

    // translation, :183-187 (1/mass folded into the step constants)
    const T ax = dot3(s.R[0], Fx, s.R[1], Fy, s.R[2], Fz);
    const T ay = dot3(s.R[3], Fx, s.R[4], Fy, s.R[5], Fz);
    const T az = dot3(s.R[6], Fx, s.R[7], Fy, s.R[8], Fz);
    s.p[0] = vfma(ax, c.c_h2m, vfma(s.v[0], c.h, s.p[0]));
    s.p[1] = vfma(ay, c.c_h2m, vfma(s.v[1], c.h, s.p[1]));
    s.p[2] = vfma(az, c.c_h2m, vfma(s.v[2], c.h, s.p[2]));
    s.v[0] = vfma(ax, c.c_hm, s.v[0]);
    s.v[1] = vfma(ay, c.c_hm, s.v[1]);
    s.v[2] = vfma(az, c.c_hm, s.v[2]);

    // rotation, :190-204
    T ahx, ahy, ahz;  // h * I^-1 * torque
    if (SIMPLE) {
        ahx = vmul(Tx, c.hI[0]); ahy = vmul(Ty, c.hI[4]); ahz = vmul(Tz, c.hI[8]);
    } else {
        ahx = dot3(bc<T>(c.hI[0]), Tx, bc<T>(c.hI[1]), Ty, bc<T>(c.hI[2]), Tz);
        ahy = dot3(bc<T>(c.hI[3]), Tx, bc<T>(c.hI[4]), Ty, bc<T>(c.hI[5]), Tz);
        ahz = dot3(bc<T>(c.hI[6]), Tx, bc<T>(c.hI[7]), Ty, bc<T>(c.hI[8]), Tz);
    }
    const T hwx = vmul(c.h, vfma(0.5f, ahx, s.om[0]));
    const T hwy = vmul(c.h, vfma(0.5f, ahy, s.om[1]));
    const T hwz = vmul(c.h, vfma(0.5f, ahz, s.om[2]));
    s.om[0] = vadd(s.om[0], ahx); s.om[1] = vadd(s.om[1], ahy); s.om[2] = vadd(s.om[2], ahz);
#pragma unroll
    for (int r = 0; r < 3; ++r) {   // R += h R [w]x
        const T r0 = s.R[3 * r], r1 = s.R[3 * r + 1], r2 = s.R[3 * r + 2];
        s.R[3 * r + 0] = vfma(r1, hwz, vfma(vneg(r2), hwy, r0));
        s.R[3 * r + 1] = vfma(r2, hwx, vfma(vneg(r0), hwz, r1));
        s.R[3 * r + 2] = vfma(r0, hwy, vfma(vneg(r1), hwx, r2));
    }
    adjugate(s.R, adj, id);                                                  // :206-208
    vsq = sq3(s.v);
    osq = sq3(s.om);
}

template <bool SIMPLE>
__device__ __forceinline__ int integrate_rk4(const QuadConst &c, QState &s, const float4 act, float adj[9], float &id,
                                             float &power);

// _check_failure (quadrotorsim.py:210-221) of lane h; the negated comparisons also catch NaN
__device__ __forceinline__ int fail_code(const QuadConst &c, float psq, float vsq, float osq)
{
    if (!(psq <= c.fail_r2)) return MGB_FAIL_RANGE;
    if (!(vsq <= c.fail_v2)) return MGB_FAIL_VELOCITY;
    if (!(osq <= c.fail_w2)) return MGB_FAIL_ANGULAR;
    return 0;
}

// `substeps` calls of _run_internal (quadrotorsim.py:295-304).  fail[h] = fail code of lane h (0 = none); the loop stops
// at the first substep after which ANY lane failed (for T = f2 the caller then redoes both envs with the scalar
// instantiation, so a failing env never changes what its pair partner computes).  power = electrical power of the
// last executed substep (:139,188).  The loop is unrolled by 5 when substeps % 5 == 0 (dt = 0.005, 0.01) so the ~40 step
// constants stay in uniform registers across the unrolled body.
template <bool SIMPLE, class T>
__device__ __forceinline__ bool integrate(const QuadConst &c, VState<T> &s, const T Vin[4], T adj[9], T &id, T &power,
                                          int fail[Lanes<T>::N])
{
    constexpr int N = Lanes<T>::N;
    // voltage clamp (:130-134) and the per-step rotor constants
    T V[4], kV[4], cw[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int h = 0; h < N; ++h) {
            const float x = lane(Vin[i], h);
            set_lane(V[i], h, x > c.vmax ? c.vmax : (x < c.vmin ? c.vmin : x));
        }
        kV[i] = vmul(c.k1, V[i]);
        cw[i] = vmul(c.hjm, vsub(kV[i], c.mm));
    }
    const T Kz = vadd(vsub(kV[1], kV[0]), vsub(kV[3], kV[2]));
    bool failed = false;
#pragma unroll
    for (int h = 0; h < N; ++h) fail[h] = 0;
    T vsq = sq3(s.v);
    T osq = sq3(s.om);
    T wl[4] = {s.w[0], s.w[1], s.w[2], s.w[3]};     // rotor speeds entering the last executed substep

    // _check_failure after every substep (:210-221)
#define MGB_QUAD_ONE_SUBSTEP()                                                                                   \
    {                                                                                                            \
        wl[0] = s.w[0]; wl[1] = s.w[1]; wl[2] = s.w[2]; wl[3] = s.w[3];                                          \
        substep<SIMPLE>(c, s, cw, Kz, adj, id, vsq, osq);                                                        \
        const T psq = sq3(s.p);                                                                                  \
        bool bad = false;                                                                                        \
        _Pragma("unroll") for (int h = 0; h < N; ++h)                                                            \
            bad |= !(lane(psq, h) <= c.fail_r2) || !(lane(vsq, h) <= c.fail_v2) || !(lane(osq, h) <= c.fail_w2); \
        if (bad) {                                                                                               \
            _Pragma("unroll") for (int h = 0; h < N; ++h)                                                        \
                fail[h] = fail_code(c, lane(psq, h), lane(vsq, h), lane(osq, h));                                \
            failed = true;                                                                                       \
            break;                                                                                               \
        }                                                                                                        \
    }
    // scalar lanes: unrolled by 5 when substeps % 5 == 0 (dt = 0.005, 0.01): the ~40 step constants stay in uniform
    // registers across the unrolled body; packed lanes: rolled (half the code, fewer registers)
    if (N == 1 && c.substeps % 5 == 0) {
#pragma unroll 1
        for (int k = 0; k < c.substeps; k += 5) {      // five copies written out (a `break` leaves this loop): nvcc does not
            MGB_QUAD_ONE_SUBSTEP()                      // unroll the body by pragma once it contains the per-lane loops
            MGB_QUAD_ONE_SUBSTEP()
            MGB_QUAD_ONE_SUBSTEP()
            MGB_QUAD_ONE_SUBSTEP()
            MGB_QUAD_ONE_SUBSTEP()
        }
    } else {
#pragma unroll 1
        for (int k = 0; k < c.substeps; ++k) MGB_QUAD_ONE_SUBSTEP()
    }
#undef MGB_QUAD_ONE_SUBSTEP
    T pw = bc<T>(0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) pw = vadd(pw, vabs(vmul(vmul(vfma(-c.k1phi, wl[i], kV[i]), c.inv_phi), V[i])));
    power = pw;
    return failed;
}

// scalar entry point (reference integrator or RK4): returns the fail code
template <bool SIMPLE>
__device__ __forceinline__ int integrate1(const QuadConst &c, QState &s, const float4 act, float adj[9], float &id,
                                          float &power)
{
    if (c.rk4_steps > 0) return integrate_rk4<SIMPLE>(c, s, act, adj, id, power);   // uniform branch
    const float V[4] = {act.x, act.y, act.z, act.w};
    int fail[1];
    integrate<SIMPLE, float>(c, s, V, adj, id, power, fail);
    return fail[0];
}

// ---------------------------------------------------------------------------------------------------------------
// Classical RK4 on the continuous-time model behind _run_internal (BASELINE.json config 3 "RK4 dt=0.005").
// The reference has NO such integrator (quadrotorsim.py:185-208 is semi-implicit Euler), so this mode cannot be
// parity-pinned; tests validate it by convergence against the float64 oracle run with a 1e-5 s substep.
//   p' = v,  v' = R F_body / m,  w' = I^-1 tau,  R' = R [w]x,  m_i' = (me_i - Mm) / Jm
// with the reference's force model: F_body = (0,0,sum T_i) + R^-1 g m - |v| Df R^-1 v, T_i = ct0 m_i^2 + ct1 m_i v1_i
// (+ ct2 v1_i |v1_i|), v1_i = (R^-1 v)_z + ((w x p_i) |p_i|)_z, tau = sum -(0,0,T_i) x p_i + yaw reaction - |w| Dm w
// (- f_grav x cg).  The substep quirks that vanish as h -> 0 (thrust from the already-updated rotor speed, the
// 0.5 h^2 a position term) are not part of the continuous model.  Scalar lanes only.
// ---------------------------------------------------------------------------------------------------------------
struct QDeriv { float p[3], v[3], om[3], w[4], R[9]; };

template <bool SIMPLE>
__device__ __forceinline__ void quad_rhs(const QuadConst &c, const QState &s, const float kV[4], QDeriv &d)
{
    float adj[9], id;
    adjugate(s.R, adj, id);
    const float bvx = dot3(adj[0], s.v[0], adj[1], s.v[1], adj[2], s.v[2]) * id;
    const float bvy = dot3(adj[3], s.v[0], adj[4], s.v[1], adj[5], s.v[2]) * id;
    const float bvz = dot3(adj[6], s.v[0], adj[7], s.v[1], adj[8], s.v[2]) * id;
    const float nvn = -vsqrt(sq3(s.v));
    const float non = -vsqrt(sq3(s.om));
    float fz = 0.f, tx = 0.f, ty = 0.f, me[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        me[i] = fmaf(-c.k1phi, s.w[i], kV[i]);
        d.w[i] = (me[i] - c.mm) * c.inv_jm;
        const float v1 = fmaf(s.om[0], c.A[i], fmaf(-s.om[1], c.B[i], bvz));
        float th = s.w[i] * fmaf(c.ct0, s.w[i], c.ct1 * v1);
        if (!SIMPLE) th = fmaf(c.ct2 * v1, fabsf(v1), th);
        fz += th;
        tx = fmaf(th, c.py[i], tx);
        ty = fmaf(-th, c.px[i], ty);
    }
    const float tz = (me[1] - me[0]) + (me[3] - me[2]);
    const float idgm = id * c.gm;
    const float Fx = fmaf(nvn * c.Df[0], bvx, adj[2] * idgm);
    const float Fy = fmaf(nvn * c.Df[1], bvy, adj[5] * idgm);
    const float Fz = fmaf(nvn * c.Df[2], bvz, fmaf(adj[8], idgm, fz));
    float Tx = fmaf(non * c.Dm[0], s.om[0], tx);
    float Ty = fmaf(non * c.Dm[1], s.om[1], ty);
    float Tz = fmaf(non * c.Dm[2], s.om[2], tz);
    if (!SIMPLE) {
        const float gx = adj[2] * idgm, gy = adj[5] * idgm, gz = adj[8] * idgm;
        Tx -= det2(gy, c.cg[2], gz, c.cg[1]);
        Ty -= det2(gz, c.cg[0], gx, c.cg[2]);
        Tz -= det2(gx, c.cg[1], gy, c.cg[0]);
    }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        d.p[r] = s.v[r];
        d.v[r] = dot3(s.R[3 * r], Fx, s.R[3 * r + 1], Fy, s.R[3 * r + 2], Fz) * c.inv_m;
        d.om[r] = dot3(c.Iinv[3 * r], Tx, c.Iinv[3 * r + 1], Ty, c.Iinv[3 * r + 2], Tz);
        const float r0 = s.R[3 * r], r1 = s.R[3 * r + 1], r2 = s.R[3 * r + 2];
        d.R[3 * r + 0] = det2(r1, s.om[2], r2, s.om[1]);
        d.R[3 * r + 1] = det2(r2, s.om[0], r0, s.om[2]);
        d.R[3 * r + 2] = det2(r0, s.om[1], r1, s.om[0]);
    }
}

__device__ __forceinline__ void quad_axpy(const QState &y, const QDeriv &k, float h, QState &out)
{
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        out.p[r] = fmaf(h, k.p[r], y.p[r]); out.v[r] = fmaf(h, k.v[r], y.v[r]); out.om[r] = fmaf(h, k.om[r], y.om[r]);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) out.w[r] = fmaf(h, k.w[r], y.w[r]);
#pragma unroll
    for (int r = 0; r < 9; ++r) out.R[r] = fmaf(h, k.R[r], y.R[r]);
}

template <bool SIMPLE>
__device__ __forceinline__ int integrate_rk4(const QuadConst &c, QState &s, const float4 act, float adj[9], float &id,
                                             float &power)
{
    float V[4] = {act.x, act.y, act.z, act.w}, kV[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        V[i] = V[i] > c.vmax ? c.vmax : (V[i] < c.vmin ? c.vmin : V[i]);
        kV[i] = c.k1 * V[i];
    }
    const float h = c.rk4_h;
    int fail = 0;
#pragma unroll 1
    for (int n = 0; n < c.rk4_steps; ++n) {
        QDeriv k, acc;
        QState t;
        quad_rhs<SIMPLE>(c, s, kV, k);                       // k1
        acc = k;
        quad_axpy(s, k, 0.5f * h, t);
        quad_rhs<SIMPLE>(c, t, kV, k);                       // k2
#pragma unroll
        for (int r = 0; r < 3; ++r) { acc.p[r] = fmaf(2.f, k.p[r], acc.p[r]); acc.v[r] = fmaf(2.f, k.v[r], acc.v[r]); acc.om[r] = fmaf(2.f, k.om[r], acc.om[r]); }
#pragma unroll
        for (int r = 0; r < 4; ++r) acc.w[r] = fmaf(2.f, k.w[r], acc.w[r]);
#pragma unroll
        for (int r = 0; r < 9; ++r) acc.R[r] = fmaf(2.f, k.R[r], acc.R[r]);
        quad_axpy(s, k, 0.5f * h, t);
        quad_rhs<SIMPLE>(c, t, kV, k);                       // k3
#pragma unroll
        for (int r = 0; r < 3; ++r) { acc.p[r] = fmaf(2.f, k.p[r], acc.p[r]); acc.v[r] = fmaf(2.f, k.v[r], acc.v[r]); acc.om[r] = fmaf(2.f, k.om[r], acc.om[r]); }
#pragma unroll
        for (int r = 0; r < 4; ++r) acc.w[r] = fmaf(2.f, k.w[r], acc.w[r]);
#pragma unroll
        for (int r = 0; r < 9; ++r) acc.R[r] = fmaf(2.f, k.R[r], acc.R[r]);
        quad_axpy(s, k, h, t);
        quad_rhs<SIMPLE>(c, t, kV, k);                       // k4
#pragma unroll
        for (int r = 0; r < 3; ++r) { acc.p[r] += k.p[r]; acc.v[r] += k.v[r]; acc.om[r] += k.om[r]; }
#pragma unroll
        for (int r = 0; r < 4; ++r) acc.w[r] += k.w[r];
#pragma unroll
        for (int r = 0; r < 9; ++r) acc.R[r] += k.R[r];
        const int ct = s.ct[0], ep = s.ep[0];
        quad_axpy(s, acc, h * (1.0f / 6.0f), t);
        s = t; s.ct[0] = ct; s.ep[0] = ep;
        const float psq = sq3(s.p);
        const float vsq = sq3(s.v);
        const float osq = sq3(s.om);
        fail = fail_code(c, psq, vsq, osq);
        if (fail) break;
    }
    adjugate(s.R, adj, id);
    float pw = 0.f;      // electrical power at the end state (the reference reports the last substep's, :139,188)
#pragma unroll
    for (int i = 0; i < 4; ++i) pw += fabsf(fmaf(-c.k1phi, s.w[i], kV[i]) * c.inv_phi * V[i]);
    power = pw;
    return fail;
}

// get_state + get_sensor + _convert_state_to_ndarray (quadrotorsim.py:260-293, env.py:193-209)
// key order: b_v xyz, b xyz, acc xyz, gyro xyz, pitch, roll, yaw, z (+ z_offset)
template <class T>
__device__ __forceinline__ void observe(const QuadConst &c, const VState<T> &s, const T adj[9], T id, T *o, T bv[3],
                                        T Ri[9])
{
#pragma unroll
    for (int k = 0; k < 9; ++k) Ri[k] = vmul(adj[k], id);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        bv[r] = dot3(Ri[3 * r], s.v[0], Ri[3 * r + 1], s.v[1], Ri[3 * r + 2], s.v[2]);
        o[r] = bv[r];
        o[3 + r] = dot3(Ri[3 * r], s.p[0], Ri[3 * r + 1], s.p[1], Ri[3 * r + 2], s.p[2]);
        o[6 + r] = vmul(Ri[3 * r + 2], -9.8f);    // body_acceleration is never updated (:22,:278): IMU = R^-1 g only
        o[9 + r] = s.om[r];
    }
    o[12] = fast_atan2(vneg(s.R[6]), vsqrt(vfma(s.R[8], s.R[8], vmul(s.R[7], s.R[7]))));   // pitch, :111-120
    o[13] = fast_atan2(s.R[7], s.R[8]);                                                     // roll
    o[14] = fast_atan2(s.R[3], s.R[0]);                                                     // yaw
    o[15] = vadd(s.p[2], c.z_off);
}

// QuadrotorSim.reset applied to lane h with the twelve uniform draws u[12] (quadrotorsim.py:239-258)
template <class T> __device__ __forceinline__ void reset_env(const QuadConst &c, VState<T> &s, int h, const double u[12])
{
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        set_lane(s.p[k], h, 0.f);
        const double sv = u[k] > 0.5 ? 1.0 : -1.0, sw = u[6 + k] > 0.5 ? 1.0 : -1.0;
        set_lane(s.v[k], h, (float)((double)c.init_v[k] + ((double)c.noise_v * u[3 + k]) * sv));
        set_lane(s.om[k], h, (float)((double)c.init_w[k] + ((double)c.noise_w * u[9 + k]) * sw));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) set_lane(s.w[k], h, 0.f);
#pragma unroll
    for (int k = 0; k < 9; ++k) set_lane(s.R[k], h, (k % 4 == 0) ? 1.f : 0.f);
}

__device__ __forceinline__ void philox_reset_draws(uint64_t seed, int64_t genv, int ep, double u[12])
{
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const uint4 r = mgb_philox4x32_10(
            make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32), (uint32_t)ep, MGB_STREAM_RESET + j), key);
        u[4 * j + 0] = (double)mgb_u01(r.x);
        u[4 * j + 1] = (double)mgb_u01(r.y);
        u[4 * j + 2] = (double)mgb_u01(r.z);
        u[4 * j + 3] = (double)mgb_u01(r.w);
    }
}

// Velocity-target rows an env needs this step.  The handle's table is time-major, [nt][n_tasks] float4 (x, y, z, 0), so
// a row is ONE 16-byte load, and the lanes of a warp at the same ct (all envs of a batch that started together) read 32
// consecutive rows: 512 contiguous bytes instead of 32 cache lines per component of the task-major [n_tasks][nt][3].
template <class T> struct TargetRows {
    T cur[3];    // velocity_targets[ct - 1]         (env.py:153)
    T nxt[3];    // velocity_targets[min(ct, nt-1)]  (env.py:270-274)
};
__device__ __forceinline__ float4 target_row(const QuadArgs &a, int task, int t)
{
    return __ldg(a.targets + (int64_t)t * a.n_tasks + task);
}
template <class T>
__device__ __forceinline__ void prefetch_targets(const QuadConst &c, const QuadArgs &a, int task, int ct, int h,
                                                 TargetRows<T> &tr)
{
    const int t = ct < c.nt - 1 ? ct : c.nt - 1;
    const float4 g = target_row(a, task, ct - 1), q = target_row(a, task, t);
    set_lane(tr.cur[0], h, g.x); set_lane(tr.cur[1], h, g.y); set_lane(tr.cur[2], h, g.z);
    set_lane(tr.nxt[0], h, q.x); set_lane(tr.nxt[1], h, q.y); set_lane(tr.nxt[2], h, q.z);
}
// env2task of env e (0 for the tasks without targets, whose handles have no env2task)
__device__ __forceinline__ int env_task(const QuadConst &c, const QuadArgs &a, int64_t e)
{
    return c.task == MGB_TASK_VELOCITY_CONTROL ? __ldg(a.env2task + e) : 0;
}

// python slice bound for a[start:stop] on an axis of length len (negative indices wrap once, then clamp)
__device__ __forceinline__ int slice_bound(double v, int len)
{
    long long x = v < -2.0e9 ? -2000000000LL : (v > 2.0e9 ? 2000000000LL : (long long)v);
    if (x < 0) { x += len; if (x < 0) x = 0; }
    if (x > len) x = len;
    return (int)x;
}

// _check_collision with an obstacle map (env.py:248-260).  x/y are float64 in the reference (float32 position +
// int64 offset from np.where), z is float32 (+ python float 5.0).
__device__ __forceinline__ bool map_collision(const QuadArgs &a, float x_old, float y_old, float z_old, float x_new,
                                              float y_new, float z_new)
{
    const double xo = (double)x_old + a.x_off, xn = (double)x_new + a.x_off;
    const double yo = (double)y_old + a.y_off, yn = (double)y_new + a.y_off;
    const double x_min = floor(fmin(xo, xn)), x_max = ceil(fmax(xo, xn));
    const double y_min = floor(fmin(yo, yn)), y_max = ceil(fmax(yo, yn));
    const int z_lo = (int)floorf(fminf(z_old, z_new)), z_hi = (int)ceilf(fmaxf(z_old, z_new));
    const int ys = slice_bound(y_min, a.map_rows), ye = slice_bound(y_max + 1.0, a.map_rows);
    const int xs = slice_bound(x_min, a.map_cols), xe = slice_bound(x_max + 1.0, a.map_cols);
    int any = 0;
    if (ys < ye && xs < xe) {
        const int W = a.map_cols + 1;
        any = (a.sat[ye * W + xe] - a.sat[ys * W + xe] - a.sat[ye * W + xs] + a.sat[ys * W + xs]) > 0 ? 1 : 0;
    }
    return z_lo < any || z_hi < any;
}

// Observation of a freshly reset env (R = I) of task `task`: cheap closed form of observe().  Written into lane h of o[].
template <class T>
__device__ __forceinline__ void observe_reset(const QuadConst &c, const QuadArgs &a, int task, const VState<T> &s, int h,
                                              T *o)
{
    set_lane(o[0], h, lane(s.v[0], h)); set_lane(o[1], h, lane(s.v[1], h)); set_lane(o[2], h, lane(s.v[2], h));
    set_lane(o[3], h, 0.f); set_lane(o[4], h, 0.f); set_lane(o[5], h, 0.f);
    set_lane(o[6], h, 0.f * -9.8f); set_lane(o[7], h, 0.f * -9.8f); set_lane(o[8], h, -9.8f);
    set_lane(o[9], h, lane(s.om[0], h)); set_lane(o[10], h, lane(s.om[1], h)); set_lane(o[11], h, lane(s.om[2], h));
    set_lane(o[12], h, -0.f); set_lane(o[13], h, 0.f); set_lane(o[14], h, 0.f);   // arctan2(-0, 1) = -0 (:114-117 at R = I)
    set_lane(o[15], h, 0.f + c.z_off);
    if (c.task == MGB_TASK_VELOCITY_CONTROL) {
        const float4 q = target_row(a, task, s.ct[h] < c.nt - 1 ? s.ct[h] : c.nt - 1);
        set_lane(o[16], h, q.x); set_lane(o[17], h, q.y); set_lane(o[18], h, q.z);
    }
}

// Task logic after the integrator: observation, reward, collision, done, counters, optional auto-reset.
// o[] receives the observation of the (pre-reset) end state; lane h of env e + h.  write_final[h]: auto-reset replaced
// the env, o[] is its terminal observation and the caller must publish observe_reset() instead.  trunc[h]: the episode
// ended through ct == nt alone (env.py:159-161): a collision clears ct first (env.py:144-150) and a failure is terminal.
template <class T>
__device__ __forceinline__ void finish_step(const QuadConst &c, const QuadArgs &a, int64_t e, VState<T> &s,
                                            const T adj[9], T id, T z_old, T x_old, T y_old, T power,
                                            const int fail[Lanes<T>::N], const TargetRows<T> &tr, T *o, T &reward,
                                            int done_flag[Lanes<T>::N], bool write_final[Lanes<T>::N],
                                            int trunc[Lanes<T>::N])
{
    constexpr int N = Lanes<T>::N;
    T bv[3], Ri[9];
    observe(c, s, adj, id, o, bv, Ri);
    if (c.task == MGB_TASK_VELOCITY_CONTROL) {                // env.py:270-274 (ct already incremented)
        o[16] = tr.nxt[0]; o[17] = tr.nxt[1]; o[18] = tr.nxt[2];
    }
    // energy term, env.py:217
    reward = vneg(vmin(vmul(c.dt, power), bc<T>(c.healthy)));
    int done[N];
#pragma unroll
    for (int h = 0; h < N; ++h) done[h] = 0;
    if (c.task == MGB_TASK_VELOCITY_CONTROL) {
        const T g0 = tr.cur[0], g1 = tr.cur[1], g2 = tr.cur[2];   // env.py:153-157
        T diff = bc<T>(0.f);
#pragma unroll
        for (int r = 0; r < 3; ++r) diff = vadd(diff, vabs(vsub(dot3(Ri[3 * r], g0, Ri[3 * r + 1], g1, Ri[3 * r + 2], g2), bv[r])));
        reward = vadd(reward, vmul(-0.001f, diff));
    } else {
        // collision, env.py:248-260: `z_min < np.any(taken_pos) or z_max < np.any(taken_pos)` compares integer
        // altitudes against a BOOL: 0 over free cells (flat map: always), 1 as soon as the window swept by the step
        // contains any obstacle cell (the obstacle's height is never used -- reference quirk)
        const T z_new = vadd(s.p[2], c.z_off);
        T bonus, vn, on;
        if (c.task == MGB_TASK_HOVERING_CONTROL) {            // env.py:222-243
            vn = vsqrt(sq3(s.v));
            on = vsqrt(sq3(s.om));
        }
#pragma unroll
        for (int h = 0; h < N; ++h) {
            bool coll;
            if (a.sat) coll = map_collision(a, lane(x_old, h), lane(y_old, h), lane(z_old, h), lane(s.p[0], h),
                                            lane(s.p[1], h), lane(z_new, h));
            else coll = fminf(lane(z_old, h), lane(z_new, h)) < 0.f;
            float tr = coll ? 0.f : c.healthy;
            if (c.task == MGB_TASK_HOVERING_CONTROL) {
                tr -= lane(vn, h) + lane(on, h);
                const float zm = fabsf(0.f - lane(s.p[2], h));     // pos_0[2] is always 0 (env.py:123, :26)
                tr += zm < 0.5f ? 10.f : fmaxf(-20.f, 0.5f - zm);
            }
            set_lane(bonus, h, tr);
            if (coll) { done[h] = 1; s.ct[h] = 0; }              // env.py:147-150
        }
        reward = vadd(reward, bonus);
    }
#pragma unroll
    for (int h = 0; h < N; ++h) {
        trunc[h] = s.ct[h] == c.nt && !fail[h];                   // before the counters are cleared
        if (s.ct[h] == c.nt) { done[h] = 1; s.ct[h] = 0; }        // env.py:159-161
        if (fail[h]) { done[h] = 1; s.ct[h] = 0; }                // the reference raises (quadrotorsim.py:212-221)
        done_flag[h] = done[h];
        write_final[h] = false;
        if (done[h] && a.auto_reset) {
            write_final[h] = true;
            s.ep[h] += 1;
            double u[12];
            philox_reset_draws(a.seed, a.env_base + e + h, s.ep[h], u);
            reset_env(c, s, h, u);
        }
    }
}

// Publish a CTA's observation tile: rows of D floats for envs [e0, e0+rows) are contiguous in global memory, so the
// whole tile is ONE bulk store (UBLKCP) when it is 16-byte sized/aligned; ragged tails fall back to scalar stores.
__device__ __forceinline__ void publish_tile(float *gobs, const float *tile, int64_t e0, int rows, int D)
{
    const uint32_t bytes = (uint32_t)rows * (uint32_t)D * 4u;
    float *dst = gobs + e0 * D;
    if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
        mgb_fence_proxy_async();
        __syncthreads();
        if (threadIdx.x == 0) {
            mgb_bulk_store(dst, tile, bytes);
            mgb_bulk_commit();
        }
    } else {
        __syncthreads();
        for (int i = threadIdx.x; i < rows * D; i += blockDim.x) dst[i] = tile[i];
    }
}

__device__ __forceinline__ void publish_tile_mirrored(const MgbMirrors &m, float *gobs, const float *tile, int64_t e0,
                                                      int rows, int D)
{
    const uint32_t bytes = (uint32_t)rows * (uint32_t)D * 4u;
    float *dst = gobs + e0 * D;
    if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
        mgb_fence_proxy_async();
        __syncthreads();
        if (threadIdx.x == 0) {
            mgb_bulk_store(dst, tile, bytes);
            mgb_mirror_bulk_store(m, dst, tile, bytes);     // deltas are 16-byte multiples (checked on the host)
            mgb_bulk_commit();
        }
    } else {
        __syncthreads();
        for (int i = threadIdx.x; i < rows * D; i += blockDim.x) {
            dst[i] = tile[i];
            mgb_mirror_store(m, dst + i, tile[i]);
        }
    }
}

// One env.step() of Lanes<T>::N consecutive envs (e, e+1) on register state: integrate, task logic, state / reward /
// done stores, observation rows into the CTA's shared-memory tile (trow = row of env e); frow receives the terminal
// observation when auto-reset replaced it (bit h of final_mask).  nact = number of valid lanes (a ragged last pair has 1).
// task[h] = env2task of lane h (velocity_control only).  EARLY: the target rows are loaded before the integrator (else
// after it); STATE_FIRST: for velocity_control the stepped state is stored before the observation work.
template <bool SIMPLE, bool EARLY, bool STATE_FIRST, class T>
__device__ __forceinline__ void step_body(const QuadConst &c, const QuadArgs &a, int64_t e, int nact, VState<T> &s,
                                          const T V[4], const int task[Lanes<T>::N], float *trow, float *frow,
                                          int &final_mask)
{
    constexpr int N = Lanes<T>::N;
    const int D = c.obs_dim;
    T adj[9], id, power;
    adjugate(s.R, adj, id);
    TargetRows<T> tr;
    int ct_now[N];
#pragma unroll
    for (int h = 0; h < N; ++h) {
        s.ct[h] += 1;                                       // env.py:128
        ct_now[h] = s.ct[h];
    }
    const bool vel = c.task == MGB_TASK_VELOCITY_CONTROL;
    if (EARLY && vel) {
#pragma unroll
        for (int h = 0; h < N; ++h) prefetch_targets(c, a, task[h], ct_now[h], h, tr);
    }
    const T z_old = vadd(s.p[2], c.z_off);                  // env.py:131-133
    const T x_old = s.p[0], y_old = s.p[1];
    int fail[N];
    if (N == 1 && c.rk4_steps > 0) {                        // uniform branch; RK4 exists for scalar lanes only
        QState s1;
        get_lane_state(s, 0, s1);
        float adj1[9], id1, pw1;
        fail[0] = integrate_rk4<SIMPLE>(c, s1, make_float4(lane(V[0], 0), lane(V[1], 0), lane(V[2], 0), lane(V[3], 0)),
                                        adj1, id1, pw1);
        set_lane_state(s, 0, s1);
#pragma unroll
        for (int k = 0; k < 9; ++k) set_lane(adj[k], 0, adj1[k]);
        set_lane(id, 0, id1);
        set_lane(power, 0, pw1);
    } else {
        const bool failed = integrate<SIMPLE, T>(c, s, V, adj, id, power, fail);
        if (N > 1 && failed) {
            // rare: some lane left the valid zone.  Redo every lane on its own with the scalar instantiation from the
            // state still in HBM, so that a failing env cannot change what its pair partner computes.
#pragma unroll 1
            for (int h = 0; h < N; ++h) {
                QState s1;
                load_state(a, e + h, s1);
                float adj1[9], id1, pw1;
                adjugate(s1.R, adj1, id1);
                const float V1[4] = {lane(V[0], h), lane(V[1], h), lane(V[2], h), lane(V[3], h)};
                int f1[1];
                integrate<SIMPLE, float>(c, s1, V1, adj1, id1, pw1, f1);
                s1.ct[0] = s.ct[h];
                s1.ep[0] = s.ep[h];
                set_lane_state(s, h, s1);
#pragma unroll
                for (int k = 0; k < 9; ++k) set_lane(adj[k], h, adj1[k]);
                set_lane(id, h, id1);
                set_lane(power, h, pw1);
                fail[h] = f1[0];
            }
        }
    }
    if (!EARLY && vel) {
#pragma unroll
        for (int h = 0; h < N; ++h) prefetch_targets(c, a, task[h], ct_now[h], h, tr);
    }
    // Velocity task, tile kernel: the state leaves before the observation and reward work, so that its stores drain
    // while that work runs instead of at the end of the step.  Its ct is final here (velocity_control has no collision
    // rule: only ct == nt and a failure end an episode, finish_step); an auto-reset rewrites the state below.
    const bool state_first = N == 1 && STATE_FIRST && vel;
    if (state_first) {
        QState s1;
        get_lane_state(s, 0, s1);
        if (s1.ct[0] == c.nt || fail[0]) s1.ct[0] = 0;
        store_state(a, e, s1);
    }
    T o[kMaxObs], reward;
    int done[N], trunc[N];
    bool wf[N];
    finish_step(c, a, e, s, adj, id, z_old, x_old, y_old, power, fail, tr, o, reward, done, wf, trunc);
    // ---- state / reward / done / fail / truncated stores
    bool stored = false;
    if constexpr (N == 2) {
        if (nact == 2) {
            store_state2(a, e, s);
            *reinterpret_cast<float2 *>(a.rew + e) = reward.v;
            *reinterpret_cast<uchar2 *>(a.done + e) = make_uchar2((uint8_t)done[0], (uint8_t)done[1]);
            if (a.fail) *reinterpret_cast<int2 *>(a.fail + e) = make_int2(fail[0], fail[1]);
            if (a.truncated) *reinterpret_cast<uchar2 *>(a.truncated + e) = make_uchar2((uint8_t)trunc[0], (uint8_t)trunc[1]);
            stored = true;
        }
    }
    if (!stored) {
#pragma unroll
        for (int h = 0; h < N; ++h) {
            if (h < nact) {
                QState s1;
                get_lane_state(s, h, s1);
                if (!state_first || wf[h]) store_state(a, e + h, s1);
                a.rew[e + h] = lane(reward, h);
                a.done[e + h] = (uint8_t)done[h];
                if (a.fail) a.fail[e + h] = fail[h];
                if (a.truncated) a.truncated[e + h] = (uint8_t)trunc[h];
            }
        }
    }
    // ---- observation rows
#pragma unroll
    for (int h = 0; h < N; ++h) {
        if (h < nact) {
            float *tr_h = trow + h * D;
            if (wf[h]) {
                if (a.final_obs) {
                    float *fr_h = frow + h * D;
#pragma unroll
                    for (int k = 0; k < 16; ++k) fr_h[k] = lane(o[k], h);
                    if (D == 19) { fr_h[16] = lane(o[16], h); fr_h[17] = lane(o[17], h); fr_h[18] = lane(o[18], h); }
                    final_mask |= 1 << h;
                }
                observe_reset(c, a, task[h], s, h, o);
            }
#pragma unroll
            for (int k = 0; k < 16; ++k) tr_h[k] = lane(o[k], h);
            if (D == 19) { tr_h[16] = lane(o[16], h); tr_h[17] = lane(o[17], h); tr_h[18] = lane(o[18], h); }
        }
    }
}

// terminal observations are rare: only CTAs that saw one write them (rows of other envs are left untouched)
__device__ __forceinline__ void publish_final(const QuadArgs &a, const float *ftile, int64_t e, int local_row, int lanes,
                                              int final_mask, int D)
{
    if (!a.final_obs) return;
    if (__syncthreads_or(final_mask)) {
        for (int h = 0; h < lanes; ++h) {
            if (final_mask & (1 << h)) {
                float *dst = a.final_obs + (e + h) * D;
                const float *frow = ftile + (local_row + h) * D;
                for (int k = 0; k < D; ++k) dst[k] = frow[k];
            }
        }
    }
}

// Scalar step kernel, 64 envs per CTA (small batches, and batches between one wave of 512-thread CTAs and the streaming
// regime).  env2task is read before the PDL wait and the two 16-byte target rows after the integrator (step_body EARLY =
// false): issued before it, with env2task already in a register, they hold eight registers across the substeps, and the
// 65 536-env step measured 1.5 % slower that way on an H100 (67 001 envs: 2 %).  For velocity_control the kernel also
// stores the stepped state right after the integrator, before the observation work (step_body; DESIGN.md section 4).
template <bool SIMPLE>
__global__ void __launch_bounds__(kThreads) quad_step_kernel(const __grid_constant__ QuadConst c,
                                                             const __grid_constant__ QuadArgs a)
{
    __shared__ __align__(128) float tile[kThreads * kMaxObs];
    __shared__ __align__(128) float ftile[kThreads * kMaxObs];
    const int64_t e0 = (int64_t)blockIdx.x * kThreads;
    const int64_t e = e0 + threadIdx.x;
    const int rows = (int)((a.n - e0) < kThreads ? (a.n - e0) : kThreads);
    const int D = c.obs_dim;
    const bool active = e < a.n;
    int final_mask = 0;

    // Programmatic dependent launch: the NEXT kernel in the stream may be scheduled now (its CTAs park at their own
    // griddepcontrol.wait), and this kernel waits here until the PREVIOUS one has completed and flushed -- the
    // launch latency of back-to-back env steps overlaps the previous step.
    // (Finer hand-offs between consecutive launches were built and measured twice: a per-tile ticket/flag protocol in round
    // 1, and in round 2 "chained" launches whose CTAs skip the grid-wide wait and wait only for the same env block of the
    // previous launch.  Both are correct (bit-identical trajectories) and neither is faster: an env block's step k+1 cannot
    // start before its own step k has stored its state, so the per-block latency chain -- not the grid barrier -- sets the
    // pace, and the register file holds barely more than one launch's worth of threads.  DESIGN.md section 4.)
    asm volatile("griddepcontrol.launch_dependents;");
    // env2task is written only by mgb_quad_set_targets, which synchronises the device, and by the first of mgb_quad_restore's
    // two kernels, never the kernel right before a step: it may be read before the wait
    const int task[1] = {active ? env_task(c, a, e) : 0};
    asm volatile("griddepcontrol.wait;" ::: "memory");

    if (active) {
        QState s;
        load_state(a, e, s);
        const float4 act = __ldg(reinterpret_cast<const float4 *>(a.act) + e);
        const float V[4] = {act.x, act.y, act.z, act.w};
        step_body<SIMPLE, false, true, float>(c, a, e, 1, s, V, task, tile + threadIdx.x * D, ftile + threadIdx.x * D,
                                              final_mask);
    }
    publish_tile(a.obs, tile, e0, rows, D);
    publish_final(a, ftile, e, threadIdx.x, 1, final_mask, D);
    if (threadIdx.x == 0) mgb_bulk_wait_read<0>();   // smem must outlive the copy; the kernel boundary flushes the writes
}

// "One CTA per SM" variant for launches that fit a single wave (N <= SMs x 512): each CTA owns `per` = ceil(N / SMs)
// envs rounded up to 4 (so that every observation tile stays 16-byte aligned for the bulk store), grid = ceil(N / per),
// and the last CTA takes the remainder (49 152 envs on 132 SMs: 130 CTAs of 376 envs and one of 272).  Target rows after
// the integrator as in quad_step_kernel: before it, 24 576 envs measured 3 % and 49 152 envs 1 % slower.
template <bool SIMPLE>
__global__ void __launch_bounds__(512, 1) quad_step_wide_kernel(const __grid_constant__ QuadConst c,
                                                                const __grid_constant__ QuadArgs a)
{
    extern __shared__ __align__(128) float wide_smem[];
    const int per = a.per_cta;
    float *tile = wide_smem, *ftile = wide_smem + (size_t)per * kMaxObs;
    const int64_t e0 = (int64_t)blockIdx.x * per;
    const int64_t e = e0 + threadIdx.x;
    int rows = (int)((a.n - e0) < per ? (a.n - e0) : per);
    if (rows < 0) rows = 0;
    const int D = c.obs_dim;
    const bool active = (int)threadIdx.x < rows;
    int final_mask = 0;
    asm volatile("griddepcontrol.launch_dependents;");
    const int task[1] = {active ? env_task(c, a, e) : 0};     // before the wait, as in quad_step_kernel
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (active) {
        QState s;
        load_state(a, e, s);
        const float4 act = __ldg(reinterpret_cast<const float4 *>(a.act) + e);
        const float V[4] = {act.x, act.y, act.z, act.w};
        step_body<SIMPLE, false, false, float>(c, a, e, 1, s, V, task, tile + threadIdx.x * D, ftile + threadIdx.x * D,
                                               final_mask);
    }
    if (rows > 0) publish_tile(a.obs, tile, e0, rows, D);
    else __syncthreads();
    publish_final(a, ftile, e, threadIdx.x, 1, final_mask, D);
    if (threadIdx.x == 0) mgb_bulk_wait_read<0>();
}

// Packed variant (MGB_PACKED=1; not the default): one thread = the env pair (e, e+1) as two independent scalar chains,
// `per` envs per CTA as in the wide kernel.  Bit-identical to the scalar kernels (tests/test_quadrotor_gpu.py).  sm_90 has
// no packed FP32 instruction, so the pair saves no floating-point issue slots; it trades half the warps for two chains of
// instruction-level parallelism per thread.
template <bool SIMPLE>
__global__ void __launch_bounds__(256, 1) quad_step2_kernel(const __grid_constant__ QuadConst c,
                                                            const __grid_constant__ QuadArgs a)
{
    extern __shared__ __align__(128) float pair_smem[];
    const int per = a.per_cta;
    float *tile = pair_smem, *ftile = pair_smem + (size_t)per * kMaxObs;
    const int64_t e0 = (int64_t)blockIdx.x * per;
    int rows = (int)((a.n - e0) < per ? (a.n - e0) : per);
    if (rows < 0) rows = 0;
    const int le = 2 * (int)threadIdx.x;               // local index of lane 0's env
    const int64_t e = e0 + le;
    const int D = c.obs_dim;
    const int nact = rows - le >= 2 ? 2 : (rows - le > 0 ? 1 : 0);
    int final_mask = 0;
    asm volatile("griddepcontrol.launch_dependents;");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (nact > 0) {
        VState<f2> s;
        load_state2(a, e, s);
        const float4 a0 = __ldg(reinterpret_cast<const float4 *>(a.act) + e);
        const float4 a1 = nact == 2 ? __ldg(reinterpret_cast<const float4 *>(a.act) + e + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        const f2 V[4] = {pack2(a0.x, a1.x), pack2(a0.y, a1.y), pack2(a0.z, a1.z), pack2(a0.w, a1.w)};
        const int task[2] = {env_task(c, a, e), env_task(c, a, nact == 2 ? e + 1 : e)};
        step_body<SIMPLE, true, false, f2>(c, a, e, nact, s, V, task, tile + le * D, ftile + le * D, final_mask);
    }
    if (rows > 0) publish_tile(a.obs, tile, e0, rows, D);
    else __syncthreads();
    publish_final(a, ftile, e, le, 2, final_mask, D);
    if (threadIdx.x == 0) mgb_bulk_wait_read<0>();
}

// Streaming variant for multi-wave launches (millions of envs): PERSISTENT CTAs loop over tiles of 128 envs and the state
// of tile i+1 (six 2 KB plane segments = one contiguous 12 KB block + 2 KB of actions) is fetched by the TMA engine
// (cp.async.bulk + mbarrier) into the other half of a double-buffered shared-memory stage while tile i integrates, so HBM
// latency is off the critical path without spending registers or occupancy on it.  Same arithmetic (step_body), same
// outputs.
constexpr int kStreamThreads = 128;

template <bool SIMPLE>
__global__ void __launch_bounds__(kStreamThreads, 4) quad_stream_kernel(const __grid_constant__ QuadConst c,
                                                                        const __grid_constant__ QuadArgs a)
{
    __shared__ __align__(128) float4 stage[2][7][kStreamThreads];    // planes 0..5 + action
    __shared__ __align__(128) float tile[kStreamThreads * kMaxObs];
    __shared__ __align__(128) float ftile[kStreamThreads * kMaxObs];
    __shared__ __align__(8) uint64_t full[2];
    const int D = c.obs_dim;
    const int64_t n_tiles = (a.n + kStreamThreads - 1) / kStreamThreads;
    const int tid = threadIdx.x;

    asm volatile("griddepcontrol.launch_dependents;");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (tid == 0) {
        mgb_mbar_init(&full[0], 1);
        mgb_mbar_init(&full[1], 1);
        mgb_fence_mbar_init();
    }
    __syncthreads();

    auto fetch = [&](int64_t t, int st) {      // one thread: 2 bulk copies land on full[st]
        const int64_t e0 = t * kStreamThreads;
        const uint32_t rows = (uint32_t)((a.n - e0) < kStreamThreads ? (a.n - e0) : kStreamThreads);
        static_assert(kStreamThreads == kTileEnvs, "one CTA iteration = one state tile");
        mgb_mbar_expect_tx(&full[st], 6u * kTileEnvs * 16u + rows * 16u);
        mgb_bulk_load(stage[st][0], a.planes + t * (6 * kTileEnvs), 6u * kTileEnvs * 16u, &full[st]);   // 12 KB, contiguous
        mgb_bulk_load(stage[st][6], reinterpret_cast<const float4 *>(a.act) + e0, rows * 16u, &full[st]);
    };

    int64_t t = blockIdx.x;
    if (tid == 0 && t < n_tiles) fetch(t, 0);
    uint32_t phase[2] = {0u, 0u};
    int st = 0;
    for (; t < n_tiles; t += gridDim.x, st ^= 1) {
        const int64_t t_next = t + gridDim.x;
        // the other stage was fully consumed one iteration ago (barrier at the end of the loop body)
        if (tid == 0 && t_next < n_tiles) fetch(t_next, st ^ 1);
        mgb_mbar_wait(&full[st], phase[st]);
        phase[st] ^= 1u;
        const int64_t e0 = t * kStreamThreads, e = e0 + tid;
        const int rows = (int)((a.n - e0) < kStreamThreads ? (a.n - e0) : kStreamThreads);
        int final_mask = 0;
        // the observation tile of the previous iteration must have been read by its bulk store
        if (tid == 0) mgb_bulk_wait_read<0>();
        __syncthreads();
        if (tid < rows) {
            QState s;
            float4 q[kPlanes];
#pragma unroll
            for (int k = 0; k < kPlanes; ++k) q[k] = stage[st][k][tid];
            unpack_state(q, s);
            const float4 act = stage[st][6][tid];
            const float V[4] = {act.x, act.y, act.z, act.w};
            const int task[1] = {env_task(c, a, e)};
            step_body<SIMPLE, true, false, float>(c, a, e, 1, s, V, task, tile + tid * D, ftile + tid * D, final_mask);
        }
        publish_tile(a.obs, tile, e0, rows, D);
        publish_final(a, ftile, e, tid, 1, final_mask, D);
        __syncthreads();      // everyone is done with stage[st] and ftile before they are refilled
    }
    if (tid == 0) mgb_bulk_wait_read<0>();
}

// T env.step()s in one launch: the state never leaves registers; per step the kernel reads 16 B of action (or draws
// it) and writes obs/reward/done.  Observation tiles are double-buffered so the bulk store of step t overlaps the
// arithmetic of step t+1.  The target rows of a step are loaded after its integrator: loaded before it, the two 16-byte
// rows stay live across the substeps of a kernel held to 128 registers, and the rollout measured 12 % slower.
// XM: 0 = outputs stored once; 1 = also at every peer mirror (NVLink P2P); 2 = stored ONLY through the multicast
// mapping (multimem.st: the switch replicates them into every rank's arena, this rank's included)
// FIN (XM == 0 only, mgb_quad_rollout_ex): also store the truncation byte of every (t, e), and the terminal observation of
// every env an auto-reset replaced at step t to final_obs + (t n + e) D, straight from registers before observe_reset
// overwrites them.  Rows of envs that did not finish are not written.
// POL (XM == 0 only, mgb_quad_rollout_policy): the action of step t is drawn from the MLP policy `pol` (mgb_policy.cuh)
// on the observation the env holds before step t, which each step leaves in the thread's column of the activation
// buffers in dynamic shared memory (at t = 0: the observation of the loaded state).  The weights are staged once per
// CTA: the one member of a population that drives the CTA's envs, or its pol.copies members back to back, each warp
// reading its own (mgb_population_stage).  The step arithmetic after the action is the code the other instantiations
// run.
// VAL (POL and FIN only, mgb_quad_rollout_critic): the output layer has the value row (mgb_mlp_forward<true>).  Step t
// stores V(s_t); a truncated step's terminal observation o[] goes through the policy once more before observe_reset
// (final_value); after the loop one more pass gives value_last, and the epilogue (mgb_gae) walks the thread's column.
template <bool SIMPLE, int XM, bool FIN, bool POL = false, bool VAL = false>
__global__ void __launch_bounds__(kThreads, POL ? 3 : 8) quad_rollout_kernel(const __grid_constant__ QuadConst c,
                                                                          const __grid_constant__ QuadArgs a,
                                                                          const __grid_constant__ MgbMlp pol,
                                                                          const __grid_constant__ mgb_critic cr)
{
    static_assert(!VAL || (POL && FIN), "value heads run on the policy rollouts with terminal outputs");
    __shared__ __align__(128) float tiles[2][kThreads * kMaxObs];
    const int64_t e0 = (int64_t)blockIdx.x * kThreads;
    const int64_t e = e0 + threadIdx.x;
    const int rows = (int)((a.n - e0) < kThreads ? (a.n - e0) : kThreads);
    const int D = c.obs_dim;
    const bool active = e < a.n;
    QState s;
    float adj[9], id = 1.f;
    if (active) {
        load_state(a, e, s);
        adjugate(s.R, adj, id);
    }
    const uint2 akey = make_uint2((uint32_t)a.act_seed, (uint32_t)(a.act_seed >> 32));
    const int64_t genv = a.env_base + e;
    const int task = active ? env_task(c, a, e) : 0;
    const float *pol_w = nullptr;           // the staged weights (mgb_population_weights)
    float *pol_x = nullptr, *pol_y = nullptr;   // the two activation buffers
    if constexpr (POL) {
        static_assert(!POL || XM == 0, "policy rollouts are not mirrored");
        extern __shared__ __align__(16) float pol_smem[];
        pol_x = pol_smem + pol.copies * pol.staged;
        pol_y = pol_x + pol.maxw * kThreads;
        pol_w = pol_smem;
        mgb_population_stage(pol, pol_smem, e0, rows, kThreads);
        if (active) {       // the observation of the loaded state: what the preceding reset() / step() returned
            float o[kMaxObs], bv[3], Ri[9];
            observe(c, s, adj, id, o, bv, Ri);
            if (c.task == MGB_TASK_VELOCITY_CONTROL) {
                const float4 q = target_row(a, task, s.ct[0] < c.nt - 1 ? s.ct[0] : c.nt - 1);
                o[16] = q.x; o[17] = q.y; o[18] = q.z;
            }
#pragma unroll
            for (int k = 0; k < kMaxObs; ++k)
                if (k < D) pol_x[k * kThreads + threadIdx.x] = o[k];
            if (pol.obs0_out) {
#pragma unroll
                for (int k = 0; k < kMaxObs; ++k)
                    if (k < D) pol.obs0_out[e * D + k] = o[k];
            }
        }
    }
    // software pipeline: the action of step t+1 is requested while step t integrates
    float4 act_next = make_float4(0.f, 0.f, 0.f, 0.f);
    if (active && a.act) act_next = __ldg(reinterpret_cast<const float4 *>(a.act) + e);
    for (int t = 0; t < a.T; ++t) {
        float *tile = tiles[t & 1];
        // the bulk store issued two steps ago must have finished READING this tile before we overwrite it
        if (threadIdx.x == 0) mgb_bulk_wait_read<1>();
        __syncthreads();
        uint32_t done_byte = 0;
        if (active) {
            float4 act;
            if constexpr (POL) {
                float mean[4], av[4], lp, v;
                mgb_population_weights(pol, pol_w, pol.staged, [&](const float *w) {
                    mgb_mlp_forward<VAL>(pol, w, pol_x, pol_y, kThreads, threadIdx.x, mean, &v);
                    lp = mgb_gaussian_action(pol, w, genv, a.t_base + (uint32_t)t, mean, av);
                });
                if constexpr (VAL) cr.value_dev[(int64_t)t * a.n + e] = v;
                act = make_float4(av[0], av[1], av[2], av[3]);
                if (a.act_out) reinterpret_cast<float4 *>(a.act_out)[(int64_t)t * a.n + e] = act;
                if (pol.logp_out) pol.logp_out[(int64_t)t * a.n + e] = lp;
            } else if (a.act) {
                act = act_next;
                if (t + 1 < a.T) act_next = __ldg(reinterpret_cast<const float4 *>(a.act) + (int64_t)(t + 1) * a.n + e);
            } else {
                const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32),
                                                             a.t_base + (uint32_t)t, MGB_STREAM_ACTION),
                                                  akey);
                const float span = c.vmax - c.vmin;
                act = make_float4(fmaf(span, mgb_u01(r.x), c.vmin), fmaf(span, mgb_u01(r.y), c.vmin),
                                  fmaf(span, mgb_u01(r.z), c.vmin), fmaf(span, mgb_u01(r.w), c.vmin));
                if (a.act_out) {
                    float4 *ap = reinterpret_cast<float4 *>(a.act_out) + (int64_t)t * a.n + e;
                    if (XM == 2) mgb_mc_st(mgb_shift(ap, a.mir.delta[0]), act);
                    else *ap = act;
                    if (XM == 1) mgb_mirror_store(a.mir, ap, act);
                }
            }
            s.ct[0] += 1;
            TargetRows<float> tr;
            const float z_old = s.p[2] + c.z_off;
            const float x_old = s.p[0], y_old = s.p[1];
            float power;
            int fail[1];
            fail[0] = integrate1<SIMPLE>(c, s, act, adj, id, power);
            if (c.task == MGB_TASK_VELOCITY_CONTROL) prefetch_targets(c, a, task, s.ct[0], 0, tr);
            float o[kMaxObs], reward;
            int done[1], trunc[1];
            bool wf[1];
            finish_step<float>(c, a, e, s, adj, id, z_old, x_old, y_old, power, fail, tr, o, reward, done, wf, trunc);
            if (FIN) {
                static_assert(!FIN || XM == 0, "terminal rows and truncation flags are not mirrored");
                if (a.truncated) a.truncated[(int64_t)t * a.n + e] = (uint8_t)trunc[0];
                if (wf[0] && a.final_obs) {
                    float *frow = a.final_obs + ((int64_t)t * a.n + e) * D;
#pragma unroll
                    for (int k = 0; k < 16; ++k) frow[k] = o[k];
                    if (D == 19) { frow[16] = o[16]; frow[17] = o[17]; frow[18] = o[18]; }
                }
            }
            if constexpr (VAL) {
                // the cut is every done (auto_reset is on): V of the terminal observation where it was truncated
                if (wf[0] && trunc[0]) {
#pragma unroll
                    for (int k = 0; k < kMaxObs; ++k)
                        if (k < D) pol_x[k * kThreads + threadIdx.x] = o[k];
                    float out4[4], v;
                    mgb_population_weights(pol, pol_w, pol.staged, [&](const float *w) {
                        mgb_mlp_forward<true>(pol, w, pol_x, pol_y, kThreads, threadIdx.x, out4, &v);
                    });
                    if (cr.final_value_dev) cr.final_value_dev[(int64_t)t * a.n + e] = v;
                }
            }
            if (wf[0]) {
                observe_reset(c, a, task, s, 0, o);
                adjugate(s.R, adj, id);
            }
            if (a.rew) {
                if (XM == 2) mgb_mc_st(mgb_shift(a.rew + (int64_t)t * a.n + e, a.mir.delta[0]), reward);
                else a.rew[(int64_t)t * a.n + e] = reward;
                if (XM == 1) mgb_mirror_store(a.mir, a.rew + (int64_t)t * a.n + e, reward);
            }
            done_byte = (uint32_t)done[0];
            if (a.done && XM != 2) {
                a.done[(int64_t)t * a.n + e] = (uint8_t)done[0];
                if (XM == 1) mgb_mirror_store(a.mir, a.done + (int64_t)t * a.n + e, (uint8_t)done[0]);
            }
            if (a.obs) {
                float *orow = tile + threadIdx.x * D;
#pragma unroll
                for (int k = 0; k < 16; ++k) orow[k] = o[k];
                if (D == 19) { orow[16] = o[16]; orow[17] = o[17]; orow[18] = o[18]; }
            }
            if constexpr (POL) {       // the policy's input at step t + 1
#pragma unroll
                for (int k = 0; k < kMaxObs; ++k)
                    if (k < D) pol_x[k * kThreads + threadIdx.x] = o[k];
            }
        }
        if (XM == 2) {
            // n % 4 == 0 (checked on the host): the four done bytes of lanes 4k..4k+3 are all valid or all not
            if (a.done) mgb_mc_st_bytes(mgb_shift(a.done + (int64_t)t * a.n + e, a.mir.delta[0]), done_byte, active);
            if (a.obs) {
                __syncthreads();
                mgb_mc_copy_tile(mgb_shift(a.obs + ((int64_t)t * a.n + e0) * D, a.mir.delta[0]), tile,
                                 (uint32_t)rows * (uint32_t)D * 4u);
            }
        } else if (a.obs) {
            if (XM == 1) publish_tile_mirrored(a.mir, a.obs + (int64_t)t * a.n * D, tile, e0, rows, D);
            else publish_tile(a.obs + (int64_t)t * a.n * D, tile, e0, rows, D);
        }
    }
    if (active) store_state(a, e, s);
    if constexpr (VAL) {
        if (active) {
            float out4[4], v;
            mgb_population_weights(pol, pol_w, pol.staged, [&](const float *w) {
                mgb_mlp_forward<true>(pol, w, pol_x, pol_y, kThreads, threadIdx.x, out4, &v);
            });
            if (cr.value_last_dev) cr.value_last_dev[e] = v;
            if (cr.adv_dev) mgb_gae(cr, a.T, a.n, e, v, a.rew, a.done, a.truncated, false);
        }
    }
    if (threadIdx.x == 0) mgb_bulk_wait_read<0>();   // smem must outlive the copy; the kernel boundary flushes the writes
}

// QuadrotorSim.reset for masked envs + observation of every env (env.py:116-125)
__global__ void __launch_bounds__(kThreads) quad_reset_kernel(const __grid_constant__ QuadConst c,
                                                              const __grid_constant__ QuadArgs a,
                                                              const uint8_t *__restrict__ mask,
                                                              const double *__restrict__ noise)
{
    const int64_t e = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= a.n) return;
    QState s;
    load_state(a, e, s);
    if (!mask || mask[e]) {
        double u[12];
        if (noise) {
#pragma unroll
            for (int k = 0; k < 12; ++k) u[k] = noise[e * 12 + k];
        } else {
            s.ep[0] += 1;
            philox_reset_draws(a.seed, a.env_base + e, s.ep[0], u);
        }
        reset_env(c, s, 0, u);
        store_state(a, e, s);
    }
    if (a.obs) {
        float adj[9], id, o[kMaxObs], bv[3], Ri[9];
        adjugate(s.R, adj, id);
        observe(c, s, adj, id, o, bv, Ri);
        if (c.task == MGB_TASK_VELOCITY_CONTROL) {
            const float4 q = target_row(a, env_task(c, a, e), s.ct[0] < c.nt - 1 ? s.ct[0] : c.nt - 1);
            o[16] = q.x; o[17] = q.y; o[18] = q.z;
        }
        float *dst = a.obs + e * c.obs_dim;
#pragma unroll
        for (int k = 0; k < 16; ++k) dst[k] = o[k];
        if (c.obs_dim == 19) { dst[16] = o[16]; dst[17] = o[17]; dst[18] = o[18]; }
    }
}

// [n][22] row-major float32 + ct  <->  state planes
__global__ void quad_state_kernel(QuadArgs a, float *state, int32_t *ct, int load)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    QState s;
    load_state(a, e, s);
    float *row = state + e * 22;
    if (load) {
        for (int k = 0; k < 3; ++k) { s.p[k] = row[k]; s.v[k] = row[3 + k]; s.om[k] = row[6 + k]; }
        for (int k = 0; k < 4; ++k) s.w[k] = row[9 + k];
        for (int k = 0; k < 9; ++k) s.R[k] = row[13 + k];
        if (ct) s.ct[0] = ct[e];
        store_state(a, e, s);
    } else {
        for (int k = 0; k < 3; ++k) { row[k] = s.p[k]; row[3 + k] = s.v[k]; row[6 + k] = s.om[k]; }
        for (int k = 0; k < 4; ++k) row[9 + k] = s.w[k];
        for (int k = 0; k < 9; ++k) row[13 + k] = s.R[k];
        if (ct) ct[e] = s.ct[0];
    }
}

__global__ void quad_init_kernel(QuadArgs a)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n_pad) return;
    QState s;
    for (int k = 0; k < 3; ++k) s.p[k] = s.v[k] = s.om[k] = 0.f;
    for (int k = 0; k < 4; ++k) s.w[k] = 0.f;
    for (int k = 0; k < 9; ++k) s.R[k] = (k % 4 == 0) ? 1.f : 0.f;
    s.ct[0] = 0;
    s.ep[0] = 0;
    store_state(a, e, s);
}

// define_velocity_control_task (quadrotorsim.py:306-319): one thread per task seed integrates nt steps from the zero
// state with host-replayed actions and records global_velocity after every step.
template <bool SIMPLE>
__global__ void quad_targets_kernel(const __grid_constant__ QuadConst c, const float *__restrict__ act, int n_tasks,
                                    float *__restrict__ tbl)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_tasks) return;
    QState s;
    for (int q = 0; q < 3; ++q) s.p[q] = s.v[q] = s.om[q] = 0.f;
    for (int q = 0; q < 4; ++q) s.w[q] = 0.f;
    for (int q = 0; q < 9; ++q) s.R[q] = (q % 4 == 0) ? 1.f : 0.f;
    s.ct[0] = 0; s.ep[0] = 0;
    float adj[9], id, power;
    adjugate(s.R, adj, id);
    for (int t = 0; t < c.nt; ++t) {
        const float4 a4 = reinterpret_cast<const float4 *>(act)[(int64_t)k * c.nt + t];
        const int fail = integrate1<SIMPLE>(c, s, a4, adj, id, power);
        float *dst = tbl + ((int64_t)k * c.nt + t) * 3;
        dst[0] = s.v[0]; dst[1] = s.v[1]; dst[2] = s.v[2];
        if (fail) {   // the reference would raise here; fill the rest with NaN so the caller notices
            for (int r = t + 1; r < c.nt; ++r) {
                float *d2 = tbl + ((int64_t)k * c.nt + r) * 3;
                d2[0] = d2[1] = d2[2] = __int_as_float(0x7fc00000);
            }
            return;
        }
    }
}

// mgb_quad_set_targets: task-major [n_tasks][nt][3] float32 -> the handle's time-major [nt][n_tasks] float4 (x, y, z, 0),
// one thread per row (values copied, not recomputed)
__global__ void quad_targets_layout_kernel(const float *__restrict__ src, int nt, int n_tasks, float4 *__restrict__ dst)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;     // = t * n_tasks + task
    if (i >= (int64_t)nt * n_tasks) return;
    const int64_t t = i / n_tasks, k = i % n_tasks;
    const float *s = src + (k * nt + t) * 3;
    dst[i] = make_float4(s[0], s[1], s[2], 0.f);
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// handle + C ABI
// ---------------------------------------------------------------------------------------------------------------
// host staging of the *_host entry points: device buffers d_*, pinned host buffers h_*
struct QuadStaging {
    MgbDev<float> d_act, d_obs, d_rew, d_final;
    MgbDev<uint8_t> d_done, d_trunc;
    MgbDev<int32_t> d_fail;
    MgbPinned<float> h_act, h_obs, h_rew, h_final;
    MgbPinned<uint8_t> h_done, h_trunc;
    MgbPinned<int32_t> h_fail;
};

struct mgb_quad {
    int device = 0;
    int64_t n = 0, n_pad = 0, env_base = 0;
    mgb_quad_cfg cfg;
    QuadConst c;
    MgbDev<float4> planes;
    MgbDev<int32_t> sat;
    int map_rows = 0, map_cols = 0, x_off = 0, y_off = 0;
    MgbDev<float4> targets;     // [nt][n_tasks] (x, y, z, 0), built by mgb_quad_set_targets
    MgbDev<int32_t> env2task;
    int n_tasks = 0;
    int auto_reset = 0;
    int num_sms = 132;
    int wide_kernel = -1;      // MGB_WIDE_KERNEL: unset = by batch size (plan_step), 1 = every single-wave launch, 0 = never
    int packed = 0;            // MGB_PACKED=1: two envs per thread (bit-identical to one env per thread)
    int stream_kernel = 1;     // persistent TMA-pipelined kernel for multi-wave launches (MGB_STREAM_KERNEL=0 disables)
    int pdl = 1;               // programmatic dependent launch of consecutive step kernels (MGB_PDL=0 disables)
    int zerocopy = 1;          // host entry point: kernel reads/writes pinned host buffers directly (MGB_HOST_ZEROCOPY=0)
    uint64_t seed = 0;
    uint32_t t_base = 0;
    int64_t launches = 0;
    uint64_t fp_map = 0, fp_targets = 0;   // fingerprints of the map (0: flat) and the target table (mgb_quad_fingerprint)
    MgbMirrors mir = {};       // mgb_quad_set_mirrors
    MgbMirrorWindow mir_win;   // mgb_quad_set_mirror_window
    QuadStaging stage;         // allocated by the first *_host call
};

static QuadArgs base_args(const mgb_quad *h)
{
    QuadArgs a;
    memset(&a, 0, sizeof(a));
    a.planes = h->planes.get();
    a.n_pad = h->n_pad;
    a.n = h->n;
    a.env_base = h->env_base;
    a.targets = h->targets.get();
    a.n_tasks = h->n_tasks;
    a.sat = h->sat.get(); a.map_rows = h->map_rows; a.map_cols = h->map_cols; a.x_off = h->x_off; a.y_off = h->y_off;
    a.env2task = h->env2task.get();
    a.seed = h->seed;
    a.auto_reset = h->auto_reset;
    return a;
}

// Calls f(std::true_type()) for a handle whose configuration takes the simplified dynamics (QuadConst::simple), else
// f(std::false_type()): the one place where the SIMPLE argument of a kernel template is chosen
template <class F> static auto with_simple(const mgb_quad *h, F &&f)
{
    return h->c.simple ? f(std::true_type()) : f(std::false_type());
}

static int derive_constants(const mgb_quad_cfg *g, QuadConst *c)
{
    memset(c, 0, sizeof(*c));
    c->h = (float)g->precision;
    c->k1 = (float)(g->phi / g->ra);
    c->k1phi = (float)(g->phi / g->ra * g->phi);
    c->inv_phi = (float)(1.0 / g->phi);
    c->hjm = (float)(g->precision / g->jm);
    c->hk = (float)(g->precision / g->jm * (g->phi / g->ra * g->phi));
    c->mm = (float)g->mm;
    c->ct0 = (float)g->ct[0]; c->ct1 = (float)g->ct[1]; c->ct2 = (float)g->ct[2];
    c->vmin = (float)g->min_voltage; c->vmax = (float)g->max_voltage;
    bool simple = (g->ct[2] == 0.0);
    for (int i = 0; i < 4; ++i) {
        c->px[i] = g->propeller[3 * i]; c->py[i] = g->propeller[3 * i + 1]; c->pz[i] = g->propeller[3 * i + 2];
        c->A[i] = (float)((double)c->py[i] * (double)g->propeller_norm[i]);
        c->B[i] = (float)((double)c->px[i] * (double)g->propeller_norm[i]);
        if (c->pz[i] != 0.f) simple = false;
    }
    for (int k = 0; k < 3; ++k) {
        c->Df[k] = g->drag_f[k]; c->Dm[k] = g->drag_m[k]; c->cg[k] = g->gravity_center[k];
        if (c->cg[k] != 0.f) simple = false;
        c->init_v[k] = g->init_velocity[k]; c->init_w[k] = g->init_angular_velocity[k];
    }
    for (int k = 0; k < 9; ++k) {
        c->hI[k] = (float)(g->precision * (double)g->inv_inertia[k]);
        if (k % 4 != 0 && g->inv_inertia[k] != 0.f) simple = false;
    }
    c->gm = (float)((double)(float)-9.8 * g->quality);
    c->c_hm = (float)(g->precision / g->quality);
    c->c_h2m = (float)(0.5 * g->precision * g->precision / g->quality);
    c->fail_r2 = (float)(g->fail_range * g->fail_range);
    c->fail_v2 = (float)(g->fail_velocity * g->fail_velocity);
    c->fail_w2 = (float)(g->fail_w * g->fail_w);
    c->dt = (float)g->dt; c->healthy = (float)g->healthy_reward; c->z_off = (float)g->z_offset;
    c->noise_v = (float)g->init_velocity_noise; c->noise_w = (float)g->init_angular_velocity_noise;
    c->nt = g->nt; c->task = g->task;
    c->substeps = (int)(g->dt / g->precision);          // quadrotorsim.py:302, evaluated in double like python
    c->rk4_steps = g->integrator == MGB_INTEGRATOR_RK4 ? (g->rk4_steps > 0 ? g->rk4_steps : 1) : 0;
    c->rk4_h = c->rk4_steps ? (float)(g->dt / c->rk4_steps) : 0.f;
    c->inv_jm = (float)(1.0 / g->jm);
    c->inv_m = (float)(1.0 / g->quality);
    for (int k = 0; k < 9; ++k) c->Iinv[k] = g->inv_inertia[k];
    c->obs_dim = g->task == MGB_TASK_VELOCITY_CONTROL ? 19 : 16;
    c->simple = simple ? 1 : 0;
    return 0;
}

extern "C" int mgb_quad_create(mgb_quad **out, int64_t n_envs, const mgb_quad_cfg *cfg, int device,
                               int64_t env_index_base)
{
    MGB_REQUIRE(out && cfg, "null argument");
    MGB_REQUIRE(n_envs > 0, "n_envs must be positive");
    MGB_REQUIRE(cfg->task >= 0 && cfg->task <= 2, "invalid task");                 // env.py:55-56
    MGB_REQUIRE(cfg->nt > 0, "nt must be positive");
    // quadrotorsim.py:299-300
    MGB_REQUIRE(!(cfg->precision < 1e-8 || cfg->precision > cfg->dt), "Inproper parameter of precision");
    int ndev = 0;
    MGB_CUDA(cudaGetDeviceCount(&ndev));
    MGB_REQUIRE(device >= 0 && device < ndev, "device index out of range");
    MgbDeviceGuard guard(device);
    std::unique_ptr<mgb_quad> h(new (std::nothrow) mgb_quad());    // deleted with its buffers on every error exit
    MGB_REQUIRE(h, "out of host memory");
    h->device = device;
    h->n = n_envs;
    h->n_pad = (n_envs + 127) / 128 * 128;
    h->env_base = env_index_base;
    h->cfg = *cfg;
    derive_constants(cfg, &h->c);
    if (const char *ev = getenv("MGB_PDL")) h->pdl = atoi(ev) != 0;
    {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) h->num_sms = prop.multiProcessorCount;
    }
    if (const char *ev = getenv("MGB_HOST_ZEROCOPY")) h->zerocopy = atoi(ev);   // 0 copies, 1 zero-copy, 2 hybrid
    if (const char *ev = getenv("MGB_STREAM_KERNEL")) h->stream_kernel = atoi(ev) != 0;
    if (const char *ev = getenv("MGB_PACKED")) h->packed = atoi(ev) != 0;
    if (const char *ev = getenv("MGB_WIDE_KERNEL")) h->wide_kernel = atoi(ev) != 0;
    {
        // the one-CTA-per-SM step kernels need up to 2 x 512 x 19 floats of dynamic shared memory; the attribute is per
        // function and device, idempotent, and set to the maximum so that handles never lower each other's limit (round-1
        // advice: the process-global high-water mark it replaces was not thread-safe), for the kernels this handle launches
        const int max_smem = 512 * kMaxObs * 4 * 2;
        with_simple(h.get(), [&](auto simple) {
            cudaFuncSetAttribute(quad_step_wide_kernel<simple>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
            cudaFuncSetAttribute(quad_step2_kernel<simple>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem);
        });
        if (cudaGetLastError() != cudaSuccess) {
            mgb_set_error("cudaFuncSetAttribute(quad_step_wide_kernel, %d bytes of shared memory) failed", max_smem);
            return MGB_ERR_CUDA;
        }
    }
    MGB_CUDA(h->planes.alloc(sizeof(float4) * 6 * h->n_pad));        // the state planes
    quad_init_kernel<<<(unsigned)((h->n_pad + 255) / 256), 256>>>(base_args(h.get()));
    MGB_CUDA(cudaDeviceSynchronize());
    h->launches += 1;
    *out = h.release();
    return MGB_OK;
}

extern "C" void mgb_quad_destroy(mgb_quad *h)
{
    if (!h) return;
    MgbDeviceGuard guard(h->device);
    cudaDeviceSynchronize();
    delete h;                  // the members free the handle's buffers while its device is current
}

extern "C" int mgb_quad_obs_dim(const mgb_quad *h) { return h ? h->c.obs_dim : MGB_ERR_ARG; }
extern "C" int64_t mgb_quad_num_envs(const mgb_quad *h) { return h ? h->n : MGB_ERR_ARG; }
extern "C" int64_t mgb_quad_launch_count(const mgb_quad *h) { return h ? h->launches : MGB_ERR_ARG; }

extern "C" int mgb_quad_set_options(mgb_quad *h, int auto_reset, uint64_t seed)
{
    MGB_REQUIRE(h, "null handle");
    h->auto_reset = auto_reset ? 1 : 0;
    h->seed = seed;
    return MGB_OK;
}

extern "C" int mgb_quad_set_map(mgb_quad *h, const int32_t *map_host, int32_t rows, int32_t cols)
{
    MGB_REQUIRE(h, "null handle");
    MgbDeviceGuard guard(h->device);
    MGB_CUDA(cudaDeviceSynchronize());
    if (!map_host) {                                            // flat default map, env.py:295-298
        h->sat.reset();
        h->map_rows = h->map_cols = h->x_off = h->y_off = 0;
        h->fp_map = 0;
        return MGB_OK;
    }
    MGB_REQUIRE(h->c.task != MGB_TASK_VELOCITY_CONTROL, "velocity_control has no map (env.py:101-104)");
    MGB_REQUIRE(rows > 0 && cols > 0 && rows <= 8192 && cols <= 8192, "map size out of range");
    int starts = 0, sr = 0, sc = 0;
    for (int r = 0; r < rows; ++r)
        for (int q = 0; q < cols; ++q)
            if (map_host[(size_t)r * cols + q] == -1) { ++starts; sr = r; sc = q; }
    MGB_REQUIRE(starts == 1, "the map must mark exactly one start cell with -1 (env.py:108-109)");
    std::vector<int32_t> sat((size_t)(rows + 1) * (cols + 1), 0);
    for (int r = 0; r < rows; ++r)
        for (int q = 0; q < cols; ++q) {
            const int v = (r == sr && q == sc) ? 0 : map_host[(size_t)r * cols + q];    // env.py:113
            sat[(size_t)(r + 1) * (cols + 1) + q + 1] = (v != 0 ? 1 : 0) + sat[(size_t)r * (cols + 1) + q + 1] +
                                                        sat[(size_t)(r + 1) * (cols + 1) + q] - sat[(size_t)r * (cols + 1) + q];
        }
    MgbDev<int32_t> d_sat;
    MGB_CUDA(d_sat.alloc(sat.size() * sizeof(int32_t)));
    MGB_CUDA(cudaMemcpy(d_sat.get(), sat.data(), sat.size() * sizeof(int32_t), cudaMemcpyHostToDevice));
    h->sat = std::move(d_sat);
    h->map_rows = rows; h->map_cols = cols; h->x_off = sc; h->y_off = sr;
    h->fp_map = mgb_fnv(mgb_fnv(mgb_fnv(MGB_FNV_BASIS, &rows, sizeof(rows)), &cols, sizeof(cols)), map_host,
                        (size_t)rows * cols * sizeof(int32_t));
    return MGB_OK;
}

extern "C" int mgb_quad_set_targets(mgb_quad *h, const float *tbl_dev, int32_t n_tasks, const int32_t *env2task_dev)
{
    MGB_REQUIRE(h && tbl_dev && env2task_dev, "null argument");
    MGB_REQUIRE(n_tasks > 0, "n_tasks must be positive");
    MgbDeviceGuard guard(h->device);
    MGB_CUDA(cudaDeviceSynchronize());
    // the kernels read the table time-major with 16-byte rows (prefetch_targets): 16 instead of 12 bytes per row
    const int64_t rows = (int64_t)h->c.nt * n_tasks;
    MgbDev<float4> targets;
    MgbDev<int32_t> env2task;
    MGB_CUDA(targets.alloc(sizeof(float4) * (size_t)rows));
    MGB_CUDA(env2task.alloc(sizeof(int32_t) * h->n));
    quad_targets_layout_kernel<<<(unsigned)((rows + 255) / 256), 256>>>(tbl_dev, h->c.nt, n_tasks, targets.get());
    MGB_CUDA(cudaGetLastError());
    MGB_CUDA(cudaMemcpy(env2task.get(), env2task_dev, sizeof(int32_t) * h->n, cudaMemcpyDeviceToDevice));
    // a device-to-device cudaMemcpy may return before the copy is done, and a step launched next on a non-blocking
    // stream would not be ordered after it (nor after the layout kernel)
    MGB_CUDA(cudaDeviceSynchronize());
    std::vector<float4> tbl((size_t)rows);
    MGB_CUDA(cudaMemcpy(tbl.data(), targets.get(), tbl.size() * sizeof(float4), cudaMemcpyDeviceToHost));
    h->targets = std::move(targets); h->env2task = std::move(env2task);
    h->n_tasks = n_tasks;
    h->fp_targets = mgb_fnv(mgb_fnv(MGB_FNV_BASIS, &n_tasks, sizeof(n_tasks)), tbl.data(), tbl.size() * sizeof(float4));
    return MGB_OK;
}

static int check_ready(const mgb_quad *h)
{
    if (h->c.task == MGB_TASK_VELOCITY_CONTROL && !h->targets) {
        mgb_set_error("velocity_control: call mgb_quad_set_targets before reset/step");
        return MGB_ERR_STATE;
    }
    return MGB_OK;
}

extern "C" int mgb_quad_make_targets(mgb_quad *h, const float *act_dev, int32_t n_tasks, float *tbl_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_make_targets");
    MGB_REQUIRE(h && act_dev && tbl_dev, "null argument");
    MGB_REQUIRE(n_tasks > 0, "n_tasks must be positive");
    MgbDeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = 32, blocks = (n_tasks + threads - 1) / threads;
    with_simple(h, [&](auto simple) {
        quad_targets_kernel<simple><<<blocks, threads, 0, st>>>(h->c, act_dev, n_tasks, tbl_dev);
    });
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

extern "C" int mgb_quad_reset(mgb_quad *h, const uint8_t *mask_dev, const double *noise_dev, float *obs_dev,
                              void *stream)
{
    MgbRange nvtx_range("mgb_quad_reset");
    MGB_REQUIRE(h, "null handle");
    int rc = check_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    QuadArgs a = base_args(h);
    a.obs = obs_dev;
    quad_reset_kernel<<<(unsigned)((h->n + kThreads - 1) / kThreads), kThreads, 0, (cudaStream_t)stream>>>(
        h->c, a, mask_dev, noise_dev);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// A step launch of this handle: the kernel and its name (mgb_quad_step_kernel reports it for the bench line), the launch
// shape, and QuadArgs::per_cta of the one-CTA-per-SM kernels (0 for the others)
struct StepPlan {
    void (*kernel)(QuadConst, QuadArgs);
    const char *name;
    dim3 grid, block;
    size_t smem = 0;
    int per_cta = 0;
};

static StepPlan plan_step(const mgb_quad *h, const QuadArgs &a)
{
#define STEP_KERNEL(k) k<simple>, simple ? #k "<true>" : #k "<false>"
    return with_simple(h, [&](auto simple) {
        const unsigned blocks = (unsigned)((a.n + kThreads - 1) / kThreads);
        const bool act16 = (reinterpret_cast<uintptr_t>(a.act) & 15u) == 0;
        // multi-wave launches stream: persistent CTAs + TMA double buffering (quad_stream_kernel)
        if (h->stream_kernel && (int64_t)blocks > (int64_t)h->num_sms * 32 && act16)
            return StepPlan{STEP_KERNEL(quad_stream_kernel), dim3((unsigned)(h->num_sms * 4)), dim3(kStreamThreads)};
        // the packed kernel stores reward / done / fail / truncated of an env pair with one 8 / 2 / 8 / 2-byte access
        const bool packed = h->packed && h->c.rk4_steps == 0 && a.n >= 2 && act16 &&
                            (reinterpret_cast<uintptr_t>(a.rew) & 7u) == 0 && (reinterpret_cast<uintptr_t>(a.done) & 1u) == 0 &&
                            (reinterpret_cast<uintptr_t>(a.fail) & 7u) == 0 && (reinterpret_cast<uintptr_t>(a.truncated) & 1u) == 0;
        // launches that fit one wave of 512-thread CTAs: one CTA per SM.  Measured on an H100 80GB HBM3 (700 W power limit,
        // velocity_control dt = 0.005, CUDA graphs of 256 steps, medians of 3 runs), us per step tile / wide: 9 473 envs
        // 4.87 / 3.09, 24 576 envs 5.26 / 4.73, 49 152 envs 6.88 / 5.89, but 65 536 envs 6.79 / 8.09 and 67 001 envs 7.39 / 7.90.
        // So by default the wide kernel takes batches of up to 384 envs per SM and the 64-env tile kernel the rest.
        const bool single_wave = a.n <= (int64_t)h->num_sms * 512 && a.n >= (int64_t)h->num_sms * 64;
        const int64_t wide_max = (int64_t)h->num_sms * (h->wide_kernel > 0 ? 512 : 384);
        if (!packed && !(h->wide_kernel != 0 && single_wave && a.n <= wide_max))
            return StepPlan{STEP_KERNEL(quad_step_kernel), dim3(blocks), dim3(kThreads)};
        // envs per CTA: one CTA per SM when the launch fits a single wave; the packed kernel also serves the other sizes
        int per = single_wave ? (int)((a.n + h->num_sms - 1) / h->num_sms) : a.n < (int64_t)h->num_sms * 64 ? 64 : 256;
        per = (per + 3) / 4 * 4;
        const dim3 grid((unsigned)((a.n + per - 1) / per)), block((unsigned)((per / (packed ? 2 : 1) + 31) / 32 * 32));
        const size_t smem = (size_t)per * kMaxObs * 4 * 2;
        if (packed) return StepPlan{STEP_KERNEL(quad_step2_kernel), grid, block, smem, per};
        return StepPlan{STEP_KERNEL(quad_step_wide_kernel), grid, block, smem, per};
    });
#undef STEP_KERNEL
}

static int launch_step(mgb_quad *h, QuadArgs a, cudaStream_t st)
{
    const StepPlan p = plan_step(h, a);
    a.per_cta = p.per_cta;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = p.grid;
    cfg.blockDim = p.block;
    cfg.dynamicSmemBytes = p.smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = h->pdl ? 1 : 0;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MGB_CUDA(cudaLaunchKernelEx(&cfg, p.kernel, h->c, a));
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

extern "C" const char *mgb_quad_step_kernel(const mgb_quad *h) { return h ? plan_step(h, base_args(h)).name : ""; }

static int step_dev(mgb_quad *h, const float *act_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                    int32_t *fail_dev, float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MGB_REQUIRE(h && act_dev && obs_dev && rew_dev && done_dev, "null argument");
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(act_dev) & 15u) == 0, "act_dev must be 16-byte aligned");
    int rc = check_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    QuadArgs a = base_args(h);
    a.act = act_dev; a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev; a.fail = fail_dev;
    a.final_obs = final_obs_dev;
    a.truncated = truncated_dev;
    return launch_step(h, a, (cudaStream_t)stream);
}

extern "C" int mgb_quad_step(mgb_quad *h, const float *act_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                             int32_t *fail_dev, float *final_obs_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_step");
    return step_dev(h, act_dev, obs_dev, rew_dev, done_dev, fail_dev, final_obs_dev, nullptr, stream);
}

extern "C" int mgb_quad_step_ex(mgb_quad *h, const float *act_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                                int32_t *fail_dev, float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_step_ex");
    return step_dev(h, act_dev, obs_dev, rew_dev, done_dev, fail_dev, final_obs_dev, truncated_dev, stream);
}

static int rollout(mgb_quad *h, int32_t T, const float *act_dev, uint64_t act_seed, float *act_out_dev, float *obs_dev,
                   float *rew_dev, uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MGB_REQUIRE(h, "null handle");
    MGB_REQUIRE(T > 0, "T must be positive");
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(act_dev) & 15u) == 0, "act_dev must be 16-byte aligned");
    const bool fin = final_obs_dev || truncated_dev;
    MGB_REQUIRE(!final_obs_dev || h->auto_reset, "final_obs needs auto_reset on (without it obs already is the terminal observation)");
    MGB_REQUIRE(!fin || h->mir.count == 0,
                "final_obs / truncated are not delivered through output mirrors or multicast (set_mirrors([]) first)");
    int rc = check_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    QuadArgs a = base_args(h);
    a.act = act_dev; a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev;
    a.T = T; a.act_seed = act_seed; a.t_base = h->t_base; a.act_out = act_out_dev;
    a.final_obs = final_obs_dev; a.truncated = truncated_dev;
    const unsigned blocks = (unsigned)((a.n + kThreads - 1) / kThreads);
    a.mir = h->mir;
    if (h->mir.count != 0)
        MGB_REQUIRE(h->mir_win.holds_rollout((uint64_t)T * h->n, obs_dev, (uint64_t)h->c.obs_dim * 4, rew_dev, 4, done_dev,
                                             act_out_dev, 16),
                    "mirrors are on but an output lies outside the mirrored arena (set_mirrors([]) first)");
    const int xm = h->mir.count == MGB_MIRROR_MULTICAST ? 2 : h->mir.count > 0 ? 1 : 0;
    if (xm == 2) {
        MGB_REQUIRE(h->n % 4 == 0, "multicast outputs need num_envs % 4 == 0");
        MGB_REQUIRE((((uintptr_t)done_dev | (uintptr_t)rew_dev | (uintptr_t)obs_dev) & 3) == 0 && ((uintptr_t)act_out_dev & 15) == 0,
                    "multicast outputs must be 4-byte (actions: 16-byte) aligned");
    }
    const auto kernel = with_simple(h, [&](auto simple) {
        return xm == 2 ? quad_rollout_kernel<simple, 2, false> : xm == 1 ? quad_rollout_kernel<simple, 1, false>
               : fin   ? quad_rollout_kernel<simple, 0, true>  : quad_rollout_kernel<simple, 0, false>;
    });
    kernel<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(h->c, a, MgbMlp{}, mgb_critic{});
    MGB_CUDA(cudaGetLastError());
    h->t_base += (uint32_t)T;
    h->launches += 1;
    return MGB_OK;
}

// A policy rollout of `members` policies (one: mgb_quad_rollout_policy), refused as `fn`; with a critic (the value
// heads of mgb_quad_rollout_critic, null for the other entry points) the policy has the value row
static int rollout_policy(const char *fn, mgb_quad *h, int32_t T, const mgb_policy *pol, int32_t members,
                          int64_t member_stride, uint64_t seed, float *act_out_dev, float *logp_out_dev,
                          float *obs0_out_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                          uint8_t *truncated_dev, void *stream, const mgb_critic *critic = nullptr, bool val = false)
{
    const auto refuse = [&](const char *why) {
        mgb_set_error("%s: %s", fn, why);
        return MGB_ERR_ARG;
    };
    if (!h) return refuse("null handle");
    if (T <= 0) return refuse("T must be positive");
    MgbMlp m;
    if (const char *why = mgb_mlp_plan(pol, h->c.obs_dim, true, m, val)) return refuse(why);
    if (const char *why = mgb_population_plan(m, h->n, members, member_stride, kThreads)) return refuse(why);
    if (logp_out_dev && m.mode != MGB_POLICY_SAMPLE)
        return refuse("logp_out needs MGB_POLICY_SAMPLE (the mean mode draws nothing)");
    if (h->mir.count != 0)
        return refuse("policy rollouts are not delivered through output mirrors or multicast (set_mirrors([]) first)");
    if (final_obs_dev && !h->auto_reset)
        return refuse("final_obs needs auto_reset on (without it obs already is the terminal observation)");
    if ((reinterpret_cast<uintptr_t>(act_out_dev) & 15u) != 0) return refuse("act_out_dev must be 16-byte aligned");
    if ((reinterpret_cast<uintptr_t>(pol->params_dev) & 3u) != 0) return refuse("params_dev must be 4-byte aligned");
    if (val) {
        if (const char *why = mgb_critic_check(critic, h->auto_reset, rew_dev, done_dev, truncated_dev)) return refuse(why);
    }
    int rc = check_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    m.seed = seed;
    m.logp_out = logp_out_dev;
    m.obs0_out = obs0_out_dev;
    const bool fin = final_obs_dev || truncated_dev;
    const auto kernel = with_simple(h, [&](auto simple) {
        return val ? quad_rollout_kernel<simple, 0, true, true, true>
               : fin ? quad_rollout_kernel<simple, 0, true, true> : quad_rollout_kernel<simple, 0, false, true>;
    });
    const size_t smem = mgb_mlp_smem_bytes(m, kThreads);
    int optin = 0;
    MGB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
    cudaFuncAttributes fa;
    MGB_CUDA(cudaFuncGetAttributes(&fa, kernel));
    if (fa.sharedSizeBytes + smem > (size_t)optin) {
        mgb_set_error("%s: the policy needs %zu bytes of shared memory per CTA (weights and activations of %d envs), "
                      "above the device's %d", fn, fa.sharedSizeBytes + smem, kThreads, optin);
        return MGB_ERR_ARG;
    }
    MGB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    QuadArgs a = base_args(h);
    a.obs = obs_dev; a.rew = rew_dev; a.done = done_dev;
    a.T = T; a.t_base = h->t_base; a.act_out = act_out_dev;
    a.final_obs = final_obs_dev; a.truncated = truncated_dev;
    const unsigned blocks = (unsigned)((a.n + kThreads - 1) / kThreads);
    kernel<<<blocks, kThreads, smem, (cudaStream_t)stream>>>(h->c, a, m, val ? *critic : mgb_critic{});
    MGB_CUDA(cudaGetLastError());
    h->t_base += (uint32_t)T;
    h->launches += 1;
    return MGB_OK;
}

extern "C" int mgb_quad_rollout_policy(mgb_quad *h, int32_t T, const mgb_policy *pol, uint64_t seed, float *act_out_dev,
                                       float *logp_out_dev, float *obs0_out_dev, float *obs_dev, float *rew_dev,
                                       uint8_t *done_dev, float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_rollout_policy");
    return rollout_policy(__func__, h, T, pol, 1, 0, seed, act_out_dev, logp_out_dev, obs0_out_dev, obs_dev, rew_dev,
                          done_dev, final_obs_dev, truncated_dev, stream);
}

extern "C" int mgb_quad_rollout_population(mgb_quad *h, int32_t T, const mgb_policy *pol, int32_t members,
                                           int64_t member_stride, uint64_t seed, float *act_out_dev, float *logp_out_dev,
                                           float *obs0_out_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                                           float *final_obs_dev, uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_rollout_population");
    return rollout_policy(__func__, h, T, pol, members, member_stride, seed, act_out_dev, logp_out_dev, obs0_out_dev,
                          obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev, stream);
}

extern "C" int mgb_quad_rollout_critic(mgb_quad *h, int32_t T, const mgb_policy *pol, int32_t members,
                                       int64_t member_stride, uint64_t seed, float *act_out_dev, float *logp_out_dev,
                                       float *obs0_out_dev, float *obs_dev, float *rew_dev, uint8_t *done_dev,
                                       float *final_obs_dev, uint8_t *truncated_dev, const mgb_critic *critic,
                                       void *stream)
{
    MgbRange nvtx_range("mgb_quad_rollout_critic");
    return rollout_policy(__func__, h, T, pol, members, member_stride, seed, act_out_dev, logp_out_dev, obs0_out_dev,
                          obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev, stream, critic, true);
}

extern "C" int mgb_quad_rollout(mgb_quad *h, int32_t T, const float *act_dev, uint64_t act_seed, float *act_out_dev,
                                float *obs_dev, float *rew_dev, uint8_t *done_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_rollout");
    return rollout(h, T, act_dev, act_seed, act_out_dev, obs_dev, rew_dev, done_dev, nullptr, nullptr, stream);
}

extern "C" int mgb_quad_rollout_ex(mgb_quad *h, int32_t T, const float *act_dev, uint64_t act_seed, float *act_out_dev,
                                   float *obs_dev, float *rew_dev, uint8_t *done_dev, float *final_obs_dev,
                                   uint8_t *truncated_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_rollout_ex");
    return rollout(h, T, act_dev, act_seed, act_out_dev, obs_dev, rew_dev, done_dev, final_obs_dev, truncated_dev,
                   stream);
}

extern "C" int mgb_quad_set_mirrors(mgb_quad *h, int count, const int64_t *byte_delta)
{
    MGB_REQUIRE(h, "null handle");
    const char *why = h->mir.set_peers(count, byte_delta);
    MGB_REQUIRE(!why, why);
    return MGB_OK;
}

extern "C" int mgb_quad_set_mirror_window(mgb_quad *h, const void *base, uint64_t bytes)
{
    MGB_REQUIRE(h, "null handle");
    h->mir_win.set(base, bytes);
    return MGB_OK;
}

extern "C" int mgb_quad_set_multicast(mgb_quad *h, int64_t byte_delta)
{
    MGB_REQUIRE(h, "null handle");
    const char *why = h->mir.set_multicast(byte_delta);
    MGB_REQUIRE(!why, why);
    return MGB_OK;
}

static int ensure_host_staging(mgb_quad *h)
{
    if (h->stage.d_act) return MGB_OK;
    const size_t n = (size_t)h->n, D = (size_t)h->c.obs_dim;
    QuadStaging s;
    MGB_CUDA(s.d_act.alloc(n * 16));
    MGB_CUDA(s.d_obs.alloc(n * D * 4));
    MGB_CUDA(s.d_rew.alloc(n * 4));
    MGB_CUDA(s.d_done.alloc(n));
    MGB_CUDA(s.d_fail.alloc(n * 4));
    MGB_CUDA(s.d_final.alloc(n * D * 4));
    MGB_CUDA(s.d_trunc.alloc(n));
    MGB_CUDA(s.h_trunc.alloc(n));
    MGB_CUDA(cudaMemset(s.d_fail.get(), 0, n * 4));
    MGB_CUDA(cudaMemset(s.d_final.get(), 0, n * D * 4));   // rows keep the last terminal observation seen, like final_obs_dev
    MGB_CUDA(s.h_act.alloc(n * 16));
    MGB_CUDA(s.h_obs.alloc(n * D * 4));
    MGB_CUDA(s.h_rew.alloc(n * 4));
    MGB_CUDA(s.h_done.alloc(n));
    MGB_CUDA(s.h_fail.alloc(n * 4));
    MGB_CUDA(s.h_final.alloc(n * D * 4));
    h->stage = std::move(s);
    return MGB_OK;
}

// Device-visible alias of a pinned (page-locked, UVA-mapped) host buffer, or nullptr for pageable memory.
static void *pinned_device_alias(const void *p)
{
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (at.type != cudaMemoryTypeHost) return nullptr;
    return at.devicePointer;
}

static int step_host(mgb_quad *h, const float *act_host, float *obs_host, float *rew_host, uint8_t *done_host,
                     int32_t *fail_host, float *final_obs_host, uint8_t *truncated_host, void *stream)
{
    MGB_REQUIRE(h && act_host && obs_host && rew_host && done_host, "null argument");
    int rc = check_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    rc = ensure_host_staging(h);
    if (rc) return rc;
    const size_t n = (size_t)h->n, D = (size_t)h->c.obs_dim;
    const QuadStaging &s = h->stage;
    // Everything is enqueued on the CALLER's stream, so the step is ordered after whatever the caller enqueued before
    // (reset, rollout, load_state ...) exactly like mgb_quad_step; the call then waits for that stream.
    cudaStream_t st = (cudaStream_t)stream;
    // Zero-copy path: when the caller's buffers are pinned, the step kernel reads the actions from and writes
    // obs/reward/done to host memory ITSELF (UVA aliases): the PCIe traffic of both directions overlaps the arithmetic
    // inside one launch, and no copy call sits between the user and the result.  MGB_HOST_ZEROCOPY=0 forces copies.
    void *da = pinned_device_alias(act_host), *dob = pinned_device_alias(obs_host), *dr = pinned_device_alias(rew_host),
         *dd = pinned_device_alias(done_host);
    void *df = fail_host ? pinned_device_alias(fail_host) : nullptr;
    void *dfo = final_obs_host ? pinned_device_alias(final_obs_host) : nullptr;
    void *dtr = truncated_host ? pinned_device_alias(truncated_host) : nullptr;
    const bool opt_ok = (!fail_host || df) && (!final_obs_host || dfo) && (!truncated_host || dtr);
    if (h->zerocopy && da && dob && dr && dd && opt_ok && (reinterpret_cast<uintptr_t>(da) & 15u) == 0) {
        QuadArgs a = base_args(h);
        a.act = (const float *)da; a.obs = (float *)dob; a.rew = (float *)dr; a.done = (uint8_t *)dd;
        a.fail = (int32_t *)df; a.final_obs = (float *)dfo; a.truncated = (uint8_t *)dtr;
        if (h->zerocopy == 2) {
            // hybrid: actions by DMA (copy engine), outputs written to host memory by the kernel
            MGB_CUDA(cudaMemcpyAsync(s.d_act.get(), act_host, n * 16, cudaMemcpyHostToDevice, st));
            a.act = s.d_act.get();
        }
        rc = launch_step(h, a, st);
        if (rc) return rc;
        MGB_CUDA(cudaStreamSynchronize(st));
        return MGB_OK;
    }
    // Copy path: pinned caller buffers are DMA'd directly; pageable ones go through the handle's pinned staging area.
    const bool pin_in = da != nullptr;
    const bool pin_out = dob && dr && dd && opt_ok;
    const float *src = act_host;
    if (!pin_in) { memcpy(s.h_act.get(), act_host, n * 16); src = s.h_act.get(); }
    MGB_CUDA(cudaMemcpyAsync(s.d_act.get(), src, n * 16, cudaMemcpyHostToDevice, st));
    QuadArgs a = base_args(h);
    a.act = s.d_act.get(); a.obs = s.d_obs.get(); a.rew = s.d_rew.get(); a.done = s.d_done.get();
    a.fail = fail_host ? s.d_fail.get() : nullptr;
    a.final_obs = final_obs_host ? s.d_final.get() : nullptr;
    a.truncated = truncated_host ? s.d_trunc.get() : nullptr;
    rc = launch_step(h, a, st);
    if (rc) return rc;
    float *o = pin_out ? obs_host : s.h_obs.get();
    float *r = pin_out ? rew_host : s.h_rew.get();
    uint8_t *d = pin_out ? done_host : s.h_done.get();
    MGB_CUDA(cudaMemcpyAsync(o, s.d_obs.get(), n * D * 4, cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaMemcpyAsync(r, s.d_rew.get(), n * 4, cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaMemcpyAsync(d, s.d_done.get(), n, cudaMemcpyDeviceToHost, st));
    if (fail_host) MGB_CUDA(cudaMemcpyAsync(pin_out ? fail_host : s.h_fail.get(), s.d_fail.get(), n * 4, cudaMemcpyDeviceToHost, st));
    if (final_obs_host)
        MGB_CUDA(cudaMemcpyAsync(pin_out ? final_obs_host : s.h_final.get(), s.d_final.get(), n * D * 4, cudaMemcpyDeviceToHost, st));
    if (truncated_host)
        MGB_CUDA(cudaMemcpyAsync(pin_out ? truncated_host : s.h_trunc.get(), s.d_trunc.get(), n, cudaMemcpyDeviceToHost, st));
    MGB_CUDA(cudaStreamSynchronize(st));
    if (!pin_out) {
        memcpy(obs_host, s.h_obs.get(), n * D * 4);
        memcpy(rew_host, s.h_rew.get(), n * 4);
        memcpy(done_host, s.h_done.get(), n);
        if (fail_host) memcpy(fail_host, s.h_fail.get(), n * 4);
        if (final_obs_host) memcpy(final_obs_host, s.h_final.get(), n * D * 4);
        if (truncated_host) memcpy(truncated_host, s.h_trunc.get(), n);
    }
    return MGB_OK;
}

extern "C" int mgb_quad_step_host(mgb_quad *h, const float *act_host, float *obs_host, float *rew_host,
                                  uint8_t *done_host, int32_t *fail_host, float *final_obs_host, void *stream)
{
    MgbRange nvtx_range("mgb_quad_step_host");
    return step_host(h, act_host, obs_host, rew_host, done_host, fail_host, final_obs_host, nullptr, stream);
}

extern "C" int mgb_quad_step_host_ex(mgb_quad *h, const float *act_host, float *obs_host, float *rew_host,
                                     uint8_t *done_host, int32_t *fail_host, float *final_obs_host,
                                     uint8_t *truncated_host, void *stream)
{
    MgbRange nvtx_range("mgb_quad_step_host_ex");
    return step_host(h, act_host, obs_host, rew_host, done_host, fail_host, final_obs_host, truncated_host, stream);
}

extern "C" int mgb_quad_state(mgb_quad *h, float *state_dev, int32_t *ct_dev, int load, void *stream)
{
    MgbRange nvtx_range("mgb_quad_state");
    MGB_REQUIRE(h && state_dev, "null argument");
    MgbDeviceGuard guard(h->device);
    QuadArgs a = base_args(h);
    quad_state_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, state_dev, ct_dev, load);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Snapshot / restore records (DESIGN.md "Snapshot, restore and clone"): the six state planes of an env as they are in
// HBM, then (velocity task, 0, 0, 0).  One thread per env, 16-byte loads and stores on both sides.
// ---------------------------------------------------------------------------------------------------------------
namespace {

constexpr int kRecordQuads = kPlanes + 1;     // uint4 per record

__global__ void quad_snapshot_kernel(QuadArgs a, uint4 *__restrict__ rec)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    QState s;
    load_state(a, e, s);
    float4 q[kPlanes];
    pack_state(s, q);
    uint4 *r = rec + e * kRecordQuads;
#pragma unroll
    for (int k = 0; k < kPlanes; ++k) r[k] = make_uint4(__float_as_uint(q[k].x), __float_as_uint(q[k].y),
                                                       __float_as_uint(q[k].z), __float_as_uint(q[k].w));
    r[kPlanes] = make_uint4(a.env2task ? (uint32_t)a.env2task[e] : 0u, 0u, 0u, 0u);
}

// env2task gets a kernel of its own, launched before quad_restore_kernel: the step kernels read env2task before their
// griddepcontrol.wait, so the kernel right before a step must not write it
__global__ void quad_restore_task_kernel(int64_t n, int32_t *__restrict__ env2task, int n_tasks, const uint4 *__restrict__ rec,
                                         int64_t n_rec, const int64_t *__restrict__ row)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    const int64_t r = row[e];
    if (r < 0 || r >= n_rec) return;
    const int t = (int)rec[r * kRecordQuads + kPlanes].x;
    if (t >= 0 && t < n_tasks) env2task[e] = t;
}

__global__ void quad_restore_kernel(QuadArgs a, const uint4 *__restrict__ rec, int64_t n_rec, const int64_t *__restrict__ row)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= a.n) return;
    const int64_t r = row[e];
    if (r < 0 || r >= n_rec) return;
    const uint4 *src = rec + r * kRecordQuads;
    float4 q[kPlanes];
#pragma unroll
    for (int k = 0; k < kPlanes; ++k) {
        const uint4 u = src[k];
        q[k] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
    }
    QState s;
    unpack_state(q, s);
    store_state(a, e, s);
}

}  // namespace

extern "C" int64_t mgb_quad_record_bytes(const mgb_quad *h) { return h ? (int64_t)kRecordQuads * 16 : MGB_ERR_ARG; }

extern "C" int mgb_quad_snapshot(mgb_quad *h, uint8_t *rec_dev, void *stream)
{
    MgbRange nvtx_range("mgb_quad_snapshot");
    MGB_REQUIRE(h && rec_dev, "null argument");
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(rec_dev) & 15u) == 0, "rec_dev must be 16-byte aligned");
    MgbDeviceGuard guard(h->device);
    QuadArgs a = base_args(h);
    quad_snapshot_kernel<<<(unsigned)((h->n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(a, reinterpret_cast<uint4 *>(rec_dev));
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

extern "C" int mgb_quad_restore(mgb_quad *h, const uint8_t *rec_dev, int64_t n_rec, const int64_t *row_of_env_dev,
                                void *stream)
{
    MgbRange nvtx_range("mgb_quad_restore");
    MGB_REQUIRE(h && rec_dev && row_of_env_dev, "null argument");
    MGB_REQUIRE(n_rec >= 0, "n_rec must not be negative");
    MGB_REQUIRE((reinterpret_cast<uintptr_t>(rec_dev) & 15u) == 0, "rec_dev must be 16-byte aligned");
    int rc = check_ready(h);
    if (rc) return rc;
    MgbDeviceGuard guard(h->device);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)((h->n + 255) / 256);
    const uint4 *rec = reinterpret_cast<const uint4 *>(rec_dev);
    if (h->env2task) {
        quad_restore_task_kernel<<<blocks, 256, 0, st>>>(h->n, h->env2task.get(), h->n_tasks, rec, n_rec, row_of_env_dev);
        MGB_CUDA(cudaGetLastError());
        h->launches += 1;
    }
    QuadArgs a = base_args(h);
    quad_restore_kernel<<<blocks, 256, 0, st>>>(a, rec, n_rec, row_of_env_dev);
    MGB_CUDA(cudaGetLastError());
    h->launches += 1;
    return MGB_OK;
}

extern "C" int mgb_quad_counters(mgb_quad *h, uint64_t *t_base, int set)
{
    MGB_REQUIRE(h && t_base, "null argument");
    if (set) h->t_base = (uint32_t)*t_base;
    else *t_base = h->t_base;
    return MGB_OK;
}

extern "C" int mgb_quad_fingerprint(const mgb_quad *h, uint64_t *out)
{
    MGB_REQUIRE(h && out, "null argument");
    const int64_t rec_bytes = (int64_t)kRecordQuads * 16;
    uint64_t f = mgb_fnv(MGB_FNV_BASIS, &h->cfg, sizeof(h->cfg));
    f = mgb_fnv(f, &h->auto_reset, sizeof(h->auto_reset));
    f = mgb_fnv(f, &h->seed, sizeof(h->seed));
    out[0] = mgb_fnv(f, &rec_bytes, sizeof(rec_bytes));
    out[1] = h->fp_map;
    out[2] = h->fp_targets;
    out[3] = 0;
    return MGB_OK;
}
