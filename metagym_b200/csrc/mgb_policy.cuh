// MLP policies evaluated inside a rollout launch (mgb_quad_rollout_policy, mgb_maze_rollout_policy; DESIGN.md
// "Policy-driven rollouts"), and the recurrent policies of mgb_maze_rollout_rnn and mgb_quad_rollout_rnn below.
//
// One thread owns one env.  The CTA stages the packed weights (mgb_policy.params_dev, torch.nn.Linear order) into shared
// memory once per launch, regrouped so that a hidden layer's outputs are computed eight at a time: for output group g
// and input i the eight weights W[8g .. 8g+7][i] are two consecutive float4, read by the whole warp as a broadcast, and
// the thread's input x[i] is one conflict-free load from its own column of the activation buffers ([k][blockDim.x]).
// The output layer (4 wide, or 5 with a value head: row 4 is the critic's V) is staged in groups of four, so 5 rows pad
// to 8.  Rows past a layer's width are zero.  Every output is a fused multiply-add chain that starts at the bias and runs
// over the inputs in index order, in float32, so rows 0..3 do not depend on whether row 4 exists.
#pragma once
#include <type_traits>
#include "mgb_common.cuh"

constexpr int kPolicyMaxLayers = MGB_POLICY_MAX_HIDDEN + 1;

// Launch-time plan of one policy: layer shapes and where each layer lives in the packed buffer and in shared memory.
struct MgbMlp {
    const float *params;          // packed buffer (global memory)
    int n_layers;                 // n_hidden + 1
    int in[kPolicyMaxLayers], out[kPolicyMaxLayers];
    int gw[kPolicyMaxLayers];     // global float offset of W of layer l (b follows at gw + out * in)
    int sw[kPolicyMaxLayers];     // shared float offset of the regrouped W of layer l
    int sb[kPolicyMaxLayers];     // shared float offset of the bias of layer l (padded to the group width)
    int g_log_std, s_log_std;     // log_std [4] (Gaussian policies), -1 if none
    int staged;                   // floats of staged weights (a multiple of 8)
    int maxw;                     // rows of each activation buffer: max(input width, hidden widths)
    int smem_off;                 // float offset of the policy's region in the kernel's dynamic shared memory
    int activation, mode;
    uint64_t seed;
    float *logp_out;              // [T][n] or null
    float *obs0_out;              // [n][in[0]] or null
    // populations (DESIGN.md "Populations"); a plan's head holds them for the whole policy, as it does seed and mode
    int packed;                   // floats of one packed buffer that the plan reads
    int copies;                   // members staged per CTA: CTA envs / member_envs when that is above 1, else 1
    int64_t member_envs;          // envs per member: member m drives the envs [m E, (m + 1) E); INT64_MAX: one policy
    int64_t member_stride;        // floats from one member's packed buffer to the next
    int member_shift;             // the warp's staged copy is threadIdx.x >> member_shift (31: the only one)
};

// Host: validate `p` and plan it for input width `in_dim` (output width 4; `log_std`: the buffer ends with log_std[4],
// the Gaussian head of the quadrotor; without it the four outputs are the logits of the maze's categorical head;
// `value`: the output layer has a fifth row, the value head of the critic entry points).
// Returns null, or the reason the policy is refused.
static inline const char *mgb_mlp_plan(const mgb_policy *p, int in_dim, bool log_std, MgbMlp &m, bool value = false)
{
    if (!p) return "null policy";
    if (!p->params_dev) return "null params_dev";
    if (p->n_hidden < 0 || p->n_hidden > MGB_POLICY_MAX_HIDDEN) return "n_hidden must be 0..3";
    for (int k = 0; k < p->n_hidden; ++k)
        if (p->width[k] < 1 || p->width[k] > MGB_POLICY_MAX_WIDTH) return "hidden widths must be 1..64";
    if (p->activation != MGB_ACT_TANH && p->activation != MGB_ACT_RELU) return "unknown activation";
    if (p->mode != MGB_POLICY_SAMPLE && p->mode != MGB_POLICY_MEAN) return "unknown policy mode";
    m = MgbMlp{};
    m.params = p->params_dev;
    m.n_layers = p->n_hidden + 1;
    m.activation = p->activation;
    m.mode = p->mode;
    int g = 0, s = 0, maxw = in_dim;
    for (int l = 0; l < m.n_layers; ++l) {
        const bool last = l == m.n_layers - 1;
        m.in[l] = l == 0 ? in_dim : p->width[l - 1];
        m.out[l] = last ? (value ? 5 : 4) : p->width[l];
        if (!last && m.out[l] > maxw) maxw = m.out[l];
        const int gwid = last ? 4 : 8, rows = (m.out[l] + gwid - 1) / gwid * gwid;
        m.gw[l] = g;
        g += m.out[l] * (m.in[l] + 1);
        m.sw[l] = s;
        s += rows * m.in[l];
        m.sb[l] = s;
        s += rows;
        s = (s + 7) / 8 * 8;
    }
    m.g_log_std = m.s_log_std = -1;
    if (log_std) {
        m.g_log_std = g;
        m.s_log_std = s;
        s += 8;
    }
    m.staged = s;
    m.maxw = maxw;
    m.packed = g + (log_std ? 4 : 0);
    m.copies = 1;
    m.member_envs = INT64_MAX;
    m.member_shift = 31;
    return nullptr;
}

// bytes of dynamic shared memory a CTA of `threads` needs: staged weights of m.copies members + two activation buffers
static inline size_t mgb_mlp_smem_bytes(const MgbMlp &m, int threads)
{
    return ((size_t)m.staged * (size_t)m.copies + 2 * (size_t)m.maxw * (size_t)threads) * sizeof(float);
}

// Device: stage the weights of `m` read at m.params + off into sm[0, m.staged) (all threads of the CTA; the caller
// synchronises)
__device__ __forceinline__ void mgb_mlp_stage(const MgbMlp &m, float *sm, int64_t off)
{
    for (int l = 0; l < m.n_layers; ++l) {
        const bool last = l == m.n_layers - 1;
        const int gwid = last ? 4 : 8, in = m.in[l], out = m.out[l];
        const int rows = (out + gwid - 1) / gwid * gwid;
        const float *W = m.params + off + m.gw[l], *b = W + out * in;
        for (int s = threadIdx.x; s < rows * in; s += blockDim.x) {
            const int r = s % gwid, rest = s / gwid, i = rest % in, j = (rest / in) * gwid + r;
            sm[m.sw[l] + s] = j < out ? __ldg(W + j * in + i) : 0.f;
        }
        for (int j = threadIdx.x; j < rows; j += blockDim.x) sm[m.sb[l] + j] = j < out ? __ldg(b + j) : 0.f;
    }
    if (m.s_log_std >= 0 && threadIdx.x < 4)
        sm[m.s_log_std + threadIdx.x] = __ldg(m.params + off + m.g_log_std + threadIdx.x);
}

__device__ __forceinline__ float mgb_mlp_activate(int activation, float x)
{
    return activation == MGB_ACT_TANH ? tanhf(x) : (x > 0.f ? x : 0.f);
}

// Device: forward pass of the thread's env.  Its input x[i] is a0[i * stride + col], i < m.in[0]; a0 and a1 are the
// two activation buffers (each m.maxw rows of `stride` floats), both clobbered.  out4 receives the four outputs, and
// with VAL (a plan of 5 outputs) *value receives the fifth, the first row of the output layer's second group.
template <bool VAL = false>
__device__ __forceinline__ void mgb_mlp_forward(const MgbMlp &m, const float *sm, float *a0, float *a1, int stride,
                                                int col, float out4[4], float *value = nullptr)
{
    const float *x = a0 + col;
    float *y = a1 + col;
    for (int l = 0; l < m.n_layers - 1; ++l) {
        const int in = m.in[l], out = m.out[l];
        const float4 *W = reinterpret_cast<const float4 *>(sm + m.sw[l]);
        const float4 *B = reinterpret_cast<const float4 *>(sm + m.sb[l]);
        for (int g = 0; g < out; g += 8) {
            const float4 b0 = B[g / 4], b1 = B[g / 4 + 1];
            float acc[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
            const float4 *w = W + (g / 8) * in * 2;
#pragma unroll 4
            for (int i = 0; i < in; ++i) {
                const float xi = x[i * stride];
                const float4 w0 = w[2 * i], w1 = w[2 * i + 1];
                acc[0] = fmaf(w0.x, xi, acc[0]); acc[1] = fmaf(w0.y, xi, acc[1]);
                acc[2] = fmaf(w0.z, xi, acc[2]); acc[3] = fmaf(w0.w, xi, acc[3]);
                acc[4] = fmaf(w1.x, xi, acc[4]); acc[5] = fmaf(w1.y, xi, acc[5]);
                acc[6] = fmaf(w1.z, xi, acc[6]); acc[7] = fmaf(w1.w, xi, acc[7]);
            }
#pragma unroll
            for (int r = 0; r < 8; ++r)
                if (g + r < out) y[(g + r) * stride] = mgb_mlp_activate(m.activation, acc[r]);
        }
        const float *t = x;
        x = y;
        y = const_cast<float *>(t);
    }
    const int l = m.n_layers - 1, in = m.in[l];
    const float4 *W = reinterpret_cast<const float4 *>(sm + m.sw[l]);
    const float4 b = *reinterpret_cast<const float4 *>(sm + m.sb[l]);
    float acc[4] = {b.x, b.y, b.z, b.w};
    float accv = 0.f;
    if constexpr (VAL) accv = sm[m.sb[l] + 4];
#pragma unroll 4
    for (int i = 0; i < in; ++i) {
        const float xi = x[i * stride];
        const float4 w = W[i];
        acc[0] = fmaf(w.x, xi, acc[0]); acc[1] = fmaf(w.y, xi, acc[1]);
        acc[2] = fmaf(w.z, xi, acc[2]); acc[3] = fmaf(w.w, xi, acc[3]);
        if constexpr (VAL) accv = fmaf(sm[m.sw[l] + 4 * (in + i)], xi, accv);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) out4[k] = acc[k];
    if constexpr (VAL) *value = accv;
}

// Device: Gaussian action of env genv at step counter t from the policy mean (MGB_POLICY_SAMPLE), or the mean itself
// (MGB_POLICY_MEAN).  Returns log pi(a | obs) for the sampling mode (0 for the mean mode).
__device__ __forceinline__ float mgb_gaussian_action(const MgbMlp &m, const float *sm, int64_t genv, uint32_t t,
                                                     const float mean[4], float a[4])
{
    if (m.mode == MGB_POLICY_MEAN) {
#pragma unroll
        for (int k = 0; k < 4; ++k) a[k] = mean[k];
        return 0.f;
    }
    const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32), t, MGB_STREAM_POLICY),
                                      make_uint2((uint32_t)m.seed, (uint32_t)(m.seed >> 32)));
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
    float z[4];
#pragma unroll
    for (int p = 0; p < 2; ++p) {
        const float u1 = (float)((w[2 * p] >> 8) + 1u) * (1.0f / 16777216.0f);      // (0, 1]: log is finite
        const float u2 = mgb_u01(w[2 * p + 1]);
        const float rad = sqrtf(-2.f * logf(u1));
        float sn, cs;
        sincospif(2.f * u2, &sn, &cs);
        z[2 * p] = rad * cs;
        z[2 * p + 1] = rad * sn;
    }
    float logp = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float ls = sm[m.s_log_std + k];
        a[k] = fmaf(expf(ls), z[k], mean[k]);
        logp += -0.5f * z[k] * z[k] - ls;
    }
    return logp - 3.6757541328186907f;     // 2 log(2 pi)
}

// Device: categorical action over the four logits l (MetaMaze2D).  MGB_POLICY_SAMPLE: inverse CDF of the float32 softmax,
// u = (x >> 8) 2^-24 of the first Philox word, the probabilities accumulated in index order; the action is the first k
// with u < c_k, else 3.  MGB_POLICY_MEAN: the argmax, ties to the lowest index.  Returns l_a - logsumexp(l) for the
// sampling mode (0 for the mean mode).
__device__ __forceinline__ float mgb_categorical_action(const MgbMlp &m, int64_t genv, uint32_t t, const float l[4],
                                                        int &action)
{
    float mx = l[0];
    int am = 0;
#pragma unroll
    for (int k = 1; k < 4; ++k)
        if (l[k] > mx) { mx = l[k]; am = k; }
    if (m.mode == MGB_POLICY_MEAN) {
        action = am;
        return 0.f;
    }
    float ex[4], sum = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        ex[k] = expf(l[k] - mx);
        sum += ex[k];
    }
    const uint4 r = mgb_philox4x32_10(make_uint4((uint32_t)genv, (uint32_t)((uint64_t)genv >> 32), t, MGB_STREAM_POLICY),
                                      make_uint2((uint32_t)m.seed, (uint32_t)(m.seed >> 32)));
    const float u = mgb_u01(r.x);
    float cdf = 0.f;
    action = 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        cdf += ex[k] / sum;
        if (u < cdf) { action = k; break; }
    }
    float la = l[0];
#pragma unroll
    for (int k = 1; k < 4; ++k)
        if (action == k) la = l[k];
    return (la - mx) - logf(sum);
}

// ---------------------------------------------------------------------------------------------------------------
// Recurrent policies (mgb_maze_rollout_rnn; DESIGN.md "Recurrent policies"): a cell of NG gates, the GRU (NG = 3, gates
// r, z, n) or the LSTM (NG = 4, gates i, f, g, o), then a head.  The cell's weights are staged in groups of kRnnGroup
// hidden units: for group g and input i the NG kRnnGroup weights W[k H + kRnnGroup g + r][i] (gate k, r < kRnnGroup)
// are consecutive float4, read by the warp as broadcasts, for weight_ih over x and then weight_hh over the previous h.
// Group g's biases are bias_ih [NG][kRnnGroup], then bias_hh [NG][kRnnGroup].  Units past H are zero.  The head is an
// MgbMlp on h, staged behind the cell.
//
// Per env the policy keeps the columns x [in], c [C], h0 [Hr], h1 [Hr], w [Hw] (rows of the CTA's env count floats):
// the input, the LSTM's cell state (C = H; the GRU has none, C = 0), the previous and the new h, which swap roles every
// step, and the head's hidden layer.  The GRU has Hr = H and Hw = its head width; the LSTM writes its head's hidden
// layer into the dead previous-h column instead, so Hr = max(H, head width) and Hw = 0.  The carried state row is
// [h (H), c (C), feedback (5 feedback)].
// ---------------------------------------------------------------------------------------------------------------

constexpr int kRnnGroup = 8;      // hidden units per pass over the inputs

template <int NG>
struct MgbRnn {
    static_assert(NG == 3 || NG == 4, "the GRU has three gates, the LSTM four");
    const float *params;          // packed buffer (global memory)
    int H, Hp, in, feedback, reset;   // Hp: H rounded up to kRnnGroup
    int Hr;                       // rows of each h column
    int g_hh, g_b;                // global float offsets of weight_hh and bias_ih (weight_ih at 0, bias_hh at g_b + NG H)
    int s_hh, s_b, s_head;        // shared float offsets of the regrouped weight_hh, the biases and the head
    int staged;                   // floats of staged weights, cell and head (a multiple of 8)
    int smem_off;                 // float offset of the policy's region in the kernel's dynamic shared memory
    int Hw;                       // rows of the w column
    MgbMlp head;                  // the head (in[0] = H); its seed, mode, logp_out and obs0_out serve the whole policy
    float *state, *state0_out, *hid_out;  // [n][H + C + 5 feedback], the same or null, [T][n][H] or null

    __host__ __device__ int C() const { return NG == 4 ? H : 0; }             // rows of the c column
    __host__ __device__ int HC() const { return NG == 4 ? 2 * H : H; }        // H + C: floats of h and c in a state row
};

// The policy kinds of the rollout kernels: none (0, open-loop), an MLP, a GRU or an LSTM, and the plan type of each
constexpr int kPolMlp = 1, kPolGru = 2, kPolLstm = 3;

template <int POL>
using MgbPolicyPlan = std::conditional_t<POL == kPolLstm, MgbRnn<4>, std::conditional_t<POL == kPolGru, MgbRnn<3>, MgbMlp>>;

// The plan of the action head: an MLP policy's own, or a recurrent policy's head
template <class Plan>
__host__ __device__ __forceinline__ auto &mgb_policy_head(Plan &p)
{
    if constexpr (std::is_same_v<std::remove_const_t<Plan>, MgbMlp>) return p;
    else return p.head;
}

// Host: the checks every recurrent cell shares.  Returns null, or the reason the policy is refused.
static inline const char *mgb_rnn_check(const mgb_rnn_policy *p)
{
    if (!p) return "null policy";
    if (!p->params_dev) return "null params_dev";
    if (p->hidden < 1 || p->hidden > MGB_RNN_MAX_HIDDEN) return "hidden must be 1..64";
    if (p->feedback != 0 && p->feedback != 1) return "feedback must be 0 or 1";
    if (p->reset != MGB_RNN_RESET_EPISODE && p->reset != MGB_RNN_RESET_TASK) return "unknown reset rule";
    if (p->head_hidden != 0 && p->head_hidden != 1) return "head_hidden must be 0 or 1";
    if (p->head_hidden && (p->head_width < 1 || p->head_width > MGB_POLICY_MAX_WIDTH)) return "head_width must be 1..64";
    if (p->cell != MGB_RNN_CELL_GRU && p->cell != MGB_RNN_CELL_LSTM) return "unknown cell";
    return nullptr;
}

// Host: validate `p` and plan it for observation width `obs_dim` (`value`: the head's output layer has the value row;
// `log_std`: the buffer ends with log_std [4], the quadrotor's Gaussian head).  Returns null, or the reason the policy
// is refused.
template <int NG>
static inline const char *mgb_rnn_plan(const mgb_rnn_policy *p, int obs_dim, MgbRnn<NG> &r, bool value = false,
                                       bool log_std = false)
{
    if (const char *why = mgb_rnn_check(p)) return why;
    r = MgbRnn<NG>{};
    r.params = p->params_dev;
    r.H = p->hidden;
    r.Hp = (r.H + kRnnGroup - 1) / kRnnGroup * kRnnGroup;
    r.in = obs_dim + 5 * p->feedback;
    r.feedback = p->feedback;
    r.reset = p->reset;
    const int head_width = p->head_hidden ? p->head_width : 0;
    r.Hr = NG == 4 && head_width > r.H ? head_width : r.H;
    r.Hw = NG == 4 ? 0 : head_width;
    r.g_hh = NG * r.H * r.in;
    r.g_b = r.g_hh + NG * r.H * r.H;
    r.s_hh = NG * r.Hp * r.in;
    r.s_b = r.s_hh + NG * r.Hp * r.H;
    r.s_head = r.s_b + 2 * NG * r.Hp;
    const mgb_policy hp = {p->params_dev + r.g_b + 2 * NG * r.H, p->head_hidden, {p->head_width, 0, 0}, p->activation,
                           p->mode};
    if (const char *why = mgb_mlp_plan(&hp, r.H, log_std, r.head, value)) return why;
    r.staged = r.s_head + r.head.staged;
    r.head.packed += r.g_b + 2 * NG * r.H;
    return nullptr;
}

// bytes of dynamic shared memory a CTA of `threads` needs: staged weights of head.copies members + the columns x, c,
// h0, h1 and w
template <int NG>
static inline size_t mgb_rnn_smem_bytes(const MgbRnn<NG> &r, int threads)
{
    return ((size_t)r.staged * (size_t)r.head.copies + (size_t)(r.in + r.C() + 2 * r.Hr + r.Hw) * (size_t)threads) *
           sizeof(float);
}

// Device: stage the cell and the head read at r.params + off into sm[0, r.staged) (all threads of the CTA; the caller
// synchronises).  HEAD = false stages the cell alone, into sm[0, r.s_head): the sequence kernels of rnn_seq.cu, whose
// packed buffer ends with bias_hh.
template <int NG, bool HEAD = true>
__device__ __forceinline__ void mgb_rnn_stage(const MgbRnn<NG> &r, float *sm, int64_t off)
{
    constexpr int G = kRnnGroup;
    const int H = r.H;
    for (int part = 0; part < 2; ++part) {
        const int K = part ? H : r.in;
        const float *W = r.params + off + (part ? r.g_hh : 0);
        float *dst = sm + (part ? r.s_hh : 0);
        for (int s = threadIdx.x; s < NG * r.Hp * K; s += blockDim.x) {
            const int u = s % G, k = (s / G) % NG, i = (s / (NG * G)) % K, j = (s / (NG * G * K)) * G + u;
            dst[s] = j < H ? __ldg(W + (k * H + j) * K + i) : 0.f;
        }
    }
    for (int s = threadIdx.x; s < 2 * NG * r.Hp; s += blockDim.x) {
        const int u = s % G, k = (s / G) % NG, kind = (s / (NG * G)) % 2, j = (s / (2 * NG * G)) * G + u;
        sm[r.s_b + s] = j < H ? __ldg(r.params + off + r.g_b + kind * NG * H + k * H + j) : 0.f;
    }
    if constexpr (HEAD) mgb_mlp_stage(r.head, sm + r.s_head, off);
}

// ---------------------------------------------------------------------------------------------------------------
// Populations (DESIGN.md "Populations"): `members` packed policies of one plan, `member_stride` floats apart; with
// E = n / members, member m drives the envs [m E, (m + 1) E) of the handle.  E is a multiple of a warp's 32 envs and
// either divides the CTA's env count or is a multiple of it.  A CTA whose envs belong to one member stages it once;
// a CTA of CTA / E members stages them back to back, `staged` floats apart, and every warp reads its own member.
// ---------------------------------------------------------------------------------------------------------------

// Host: spread the population over the n envs of a handle whose policy CTA holds `cta` envs, into the plan's head.
// Returns null, or the reason the population is refused.  One member reads no stride and leaves the plan as it is.
static inline const char *mgb_population_plan(MgbMlp &head, int64_t n, int32_t members, int64_t member_stride, int cta)
{
    if (members < 1) return "members must be at least 1";
    if (n % members != 0) return "num_envs must be a multiple of members";
    if (members == 1) return nullptr;
    const int64_t E = n / members;
    if (E % MGB_POLICY_MEMBER_WARP != 0 || (E < cta ? cta % E : E % cta) != 0)
        return "envs per member (num_envs / members) must be a multiple of 32 that divides the policy CTA's envs or is a "
               "multiple of them (MGB_QUAD_POLICY_CTA_ENVS, MGB_QUAD_RNN_CTA_ENVS, MGB_MAZE2D_POLICY_CTA_ENVS)";
    if (member_stride < head.packed) return "member_stride is shorter than one member's packed policy";
    head.member_envs = E;
    head.member_stride = member_stride;
    head.copies = E < cta ? (int)(cta / E) : 1;
    if (E < cta) head.member_shift = E == 32 ? 5 : 6;        // E divides a CTA of 64 or 128: 32 or 64
    return nullptr;
}

// Device: stage the members that drive the CTA's envs [e0, e0 + rows) into sm, `staged` floats apart (all threads of
// the CTA; the caller synchronises).  One policy (member_stride 0) stages from the buffer's start.
template <class Plan>
__device__ __forceinline__ void mgb_population_stage(const Plan &p, float *sm, int64_t e0, int rows, int cta)
{
    const MgbMlp &head = mgb_policy_head(p);
    const int64_t E = head.member_envs, m0 = head.member_stride ? e0 / E : 0;
    const int here = E < cta ? (int)((rows + E - 1) / E) : 1;      // a partial last CTA holds fewer members
    for (int j = 0; j < here; ++j) {
        if constexpr (std::is_same_v<Plan, MgbMlp>) mgb_mlp_stage(p, sm + j * p.staged, (m0 + j) * head.member_stride);
        else mgb_rnn_stage(p, sm + j * p.staged, (m0 + j) * head.member_stride);
    }
}

// Device: f(w) with w the staged copy the thread's warp reads, of the copies mgb_population_stage left at sm.  With one
// copy per CTA (one policy, or a member per CTA or more) w is sm itself, and the compiler keeps the weight addresses in
// uniform registers; it cannot for the warp's copy (threadIdx.x >> member_shift), and a single-policy MetaMaze2D MLP
// rollout through that address alone measured 6.5 % slower.  So f is compiled for both.  The empty asm ends the two
// arms differently, so that the compiler does not sink their common code below the branch and make w one per-thread
// value again.
template <class F>
__device__ __forceinline__ void mgb_population_weights(const MgbMlp &head, const float *sm, int staged, F &&f)
{
    if (head.copies == 1) {
        f(sm);
    } else {
        f(sm + ((int)threadIdx.x >> head.member_shift) * staged);
        asm volatile("");
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Value heads and GAE (DESIGN.md "Value heads and GAE", header "value heads and GAE")
// ---------------------------------------------------------------------------------------------------------------

// Host: the checks of a critic (header "value heads and GAE") that the entry point's own checks do not make.  Returns
// null, or the reason the call is refused.
static inline const char *mgb_critic_check(const mgb_critic *cr, bool auto_reset, const void *rew, const void *done,
                                           const void *truncated)
{
    if (!cr) return "null critic";
    if (!auto_reset) return "a critic needs auto_reset on (the value of a finished env's next state is a new episode's)";
    if (!cr->value_dev) return "null value_dev";
    if (!cr->adv_dev != !cr->ret_dev) return "adv_dev and ret_dev go together";
    if (cr->adv_dev && !(rew && done && truncated && cr->final_value_dev))
        return "adv / ret need rew, done, truncated and final_value";
    if (!(cr->gamma >= 0.f && cr->gamma <= 1.f)) return "gamma must be finite and in [0, 1]";
    if (!(cr->lambda >= 0.f && cr->lambda <= 1.f)) return "lambda must be finite and in [0, 1]";
    return nullptr;
}

// Device: GAE(gamma, lambda) of the thread's env e, walking its column backwards from v_last = V(s_T).  It reads back
// only what the thread itself stored in this launch with ordinary stores (rew, done, truncated, value, final_value, and
// with cut_in_adv the cut flags the loop left in adv), so no fence is needed.  Every operation is rounded to nearest
// with no contraction, so that a float32 NumPy restatement is bit exact.
template <class R>
__device__ __forceinline__ void mgb_gae(const mgb_critic &cr, int T, int64_t n, int64_t e, float v_last, const R *rew,
                                        const uint8_t *done, const uint8_t *truncated, bool cut_in_adv)
{
    const float gamma = cr.gamma, gl = __fmul_rn(cr.gamma, cr.lambda);
    float nv_next = v_last, A = 0.f;
    for (int t = T - 1; t >= 0; --t) {
        const int64_t i = (int64_t)t * n + e;
        const float v = cr.value_dev[i];
        const bool cut = cut_in_adv ? cr.adv_dev[i] != 0.f : done[i] != 0;
        const float nv = cut ? (truncated[i] ? cr.final_value_dev[i] : 0.f) : nv_next;
        float r;
        if constexpr (std::is_same_v<R, double>) r = __double2float_rn(rew[i]);
        else r = rew[i];
        const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(gamma, nv)), v);
        A = __fadd_rn(delta, cut ? 0.f : __fmul_rn(gl, A));
        cr.adv_dev[i] = A;
        if (cr.ret_dev) cr.ret_dev[i] = __fadd_rn(A, v);
        nv_next = v;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Whole-episode evaluation (mgb_quad_evaluate, mgb_maze_evaluate; DESIGN.md "Whole-episode evaluation").  The EVAL
// instantiations of the policy rollout kernels take this in place of the critic: each env steps until its
// `episodes`-th done and stores one entry per episode, at the done that ends it.
// ---------------------------------------------------------------------------------------------------------------

struct MgbEval {
    double *ret;          // [episodes][n]: the float64 sum of the episode's rewards, in step order
    int32_t *len;         // [episodes][n]: its steps
    uint8_t *trunc;       // [episodes][n]: the rollout's truncated flag at the done that ended it
    int episodes;
};

// The last kernel parameter of a policy rollout: the critic, or with EVAL the evaluation's outputs
template <bool EVAL>
using MgbCriticOrEval = std::conditional_t<EVAL, MgbEval, mgb_critic>;

// Host: the checks an evaluation makes besides the rollout's; `limit` is the time limit in steps.  Returns null, or
// the reason the call is refused, and sets T to the step bound episodes * limit.
static inline const char *mgb_eval_check(int32_t episodes, int64_t limit, bool auto_reset, const void *mlp,
                                         const void *rnn, const float *state, int32_t value_row, const void *ret,
                                         const void *len, const void *trunc, int32_t &T)
{
    if (!auto_reset) return "evaluation needs auto_reset on (an env steps on into its next episode)";
    if (episodes < 1) return "episodes must be at least 1";
    if ((int64_t)episodes * limit > INT32_MAX) return "episodes * the time limit must be at most 2^31 - 1 steps";
    if (!mlp == !rnn) return "exactly one of mlp and rnn must be set";
    if (rnn && !state) return "null state (a recurrent policy carries its state)";
    if (mlp && state) return "state goes with a recurrent policy";
    if (value_row != 0 && value_row != 1) return "value_row must be 0 or 1";
    if (!ret || !len || !trunc) return "null output";
    T = (int32_t)((int64_t)episodes * limit);
    return nullptr;
}

// Device: one step's reward into the thread's episode.  At a done it stores the episode and starts the next; returns
// false once the env has finished its last episode.
__device__ __forceinline__ bool mgb_eval_step(const MgbEval &ev, int64_t n, int64_t e, double reward, bool done,
                                              bool truncated, double &ret, int &len, int &ep)
{
    ret += reward;
    len += 1;
    if (!done) return true;
    const int64_t i = (int64_t)ep * n + e;
    ev.ret[i] = ret;
    ev.len[i] = len;
    ev.trunc[i] = truncated ? 1 : 0;
    ret = 0.0;
    len = 0;
    return ++ep < ev.episodes;
}

__device__ __forceinline__ float mgb_sigmoid(float v) { return 1.f / (1.f + expf(-v)); }

// What mgb_rnn_cell hands its `save` for unit j: nothing by default (the rollouts)
struct MgbRnnNoSave {
    template <class... V>
    __device__ __forceinline__ void operator()(int, V...) const {}
};

// Device: one step of the cell for the thread's env (header "Recurrent policies" for the arithmetic): h = GRU(x, hp),
// or (h, c) = LSTM(x, (hp, c)) with c updated in place (unit j reads and writes only c[j]; the GRU ignores c).  x, hp,
// c and h are column buffers (rows of `stride` floats; the thread's column is `col`); h must not alias x, hp or c.
// save(j, ...) receives unit j's values the backward pass of mgb_rnn_seq_backward needs: the GRU's r, z, n and
// W_hn hp + b_hn, the LSTM's i, f, g, o and c'.
template <int NG, class Save = MgbRnnNoSave>
__device__ __forceinline__ void mgb_rnn_cell(const MgbRnn<NG> &r, const float *sm, const float *xb, const float *hpb,
                                             float *cb, float *hb, int stride, int col, Save save = {})
{
    constexpr int G = kRnnGroup, Q = NG * G / 4;     // Q: float4 weights per input of a group
    const float *x = xb + col, *hp = hpb + col;
    float *c = cb + col, *h = hb + col;
    const int in = r.in, H = r.H;
    const float4 *B = reinterpret_cast<const float4 *>(sm + r.s_b);
    for (int u = 0; u < H; u += G) {
        const int grp = u / G;
        float gi[NG * G], gh[NG * G];
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const float4 bi = B[grp * (2 * Q) + q], bh = B[grp * (2 * Q) + Q + q];
            gi[4 * q] = bi.x; gi[4 * q + 1] = bi.y; gi[4 * q + 2] = bi.z; gi[4 * q + 3] = bi.w;
            gh[4 * q] = bh.x; gh[4 * q + 1] = bh.y; gh[4 * q + 2] = bh.z; gh[4 * q + 3] = bh.w;
        }
        const float4 *w = reinterpret_cast<const float4 *>(sm) + grp * in * Q;
#pragma unroll 2
        for (int i = 0; i < in; ++i) {
            const float xi = x[i * stride];
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                const float4 wq = w[Q * i + q];
                gi[4 * q] = fmaf(wq.x, xi, gi[4 * q]); gi[4 * q + 1] = fmaf(wq.y, xi, gi[4 * q + 1]);
                gi[4 * q + 2] = fmaf(wq.z, xi, gi[4 * q + 2]); gi[4 * q + 3] = fmaf(wq.w, xi, gi[4 * q + 3]);
            }
        }
        w = reinterpret_cast<const float4 *>(sm + r.s_hh) + grp * H * Q;
#pragma unroll 2
        for (int i = 0; i < H; ++i) {
            const float hi = hp[i * stride];
#pragma unroll
            for (int q = 0; q < Q; ++q) {
                const float4 wq = w[Q * i + q];
                gh[4 * q] = fmaf(wq.x, hi, gh[4 * q]); gh[4 * q + 1] = fmaf(wq.y, hi, gh[4 * q + 1]);
                gh[4 * q + 2] = fmaf(wq.z, hi, gh[4 * q + 2]); gh[4 * q + 3] = fmaf(wq.w, hi, gh[4 * q + 3]);
            }
        }
#pragma unroll
        for (int v = 0; v < G; ++v)
            if (u + v < H) {
                if constexpr (NG == 3) {
                    const float rg = mgb_sigmoid(gi[v] + gh[v]);
                    const float zg = mgb_sigmoid(gi[G + v] + gh[G + v]);
                    const float ng = tanhf(fmaf(rg, gh[2 * G + v], gi[2 * G + v]));
                    h[(u + v) * stride] = fmaf(zg, hp[(u + v) * stride], (1.f - zg) * ng);
                    save(u + v, rg, zg, ng, gh[2 * G + v]);
                } else {
                    const float ig = mgb_sigmoid(gi[v] + gh[v]);
                    const float fg = mgb_sigmoid(gi[G + v] + gh[G + v]);
                    const float gg = tanhf(gi[2 * G + v] + gh[2 * G + v]);
                    const float og = mgb_sigmoid(gi[3 * G + v] + gh[3 * G + v]);
                    const float cn = fmaf(fg, c[(u + v) * stride], ig * gg);
                    c[(u + v) * stride] = cn;
                    h[(u + v) * stride] = og * tanhf(cn);
                    save(u + v, ig, fg, gg, og, cn);
                }
            }
    }
}
