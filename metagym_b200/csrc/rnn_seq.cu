// Recurrent cell sequences (mgb_rnn_seq_forward, mgb_rnn_seq_backward; DESIGN.md "Fused unroll"): the GRU or LSTM cell of
// the recurrent rollouts run over T given steps, forward and backward, for the learner's backpropagation through time.
//
// One thread owns one env and walks its steps in order, as in the rollout.  The forward stages the cell as the rollout
// does (mgb_rnn_stage without the head) and runs the rollout's own mgb_rnn_cell on shared columns x [in], c [C], and h
// twice (previous and new), so h_t is the rollout's bit for bit; the cell hands the gates to a saver that writes them
// env-minor.  The backward walks t = T-1 .. 0 with the carried dh (and the LSTM's dc) in shared columns, computes unit
// j's gate gradients from the saved gates and feeds each of them to all H accumulators of W_hh^T dG through warp-uniform
// float4 broadcasts of weight_hh row k H + j, staged row-major with HA (16, 32 or 64) floats per row.  dL/dh_t and, for
// the GRU, h_{t-1} arrive [n][H] env-major; the CTA reads its block of them coalesced into its columns.
#include <algorithm>

#include "mgb_policy.cuh"

namespace {

constexpr int kSeqCta = MGB_RNN_SEQ_CTA_ENVS;

// saved values per unit: the GRU's r, z, n, W_hn h + b_hn; the LSTM's i, f, g, o, c
template <int NG>
constexpr int kSeqSaved = NG == 3 ? 4 : 5;

// mgb_rnn_cell's saver: value s of unit j at g[s block + j n] (g: the step's gates + e, block = H n)
struct SeqSave {
    float *g;
    int64_t n, block;
    template <class... V>
    __device__ __forceinline__ void operator()(int j, V... v) const
    {
        const float vals[] = {v...};
#pragma unroll
        for (int s = 0; s < (int)sizeof...(V); ++s) g[s * block + (int64_t)j * n] = vals[s];
    }
};

template <int NG, bool SAVE>
__global__ void __launch_bounds__(kSeqCta, 1) rnn_seq_forward_kernel(const MgbRnn<NG> r, const mgb_rnn_seq a)
{
    constexpr int B = kSeqCta;
    extern __shared__ float4 smem4[];
    float *sm = reinterpret_cast<float *>(smem4);
    const int H = r.H, in = r.in, tid = threadIdx.x;
    float *xc = sm + r.s_head, *cc = xc + in * B, *hp = cc + r.C() * B, *hn = hp + H * B;
    const int64_t n = a.n, e0 = (int64_t)blockIdx.x * B, e = e0 + tid;
    const int rows = (int)min((int64_t)B, n - e0);
    const bool live = tid < rows;
    mgb_rnn_stage<NG, false>(r, sm, 0);
    if (live)
        for (int j = 0; j < r.HC(); ++j) {
            const float v = a.state0_dev[e * r.HC() + j];
            if (j < H) hp[j * B + tid] = v;
            else cc[(j - H) * B + tid] = v;
        }
    __syncthreads();
    const int64_t block = (int64_t)H * n;
    for (int t = 0; t < a.T; ++t) {
        if (live) {
            if (t > 0 && a.wipe_dev[(int64_t)(t - 1) * n + e])
                for (int j = 0; j < H; ++j) {
                    hp[j * B + tid] = 0.f;
                    if constexpr (NG == 4) cc[j * B + tid] = 0.f;
                }
            const float *x = a.x_dev + (int64_t)t * in * n + e;
            for (int i = 0; i < in; ++i) xc[i * B + tid] = x[(int64_t)i * n];
            if constexpr (SAVE)
                mgb_rnn_cell(r, sm, xc, hp, cc, hn, B, tid,
                             SeqSave{a.gates_dev + (int64_t)t * kSeqSaved<NG> * block + e, n, block});
            else
                mgb_rnn_cell(r, sm, xc, hp, cc, hn, B, tid);
        }
        __syncthreads();
        float *ho = a.h_dev + ((int64_t)t * n + e0) * H;
        for (int s = tid; s < rows * H; s += B) ho[s] = hn[(s % H) * B + s / H];
        __syncthreads();         // the next step may zero hn's columns (now hp)
        float *tmp = hp;
        hp = hn;
        hn = tmp;
    }
}

template <int NG, int HA>
__global__ void __launch_bounds__(kSeqCta, 1) rnn_seq_backward_kernel(const MgbRnn<NG> r, const mgb_rnn_seq a)
{
    constexpr int B = kSeqCta, S = kSeqSaved<NG>, Q = HA / 4;
    extern __shared__ float4 smem4[];
    float *sm = reinterpret_cast<float *>(smem4);
    const int H = r.H, HC = r.HC(), tid = threadIdx.x;
    float *dhc = sm + NG * H * HA;        // dL/dh_t, then the gradient carried to h_{t-1}
    float *aux = dhc + H * B;             // GRU: h_{t-1}; LSTM: the carried dc
    const int64_t n = a.n, e0 = (int64_t)blockIdx.x * B, e = e0 + tid, block = (int64_t)H * n;
    const int rows = (int)min((int64_t)B, n - e0);
    const bool live = tid < rows;
    const float *Whh = r.params + r.g_hh;
    for (int s = tid; s < NG * H * HA; s += B) {
        const int row = s / HA, i = s % HA;
        sm[s] = i < H ? __ldg(Whh + row * H + i) : 0.f;
    }
    for (int j = 0; j < H; ++j) {
        dhc[j * B + tid] = 0.f;
        aux[j * B + tid] = 0.f;
    }
    const float4 *W4 = reinterpret_cast<const float4 *>(sm);
    for (int t = a.T - 1; t >= 0; --t) {
        __syncthreads();
        const float *dh = a.dh_dev + ((int64_t)t * n + e0) * H;
        for (int s = tid; s < rows * H; s += B) dhc[(s % H) * B + s / H] += dh[s];
        if constexpr (NG == 3) {
            if (t > 0) {
                const float *hprev = a.h_dev + ((int64_t)(t - 1) * n + e0) * H;
                const uint8_t *wp = a.wipe_dev + (int64_t)(t - 1) * n + e0;
                for (int s = tid; s < rows * H; s += B) aux[(s % H) * B + s / H] = wp[s / H] ? 0.f : hprev[s];
            } else {
                for (int s = tid; s < rows * H; s += B) aux[(s % H) * B + s / H] = a.state0_dev[e0 * H + s];
            }
        }
        __syncthreads();
        if (!live) continue;
        const bool wiped = t > 0 && a.wipe_dev[(int64_t)(t - 1) * n + e];
        const float *G = a.gates_dev + (int64_t)t * S * block + e;
        float *dgi = a.dgi_dev + (int64_t)t * NG * block + e;
        float acc[HA];
#pragma unroll
        for (int i = 0; i < HA; ++i) acc[i] = 0.f;
        for (int j = 0; j < H; ++j) {
            const int64_t o = (int64_t)j * n;
            const float dhj = dhc[j * B + tid];
            float d[NG];       // dL/d(W_hh h + b_hh) of unit j, gate by gate
            if constexpr (NG == 3) {
                const float rg = G[o], zg = G[block + o], ng = G[2 * block + o], hn = G[3 * block + o];
                const float dnp = dhj * (1.f - zg) * (1.f - ng * ng);
                const float dzp = dhj * (aux[j * B + tid] - ng) * zg * (1.f - zg);
                const float drp = dnp * hn * rg * (1.f - rg);
                dgi[o] = drp;
                dgi[block + o] = dzp;
                dgi[2 * block + o] = dnp;
                d[0] = drp;
                d[1] = dzp;
                d[2] = dnp * rg;
                a.dghn_dev[(int64_t)t * block + e + o] = d[2];
                dhc[j * B + tid] = dhj * zg;
            } else {
                const float ig = G[o], fg = G[block + o], gg = G[2 * block + o], og = G[3 * block + o];
                const float cn = G[4 * block + o];
                const float cp = t == 0 ? a.state0_dev[e * HC + H + j]
                                 : wiped ? 0.f
                                         : G[4 * block + o - (int64_t)S * block];
                const float tc = tanhf(cn);
                const float dc = aux[j * B + tid] + dhj * og * (1.f - tc * tc);
                d[0] = dc * gg * ig * (1.f - ig);
                d[1] = dc * cp * fg * (1.f - fg);
                d[2] = dc * ig * (1.f - gg * gg);
                d[3] = dhj * tc * og * (1.f - og);
#pragma unroll
                for (int k = 0; k < 4; ++k) dgi[k * block + o] = d[k];
                aux[j * B + tid] = dc * fg;
                dhc[j * B + tid] = 0.f;
            }
#pragma unroll
            for (int k = 0; k < NG; ++k) {
                const float4 *w = W4 + (k * H + j) * Q;
#pragma unroll
                for (int q = 0; q < Q; ++q) {
                    const float4 wq = w[q];
                    acc[4 * q] = fmaf(wq.x, d[k], acc[4 * q]);
                    acc[4 * q + 1] = fmaf(wq.y, d[k], acc[4 * q + 1]);
                    acc[4 * q + 2] = fmaf(wq.z, d[k], acc[4 * q + 2]);
                    acc[4 * q + 3] = fmaf(wq.w, d[k], acc[4 * q + 3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < HA; ++i)
            if (i < H) {
                const float v = dhc[i * B + tid] + acc[i];
                if (t == 0) {
                    a.dstate0_dev[e * HC + i] = v;
                    if constexpr (NG == 4) a.dstate0_dev[e * HC + H + i] = aux[i * B + tid];
                } else {
                    dhc[i * B + tid] = wiped ? 0.f : v;
                    if constexpr (NG == 4)
                        if (wiped) aux[i * B + tid] = 0.f;
                }
            }
    }
}

// Host: the plan of the cell alone (no head, no feedback: x is the whole input), or the reason the call is refused
template <int NG>
const char *seq_plan(const mgb_rnn_seq *a, MgbRnn<NG> &r)
{
    const mgb_rnn_policy p = {a->params_dev, a->hidden, 0, MGB_RNN_RESET_EPISODE, 0, 0, MGB_ACT_TANH,
                              MGB_POLICY_SAMPLE, a->cell};
    return mgb_rnn_plan<NG>(&p, a->in, r);
}

const char *seq_check(const mgb_rnn_seq *a, bool backward)
{
    if (!a) return "null seq";
    if (a->cell != MGB_RNN_CELL_GRU && a->cell != MGB_RNN_CELL_LSTM) return "unknown cell";
    if (a->hidden < 1 || a->hidden > MGB_RNN_MAX_HIDDEN) return "hidden must be 1..64";
    if (a->in < 1) return "in must be at least 1";
    if (a->T < 1) return "T must be at least 1";
    if (a->n < 1) return "n must be at least 1";
    if (!a->params_dev || !a->wipe_dev || !a->state0_dev) return "null params_dev, wipe_dev or state0_dev";
    if (!backward) return a->x_dev && a->h_dev ? nullptr : "null x_dev or h_dev";
    if (!a->gates_dev || !a->dh_dev || !a->dgi_dev || !a->dstate0_dev)
        return "null gates_dev, dh_dev, dgi_dev or dstate0_dev";
    if (a->cell == MGB_RNN_CELL_GRU && (!a->h_dev || !a->dghn_dev)) return "the GRU needs h_dev and dghn_dev";
    return nullptr;
}

// Host: refuse (as fn) a kernel footprint beyond the current device's opt-in shared memory, else allow it
int seq_fits(const char *fn, const void *kernel, size_t sm, const char *what)
{
    int dev = 0, optin = 0;
    MGB_CUDA(cudaGetDevice(&dev));
    MGB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    if (sm > (size_t)optin) {
        mgb_set_error("%s: the %s needs %zu bytes of shared memory per CTA of %d envs, more than the %d the device "
                      "allows", fn, what, sm, kSeqCta, optin);
        return MGB_ERR_ARG;
    }
    MGB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    return MGB_OK;
}

unsigned seq_blocks(int64_t n) { return (unsigned)((n + kSeqCta - 1) / kSeqCta); }

template <int NG>
int seq_forward(const mgb_rnn_seq *a, cudaStream_t st)
{
    MgbRnn<NG> r;
    if (const char *why = seq_plan(a, r)) {
        mgb_set_error("mgb_rnn_seq_forward: %s", why);
        return MGB_ERR_ARG;
    }
    const size_t sm = ((size_t)r.s_head + (size_t)(r.in + r.C() + 2 * r.H) * kSeqCta) * sizeof(float);
    const auto kernel = a->gates_dev ? rnn_seq_forward_kernel<NG, true> : rnn_seq_forward_kernel<NG, false>;
    if (int rc = seq_fits("mgb_rnn_seq_forward", (const void *)kernel, sm, "forward (cell weights, columns x, c, h)"))
        return rc;
    kernel<<<seq_blocks(a->n), kSeqCta, sm, st>>>(r, *a);
    MGB_CUDA(cudaGetLastError());
    return MGB_OK;
}

template <int NG, int HA>
int seq_backward_ha(const mgb_rnn_seq *a, const MgbRnn<NG> &r, cudaStream_t st)
{
    const size_t sm = ((size_t)NG * r.H * HA + 2 * (size_t)r.H * kSeqCta) * sizeof(float);
    const auto kernel = rnn_seq_backward_kernel<NG, HA>;
    if (int rc = seq_fits("mgb_rnn_seq_backward", (const void *)kernel, sm, "backward (weight_hh, two columns)"))
        return rc;
    kernel<<<seq_blocks(a->n), kSeqCta, sm, st>>>(r, *a);
    MGB_CUDA(cudaGetLastError());
    return MGB_OK;
}

template <int NG>
int seq_backward(const mgb_rnn_seq *a, cudaStream_t st)
{
    MgbRnn<NG> r;
    if (const char *why = seq_plan(a, r)) {
        mgb_set_error("mgb_rnn_seq_backward: %s", why);
        return MGB_ERR_ARG;
    }
    return r.H <= 16 ? seq_backward_ha<NG, 16>(a, r, st)
         : r.H <= 32 ? seq_backward_ha<NG, 32>(a, r, st)
                     : seq_backward_ha<NG, 64>(a, r, st);
}

}  // namespace

extern "C" int mgb_rnn_seq_forward(const mgb_rnn_seq *seq, void *stream)
{
    MgbRange range(__func__);
    if (const char *why = seq_check(seq, false)) {
        mgb_set_error("%s: %s", __func__, why);
        return MGB_ERR_ARG;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    return seq->cell == MGB_RNN_CELL_GRU ? seq_forward<3>(seq, st) : seq_forward<4>(seq, st);
}

extern "C" int mgb_rnn_seq_backward(const mgb_rnn_seq *seq, void *stream)
{
    MgbRange range(__func__);
    if (const char *why = seq_check(seq, true)) {
        mgb_set_error("%s: %s", __func__, why);
        return MGB_ERR_ARG;
    }
    const cudaStream_t st = (cudaStream_t)stream;
    return seq->cell == MGB_RNN_CELL_GRU ? seq_backward<3>(seq, st) : seq_backward<4>(seq, st);
}
