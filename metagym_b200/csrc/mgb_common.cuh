// Shared helpers of libmgb200: error reporting, counter-based RNG, bulk (TMA) copies.  sm_90a.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include <nvtx3/nvToolsExt.h>      // header-only; a no-op unless a profiler (nsys / ncu --nvtx) is attached

#include "mgb200.h"

void mgb_set_error(const char *fmt, ...);

// NVTX range over one C-ABI call (SURVEY.md section 5, tracing): shows the host-side extent of every entry point on a
// profiler timeline.  Costs a few nanoseconds when nothing is attached.
struct MgbRange {
    explicit MgbRange(const char *name) { nvtxRangePushA(name); }
    ~MgbRange() { nvtxRangePop(); }
};

#define MGB_CUDA(call)                                                                                   \
    do {                                                                                                 \
        cudaError_t e__ = (call);                                                                        \
        if (e__ != cudaSuccess) {                                                                        \
            mgb_set_error("%s -> %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__);      \
            return MGB_ERR_CUDA;                                                                         \
        }                                                                                                \
    } while (0)

#define MGB_REQUIRE(cond, msg)                                                                           \
    do {                                                                                                 \
        if (!(cond)) {                                                                                   \
            mgb_set_error("%s: %s", __func__, msg);                                                      \
            return MGB_ERR_ARG;                                                                          \
        }                                                                                                \
    } while (0)

// FNV-1a over bytes, chained through h (start from MGB_FNV_BASIS): the host-side fingerprints of mgb_*_fingerprint
#define MGB_FNV_BASIS 0xcbf29ce484222325ull
static inline uint64_t mgb_fnv(uint64_t h, const void *p, size_t bytes)
{
    const unsigned char *b = static_cast<const unsigned char *>(p);
    for (size_t i = 0; i < bytes; ++i) h = (h ^ b[i]) * 0x100000001b3ull;
    return h;
}

// RAII "make this device current for the duration of the call"
struct MgbDeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit MgbDeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
        want = dev;
    }
    ~MgbDeviceGuard() {
        if (prev >= 0 && prev != want) cudaSetDevice(prev);
    }
    int want = -1;
};

// Owner of one buffer from Mem::alloc (device memory: MgbDev, pinned host memory: MgbPinned).  Handles keep every buffer
// in one of these, so an error exit, a replaced buffer or a destroyed handle frees it exactly once.  A buffer is freed
// when it is reset, assigned over or destroyed, which must happen with the buffer's device current: the entry points'
// MgbDeviceGuard.
struct MgbDeviceMem {
    static cudaError_t alloc(void **p, size_t bytes) { return cudaMalloc(p, bytes); }
    static void free(void *p) { cudaFree(p); }
};
struct MgbPinnedMem {
    static cudaError_t alloc(void **p, size_t bytes) { return cudaMallocHost(p, bytes); }
    static void free(void *p) { cudaFreeHost(p); }
};
template <typename T, class Mem> class MgbBuf {
  public:
    MgbBuf() = default;
    MgbBuf(const MgbBuf &) = delete;
    MgbBuf &operator=(const MgbBuf &) = delete;
    MgbBuf(MgbBuf &&o) noexcept : p_(o.release()) {}
    MgbBuf &operator=(MgbBuf &&o) noexcept
    {
        if (this != &o) {
            reset();
            p_ = o.release();
        }
        return *this;
    }
    ~MgbBuf() { reset(); }

    T *get() const { return p_; }
    explicit operator bool() const { return p_ != nullptr; }
    // frees the buffer held, then allocates `bytes`; on an error the owner holds nothing
    cudaError_t alloc(size_t bytes)
    {
        reset();
        void *p = nullptr;
        const cudaError_t e = Mem::alloc(&p, bytes);
        if (e == cudaSuccess) p_ = static_cast<T *>(p);
        return e;
    }
    void reset()
    {
        if (p_) Mem::free(p_);
        p_ = nullptr;
    }
    T *release()
    {
        T *p = p_;
        p_ = nullptr;
        return p;
    }

  private:
    T *p_ = nullptr;
};
template <typename T> using MgbDev = MgbBuf<T, MgbDeviceMem>;
template <typename T> using MgbPinned = MgbBuf<T, MgbPinnedMem>;

// Owner of one cudaEvent_t, destroyed like an MgbBuf is freed
class MgbEvent {
  public:
    MgbEvent() = default;
    MgbEvent(const MgbEvent &) = delete;
    MgbEvent &operator=(const MgbEvent &) = delete;
    ~MgbEvent()
    {
        if (e_) cudaEventDestroy(e_);
    }

    cudaEvent_t get() const { return e_; }
    explicit operator bool() const { return e_ != nullptr; }
    cudaError_t create(unsigned flags)
    {
        if (e_) cudaEventDestroy(e_);
        e_ = nullptr;
        return cudaEventCreateWithFlags(&e_, flags);
    }

  private:
    cudaEvent_t e_ = nullptr;
};

// ---------------------------------------------------------------------------------------------------------------
// Philox4x32-10 (Salmon et al., SC'11): counter-based, so every env owns a stream keyed by its GLOBAL index and the
// results do not depend on how envs are sharded over GPUs or blocks.
// ---------------------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t mgb_mulhi32(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
    return __umulhi(a, b);
#else
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}

__host__ __device__ __forceinline__ uint4 mgb_philox4x32_10(uint4 ctr, uint2 key)
{
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint32_t hi0 = mgb_mulhi32(M0, ctr.x), lo0 = M0 * ctr.x;
        uint32_t hi1 = mgb_mulhi32(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0;
        key.y += W1;
    }
    return ctr;
}

// 24-bit uniform in [0, 1)
__host__ __device__ __forceinline__ float mgb_u01(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }

// RNG stream ids (ctr.w)
#define MGB_STREAM_RESET 0x100u   // + j, j = 0..2: twelve reset draws
#define MGB_STREAM_ACTION 0x200u  // rollout actions
#define MGB_STREAM_POLICY 0x400u  // draws of policy-driven rollouts (mgb_policy.cuh)
#define MGB_STREAM_EXPERT 0x800u  // draws of the maze expert (maze.cu, expert_action)

// ---------------------------------------------------------------------------------------------------------------
// Bulk asynchronous copies (the TMA engine's 1-D form: cp.async.bulk, SASS UBLKCP)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t mgb_smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// generic-proxy writes to smem -> visible to the async proxy (must precede a bulk store reading that smem)
__device__ __forceinline__ void mgb_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// smem -> global, bytes % 16 == 0, both 16 B aligned.  Issued by ONE thread.
__device__ __forceinline__ void mgb_bulk_store(void *gdst, const void *ssrc, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(mgb_smem_addr(ssrc)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mgb_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the smem SOURCE of all but the newest n groups has been read (smem reusable)
template <int N> __device__ __forceinline__ void mgb_bulk_wait_read()
{
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N> __device__ __forceinline__ void mgb_bulk_wait()
{
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// Output mirrors: a rollout kernel can store every trajectory output a second, third, ... time at `pointer + delta[i]`.
// With the outputs placed in this rank's slot of a receive arena and delta[i] = (peer i's arena base - local arena base)
// over NVLink peer mappings (mgb_peer_open), the kernel itself performs the all-gather of the trajectory chunk:
// the remote stores drain through NVLink/NVSwitch while the next env-step integrates.
// ---------------------------------------------------------------------------------------------------------------
struct MgbMirrors {
    int count;                        // > 0: peer mirrors; MGB_MIRROR_MULTICAST: delta[0] = multicast base - local base
#define MGB_MIRROR_MULTICAST (-1)
    int64_t delta[MGB_MAX_MIRRORS];   // bytes

    // The bodies of mgb_*_set_mirrors and mgb_*_set_multicast: the refusal, or nullptr once *this holds the new
    // mirrors (left unchanged on a refusal).  The callers refuse in their own name.
    const char *set_peers(int n, const int64_t *byte_delta)
    {
        if (!(n >= 0 && n <= MGB_MAX_MIRRORS && (n == 0 || byte_delta))) return "count out of range";
        MgbMirrors m = {};
        for (int i = 0; i < n; ++i) {
            if ((byte_delta[i] & 15) != 0) return "mirror deltas must be multiples of 16 bytes";
            m.delta[i] = byte_delta[i];
        }
        m.count = n;
        *this = m;
        return nullptr;
    }
    const char *set_multicast(int64_t byte_delta)
    {
        if ((byte_delta & 15) != 0) return "multicast delta must be a multiple of 16 bytes";
        MgbMirrors m = {};
        if (byte_delta != 0) { m.count = MGB_MIRROR_MULTICAST; m.delta[0] = byte_delta; }
        *this = m;
        return nullptr;
    }
};
struct MgbMirrorWindow {             // host side: where mirrored outputs must lie (0 bytes = unchecked)
    uintptr_t base = 0;
    uint64_t bytes = 0;
    void set(const void *p, uint64_t len)
    {
        base = reinterpret_cast<uintptr_t>(p);
        bytes = len;
    }
    // the whole extent [p, p + len) must lie inside the window: a rollout with a larger T or N than the arena slot was
    // laid out for would otherwise store `ptr + delta` past the peer's slot
    bool holds(const void *p, uint64_t len) const
    {
        const uintptr_t q = reinterpret_cast<uintptr_t>(p);
        return p == nullptr || bytes == 0 || (q >= base && len <= bytes && q - base <= bytes - len);
    }
    // every output of a rollout of `env_steps` = T x n env-steps: observations, rewards, done flags and recorded
    // actions of obs_bytes / rew_bytes / 1 / act_bytes bytes per env-step
    bool holds_rollout(uint64_t env_steps, const void *obs, uint64_t obs_bytes, const void *rew, uint64_t rew_bytes,
                       const void *done, const void *act, uint64_t act_bytes) const
    {
        return holds(obs, env_steps * obs_bytes) && holds(rew, env_steps * rew_bytes) && holds(done, env_steps) &&
               holds(act, env_steps * act_bytes);
    }
};
template <typename T> __device__ __forceinline__ void mgb_mirror_store(const MgbMirrors &m, T *p, const T v)
{
    for (int i = 0; i < m.count; ++i) *reinterpret_cast<T *>(reinterpret_cast<char *>(p) + m.delta[i]) = v;
}
// issued by ONE thread, before mgb_bulk_commit(): the same smem tile to every mirror of gdst
__device__ __forceinline__ void mgb_mirror_bulk_store(const MgbMirrors &m, void *gdst, const void *ssrc, uint32_t bytes)
{
    for (int i = 0; i < m.count; ++i) mgb_bulk_store(reinterpret_cast<char *>(gdst) + m.delta[i], ssrc, bytes);
}

// ---------------------------------------------------------------------------------------------------------------
// NVSwitch multicast stores (NVLS): ONE store to a multicast address is replicated by the switch into the bound memory of
// every GPU of the group, so an all-gather costs each GPU its own bytes once instead of (world-1) times.  The address
// must come from a multicast mapping (cuMulticast*; torch's symmetric memory does that plumbing) and may only be touched
// with multimem.* instructions.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mgb_mc_st(float *p, float v) { asm volatile("multimem.st.weak.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }
__device__ __forceinline__ void mgb_mc_st(double *p, double v) { asm volatile("multimem.st.weak.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory"); }
__device__ __forceinline__ void mgb_mc_st(uint32_t *p, uint32_t v) { asm volatile("multimem.st.weak.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void mgb_mc_st(int32_t *p, int32_t v) { asm volatile("multimem.st.weak.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void mgb_mc_st(float4 *p, float4 v)
{
    asm volatile("multimem.st.weak.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
template <typename T> __device__ __forceinline__ T *mgb_shift(T *p, int64_t bytes)
{
    return reinterpret_cast<T *>(reinterpret_cast<char *>(p) + bytes);
}
// whole-CTA copy of a shared-memory tile to a multicast address (call after __syncthreads())
__device__ __forceinline__ void mgb_mc_copy_tile(float *mc_dst, const float *tile, uint32_t bytes)
{
    if ((bytes & 15u) == 0 && ((reinterpret_cast<uintptr_t>(mc_dst) & 15u) == 0)) {
        const float4 *src = reinterpret_cast<const float4 *>(tile);
        float4 *dst = reinterpret_cast<float4 *>(mc_dst);
        for (uint32_t i = threadIdx.x; i < bytes / 16u; i += blockDim.x) mgb_mc_st(dst + i, src[i]);
    } else {
        for (uint32_t i = threadIdx.x; i < bytes / 4u; i += blockDim.x) mgb_mc_st(mc_dst + i, tile[i]);
    }
}
// one byte per lane -> 32-bit multicast stores by every fourth lane (all 32 lanes must call; idx % 4 == lane % 4)
__device__ __forceinline__ void mgb_mc_st_bytes(uint8_t *mc_p, uint32_t byte, bool valid)
{
    const uint32_t b1 = __shfl_down_sync(0xffffffffu, byte, 1), b2 = __shfl_down_sync(0xffffffffu, byte, 2),
                   b3 = __shfl_down_sync(0xffffffffu, byte, 3);
    if (valid && (threadIdx.x & 3) == 0)
        mgb_mc_st(reinterpret_cast<uint32_t *>(mc_p), byte | (b1 << 8) | (b2 << 16) | (b3 << 24));
}

// mbarrier + global -> smem bulk load
__device__ __forceinline__ void mgb_mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mgb_smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mgb_fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mgb_mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mgb_smem_addr(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mgb_mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(mgb_smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mgb_bulk_load(void *sdst, const void *gsrc, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     mgb_smem_addr(sdst)),
                 "l"(gsrc), "r"(bytes), "r"(mgb_smem_addr(bar))
                 : "memory");
}
__device__ __forceinline__ void mgb_mbar_wait(uint64_t *bar, uint32_t phase)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(mgb_smem_addr(bar)),
        "r"(phase)
        : "memory");
}
