// What do the velocity-target gathers of one quadrotor step cost at 65 536 envs, 64 tasks, nt = 1000 (env e flies task
// e % 64)?  Each env reads the rows ct-1 and min(ct, nt-1) of its task.  A launch here does only that: read env2task,
// gather the two rows, write one float per env.  Layouts:
//   task-major [n_tasks][nt][3] float32 : six 4-byte loads per env, a warp's 32 lanes hit 32 tasks 12 000 B apart
//   time-major [nt][n_tasks] float4     : two 16-byte loads per env, lanes at one ct read 512 contiguous bytes
// with every env at the same ct (what an auto-reset batch started together does) and with a random ct per env.
// "floor" is the same launch without the row loads.  64-thread CTAs as in quad_step_kernel, graph of 256 launches,
// programmatic dependent launch between them.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o targetgather.bin targetgather.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

struct Args {
    const float *tbl3;        // [n_tasks][nt][3]
    const float4 *tbl4;       // [nt][n_tasks]
    const int32_t *env2task;  // [n]
    const int32_t *ct_env;    // [n] per-env step counter in [0, nt), or null: every env at ct_all
    int ct_all, nt, n_tasks, n;
    float *out;               // [n]
};

// LAYOUT: 0 = no row loads (floor), 1 = task-major float32, 2 = time-major float4
template <int LAYOUT> __global__ void __launch_bounds__(64) gather_kernel(const __grid_constant__ Args a)
{
    asm volatile("griddepcontrol.launch_dependents;");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int e = blockIdx.x * 64 + threadIdx.x;
    if (e >= a.n) return;
    const int task = __ldg(a.env2task + e);
    const int ct = (a.ct_env ? __ldg(a.ct_env + e) : a.ct_all) + 1;          // 1..nt, as after the step's ct += 1
    const int t = ct < a.nt - 1 ? ct : a.nt - 1;
    float s = (float)task;
    if (LAYOUT == 1) {
        const float *row = a.tbl3 + (int64_t)task * a.nt * 3;
        const float *g = row + 3 * (ct - 1), *q = row + 3 * t;
        s += __ldg(g) + __ldg(g + 1) + __ldg(g + 2) + __ldg(q) + __ldg(q + 1) + __ldg(q + 2);
    } else if (LAYOUT == 2) {
        const float4 g = __ldg(a.tbl4 + (int64_t)(ct - 1) * a.n_tasks + task);
        const float4 q = __ldg(a.tbl4 + (int64_t)t * a.n_tasks + task);
        s += g.x + g.y + g.z + q.x + q.y + q.z;
    }
    a.out[e] = s;
}

template <typename F> static float time_graph(cudaStream_t st, int nodes, int replays, F launch)
{
    cudaGraph_t g; cudaGraphExec_t ge;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeGlobal));
    for (int i = 0; i < nodes; ++i) launch(i);
    CK(cudaStreamEndCapture(st, &g));
    CK(cudaGraphInstantiate(&ge, g, 0));
    for (int i = 0; i < 3; ++i) CK(cudaGraphLaunch(ge, st));
    CK(cudaStreamSynchronize(st));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0, st));
    for (int i = 0; i < replays; ++i) CK(cudaGraphLaunch(ge, st));
    CK(cudaEventRecord(e1, st));
    CK(cudaStreamSynchronize(st));
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
    return ms * 1e3f / (nodes * replays);
}

template <typename K> static void launch_pdl(K kern, int grid, cudaStream_t st, const Args &a)
{
    cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(64); cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    CK(cudaLaunchKernelEx(&cfg, kern, a));
}

int main()
{
    const int n = 65536, n_tasks = 64, nt = 1000, reps = 7;
    std::vector<float> h3((size_t)n_tasks * nt * 3);
    std::vector<float> h4((size_t)nt * n_tasks * 4, 0.f);
    for (int k = 0; k < n_tasks; ++k)
        for (int t = 0; t < nt; ++t)
            for (int j = 0; j < 3; ++j) {
                const float v = (float)(k * 1000003 + t * 7 + j) * 1e-6f;
                h3[((size_t)k * nt + t) * 3 + j] = v;
                h4[((size_t)t * n_tasks + k) * 4 + j] = v;
            }
    std::vector<int32_t> e2t(n), ctr(n);
    uint32_t x = 12345u;
    for (int e = 0; e < n; ++e) {
        e2t[e] = e % n_tasks;
        x = x * 1664525u + 1013904223u;
        ctr[e] = (int)((x >> 8) % (uint32_t)nt);
    }
    float *d3, *out; float4 *d4; int32_t *de2t, *dct;
    CK(cudaMalloc(&d3, h3.size() * 4)); CK(cudaMalloc(&d4, h4.size() * 4));
    CK(cudaMalloc(&de2t, n * 4)); CK(cudaMalloc(&dct, n * 4)); CK(cudaMalloc(&out, n * 4));
    CK(cudaMemcpy(d3, h3.data(), h3.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d4, h4.data(), h4.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(de2t, e2t.data(), n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dct, ctr.data(), n * 4, cudaMemcpyHostToDevice));
    cudaStream_t st; CK(cudaStreamCreate(&st));
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    const int grid = (n + 63) / 64;

    // both layouts must gather the same values
    std::vector<float> o1(n), o2(n);
    for (int mode = 0; mode < 2; ++mode) {
        Args a = {d3, d4, de2t, mode ? dct : nullptr, 417, nt, n_tasks, n, out};
        launch_pdl(gather_kernel<1>, grid, st, a);
        CK(cudaStreamSynchronize(st));
        CK(cudaMemcpy(o1.data(), out, n * 4, cudaMemcpyDeviceToHost));
        launch_pdl(gather_kernel<2>, grid, st, a);
        CK(cudaStreamSynchronize(st));
        CK(cudaMemcpy(o2.data(), out, n * 4, cudaMemcpyDeviceToHost));
        if (memcmp(o1.data(), o2.data(), n * 4) != 0) { printf("layouts disagree (mode %d)\n", mode); return 1; }
    }

    printf("%s, %d SMs; %d envs, %d tasks, nt %d, 64-thread CTAs, PDL, graphs of 256 launches;\n", prop.name,
           prop.multiProcessorCount, n, n_tasks, nt);
    printf("us per launch, median of %d graph replays (min-max)\n", reps);
    const char *names[3] = {"floor (env2task only)", "task-major f32 x6", "time-major float4 x2"};
    for (int mode = 0; mode < 2; ++mode) {
        printf("%s\n", mode ? "random ct per env:" : "every env at the same ct (ct advances every launch):");
        float med[3];
        for (int layout = 0; layout < 3; ++layout) {
            std::vector<float> v;
            for (int r = 0; r < reps; ++r)
                v.push_back(time_graph(st, 256, 20, [&](int i) {
                    const Args a = {d3, d4, de2t, mode ? dct : nullptr, i % nt, nt, n_tasks, n, out};
                    if (layout == 0) launch_pdl(gather_kernel<0>, grid, st, a);
                    else if (layout == 1) launch_pdl(gather_kernel<1>, grid, st, a);
                    else launch_pdl(gather_kernel<2>, grid, st, a);
                }));
            std::vector<float> s = v;
            for (size_t i = 0; i < s.size(); ++i)
                for (size_t j = i + 1; j < s.size(); ++j)
                    if (s[j] < s[i]) { float tmp = s[i]; s[i] = s[j]; s[j] = tmp; }
            med[layout] = s[s.size() / 2];
            printf("  %-24s %.3f  (%.3f-%.3f)", names[layout], med[layout], s.front(), s.back());
            if (layout > 0) printf("   gathers over the floor: %.3f", med[layout] - med[0]);
            printf("\n");
        }
    }
    CK(cudaGetLastError());
    cudaFree(d3); cudaFree(d4); cudaFree(de2t); cudaFree(dct); cudaFree(out);
    return 0;
}
