/* One-off micro-benchmark: what the PCG kernel's grid-wide synchronisation
 * costs by itself (no SpMV, no vector update), for variants of the barrier
 * and of the re-summation of the per-CTA partial sums. `barrier 1 sums 1` is
 * what cg_kernel uses; the `per-CTA flags` variants (one flag per CTA instead
 * of one counter, polled by every CTA) were measured slower and not kept.
 *   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o barrier_probe barrier_probe.cu
 *   ./barrier_probe            (2 CTAs per SM x 256 threads, cooperative)
 */
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CHECK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { \
    fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

constexpr int THREADS = 256, WARPS = THREADS / 32, MAXB = 1024;

template <int B>
__device__ __forceinline__ void
grid_barrier (unsigned int* counter, unsigned int& epoch)
{
    __syncthreads();
    if (threadIdx.x == 0)
    {
        epoch += 1;
        unsigned int const target = epoch * gridDim.x;
        if (B == 0 || B == 2)
        {
            __threadfence();
            atomicAdd(counter, 1u);
        }
        else
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;"
                :: "l"(counter) : "memory");
        unsigned int v;
        do {
            asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];"
                : "=r"(v) : "l"(counter) : "memory");
        } while (v < target);
        if (B == 0)
            __threadfence();
        else
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];"
                : "=r"(v) : "l"(counter) : "memory");
    }
    __syncthreads();
}

template <int S, int NV>
__device__ __forceinline__ void
all_sums (double const* partials, int first_slot, double* s_bcast)
{
    __syncthreads();
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int const nb = gridDim.x;
    for (int j = warp; j < NV; j += WARPS)
    {
        double const* p = partials + (first_slot + j) * MAXB;
        double v = 0.0;
        constexpr int U = (S == 0) ? 8 : 12;
        for (int base = lane; base < nb; base += 32 * U)
        {
            double t[U];
#pragma unroll
            for (int u = 0; u < U; ++u)
                t[u] = (base + 32 * u < nb) ? __ldcg(p + base + 32 * u) : 0.0;
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (base + 32 * u < nb)
                    v += t[u];
        }
        for (int off = 16; off > 0; off >>= 1)
            v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0)
            s_bcast[j] = v;
    }
    __syncthreads();
}

template <int B, int S>
__global__ void __launch_bounds__(THREADS, 2)
probe (unsigned int* counter, double* partials, double* vec, int iters,
    double* out)
{
    __shared__ double s_bcast[3];
    unsigned int epoch = 0;
    size_t const me = static_cast<size_t>(blockIdx.x) * THREADS + threadIdx.x;
    size_t const n = static_cast<size_t>(gridDim.x) * THREADS;
    double acc = 0.0;
    for (int it = 1; it <= iters; ++it)
    {
        int const slot = 2 + 4 * (it & 1);
        /* "SpMV": two stores per thread, one partial per CTA */
        vec[me] = acc + it; vec[n + me] = acc - it;
        __syncthreads();
        if (threadIdx.x == 0)
            partials[slot * MAXB + blockIdx.x] = 1.0 + blockIdx.x * 1e-3;
        grid_barrier<B>(counter, epoch);
        all_sums<S, 1>(partials, slot, s_bcast);
        acc += s_bcast[0];
        __syncthreads();
        /* "update": three stores, three partials */
        vec[2 * n + me] = acc; vec[3 * n + me] = -acc; vec[4 * n + me] = it;
        __syncthreads();
        if (threadIdx.x < 3)
            partials[(slot + 1 + threadIdx.x) * MAXB + blockIdx.x]
                = 0.5 + threadIdx.x + blockIdx.x * 1e-3;
        grid_barrier<B>(counter, epoch);
        all_sums<S, 3>(partials, slot + 1, s_bcast);
        acc += s_bcast[0] + s_bcast[1] + s_bcast[2];
        __syncthreads();
    }
    if (me == 0)
        out[0] = acc;
}

template <int B, int S>
void run (int grid, int iters, unsigned int* counter, double* partials,
    double* vec, double* out)
{
    cudaEvent_t e0, e1;
    CHECK(cudaEventCreate(&e0)); CHECK(cudaEventCreate(&e1));
    float best = 1e30f;
    double res = 0;
    for (int rep = 0; rep < 3; ++rep)
    {
        CHECK(cudaMemset(counter, 0, sizeof(unsigned int)));
        void* args[] = { &counter, &partials, &vec, &iters, &out };
        CHECK(cudaEventRecord(e0));
        CHECK(cudaLaunchCooperativeKernel((void const*)probe<B, S>, dim3(grid),
            dim3(THREADS), args, 0, nullptr));
        CHECK(cudaEventRecord(e1));
        CHECK(cudaEventSynchronize(e1));
        float ms; CHECK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
        CHECK(cudaMemcpy(&res, out, sizeof(double), cudaMemcpyDeviceToHost));
    }
    printf("barrier %d sums %d grid %d: %.3f us per iteration (two barriers + "
        "re-sums), checksum %.6f\n", B, S, grid, best * 1e3 / iters, res);
}


/* Barrier and re-summation by warp 0 alone: lane j < NV publishes the CTA's
 * partial j, lane 0 arrives (release), all lanes poll, acquire, load their
 * share of every CTA's partials, add in the fixed order, shuffle. */
template <int NV, bool ACQ_POLL>
__device__ __forceinline__ void
sync_and_sum (unsigned int* counter, unsigned int& epoch, double* partials,
    int first_slot, double const* mine, double* s_bcast)
{
    __syncthreads();
    if (threadIdx.x < 32)
    {
        int const lane = threadIdx.x;
        if (lane < NV)
            partials[(first_slot + lane) * MAXB + blockIdx.x] = mine[lane];
        __syncwarp();
        epoch += 1;
        unsigned int const target = epoch * gridDim.x;
        if (lane == 0)
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;"
                :: "l"(counter) : "memory");
        unsigned int v;
        if (ACQ_POLL)
        {
            do {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];"
                    : "=r"(v) : "l"(counter) : "memory");
            } while (v < target);
        }
        else
        {
            do {
                asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];"
                    : "=r"(v) : "l"(counter) : "memory");
            } while (v < target);
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];"
                : "=r"(v) : "l"(counter) : "memory");
        }
        int const nb = gridDim.x;
        constexpr int U = 12;
        double t[NV][U];
#pragma unroll
        for (int j = 0; j < NV; ++j)
#pragma unroll
            for (int u = 0; u < U; ++u)
                t[j][u] = (lane + 32 * u < nb)
                    ? __ldcg(partials + (first_slot + j) * MAXB + lane + 32 * u)
                    : 0.0;
#pragma unroll
        for (int j = 0; j < NV; ++j)
        {
            double s = 0.0;
#pragma unroll
            for (int u = 0; u < U; ++u)
                if (lane + 32 * u < nb)
                    s += t[j][u];
            for (int off = 16; off > 0; off >>= 1)
                s += __shfl_down_sync(0xffffffffu, s, off);
            if (lane == 0)
                s_bcast[j] = s;
        }
    }
    __syncthreads();
}

template <bool ACQ_POLL>
__global__ void __launch_bounds__(THREADS, 2)
probe_fused (unsigned int* counter, double* partials, double* vec, int iters,
    double* out)
{
    __shared__ double s_bcast[3];
    unsigned int epoch = 0;
    size_t const me = static_cast<size_t>(blockIdx.x) * THREADS + threadIdx.x;
    size_t const n = static_cast<size_t>(gridDim.x) * THREADS;
    double acc = 0.0;
    for (int it = 1; it <= iters; ++it)
    {
        int const slot = 2 + 4 * (it & 1);
        vec[me] = acc + it; vec[n + me] = acc - it;
        double m1[1] = { 1.0 + blockIdx.x * 1e-3 };
        sync_and_sum<1, ACQ_POLL>(counter, epoch, partials, slot, m1, s_bcast);
        acc += s_bcast[0];
        __syncthreads();
        vec[2 * n + me] = acc; vec[3 * n + me] = -acc; vec[4 * n + me] = it;
        double m3[3] = { 0.5 + blockIdx.x * 1e-3, 1.5 + blockIdx.x * 1e-3,
            2.5 + blockIdx.x * 1e-3 };
        sync_and_sum<3, ACQ_POLL>(counter, epoch, partials, slot + 1, m3,
            s_bcast);
        acc += s_bcast[0] + s_bcast[1] + s_bcast[2];
        __syncthreads();
    }
    if (me == 0)
        out[0] = acc;
}

template <bool ACQ_POLL>
void run_fused (int grid, int iters, unsigned int* counter, double* partials,
    double* vec, double* out)
{
    cudaEvent_t e0, e1;
    CHECK(cudaEventCreate(&e0)); CHECK(cudaEventCreate(&e1));
    float best = 1e30f;
    double res = 0;
    for (int rep = 0; rep < 3; ++rep)
    {
        CHECK(cudaMemset(counter, 0, sizeof(unsigned int)));
        void* args[] = { &counter, &partials, &vec, &iters, &out };
        CHECK(cudaEventRecord(e0));
        CHECK(cudaLaunchCooperativeKernel((void const*)probe_fused<ACQ_POLL>,
            dim3(grid), dim3(THREADS), args, 0, nullptr));
        CHECK(cudaEventRecord(e1));
        CHECK(cudaEventSynchronize(e1));
        float ms; CHECK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
        CHECK(cudaMemcpy(&res, out, sizeof(double), cudaMemcpyDeviceToHost));
    }
    printf("fused by warp 0, %s: grid %d: %.3f us per iteration, checksum %.6f\n",
        ACQ_POLL ? "acquire polls" : "relaxed polls + one acquire", grid,
        best * 1e3 / iters, res);
}

/* Per-CTA flags fused with the re-summation (tried for cg_kernel, slower than
 * the counter: every CTA reads every flag, 264 x 9 lines per poll round at
 * 264 CTAs, against one line for the counter).
 * Thread 0 release-stores the epoch into the CTA's flag after a bar.sync; the
 * reader warps (one per sum, or warp 0 alone if ONE_POLLER, followed by a
 * bar.sync) poll all flags with relaxed loads, acquire with one fence, load
 * the partials. */
template <int NV, bool ONE_POLLER>
__device__ __forceinline__ void
flag_sums (unsigned int* flags, unsigned int& epoch, double const* partials,
    int first_slot, double* s_bcast)
{
    __syncthreads();
    epoch += 1;
    if (threadIdx.x == 0)
        asm volatile("st.release.gpu.global.u32 [%0], %1;"
            :: "l"(flags + blockIdx.x), "r"(epoch) : "memory");
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int const nb = gridDim.x;
    if (warp < (ONE_POLLER ? 1 : NV))
    {
        bool all;
        do {
            bool mine = true;
            for (int base = lane; base < nb; base += 32 * 12)
            {
                unsigned int f[12];
#pragma unroll
                for (int u = 0; u < 12; ++u)
                {
                    f[u] = epoch;
                    if (base + 32 * u < nb)
                        asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];"
                            : "=r"(f[u]) : "l"(flags + base + 32 * u)
                            : "memory");
                }
#pragma unroll
                for (int u = 0; u < 12; ++u)
                    mine = mine && f[u] >= epoch;
            }
            all = __all_sync(0xffffffffu, mine);
        } while (!all);
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
    if (ONE_POLLER)
        __syncthreads();
    if (warp < NV)
    {
        double const* p = partials + (first_slot + warp) * MAXB;
        double v = 0.0;
        for (int base = lane; base < nb; base += 32 * 12)
        {
            double t[12];
#pragma unroll
            for (int u = 0; u < 12; ++u)
                t[u] = (base + 32 * u < nb) ? __ldcg(p + base + 32 * u) : 0.0;
#pragma unroll
            for (int u = 0; u < 12; ++u)
                if (base + 32 * u < nb)
                    v += t[u];
        }
        for (int off = 16; off > 0; off >>= 1)
            v += __shfl_down_sync(0xffffffffu, v, off);
        if (lane == 0)
            s_bcast[warp] = v;
    }
    __syncthreads();
}

template <bool ONE_POLLER>
__global__ void __launch_bounds__(THREADS, 2)
probe_flags (unsigned int* flags, double* partials, double* vec, int iters,
    double* out)
{
    __shared__ double s_bcast[3];
    unsigned int epoch = 0;
    size_t const me = static_cast<size_t>(blockIdx.x) * THREADS + threadIdx.x;
    size_t const n = static_cast<size_t>(gridDim.x) * THREADS;
    double acc = 0.0;
    for (int it = 1; it <= iters; ++it)
    {
        int const slot = 2 + 4 * (it & 1);
        vec[me] = acc + it; vec[n + me] = acc - it;
        __syncthreads();
        if (threadIdx.x == 0)
            partials[slot * MAXB + blockIdx.x] = 1.0 + blockIdx.x * 1e-3;
        flag_sums<1, ONE_POLLER>(flags, epoch, partials, slot, s_bcast);
        acc += s_bcast[0];
        __syncthreads();
        vec[2 * n + me] = acc; vec[3 * n + me] = -acc; vec[4 * n + me] = it;
        __syncthreads();
        if (threadIdx.x < 3)
            partials[(slot + 1 + threadIdx.x) * MAXB + blockIdx.x]
                = 0.5 + threadIdx.x + blockIdx.x * 1e-3;
        flag_sums<3, ONE_POLLER>(flags, epoch, partials, slot + 1, s_bcast);
        acc += s_bcast[0] + s_bcast[1] + s_bcast[2];
        __syncthreads();
    }
    if (me == 0)
        out[0] = acc;
}

template <bool ONE_POLLER>
void run_flags (int grid, int iters, unsigned int* flags, double* partials,
    double* vec, double* out)
{
    cudaEvent_t e0, e1;
    CHECK(cudaEventCreate(&e0)); CHECK(cudaEventCreate(&e1));
    float best = 1e30f;
    double res = 0;
    for (int rep = 0; rep < 3; ++rep)
    {
        CHECK(cudaMemset(flags, 0, sizeof(unsigned int) * grid));
        void* args[] = { &flags, &partials, &vec, &iters, &out };
        CHECK(cudaEventRecord(e0));
        CHECK(cudaLaunchCooperativeKernel((void const*)probe_flags<ONE_POLLER>,
            dim3(grid), dim3(THREADS), args, 0, nullptr));
        CHECK(cudaEventRecord(e1));
        CHECK(cudaEventSynchronize(e1));
        float ms; CHECK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
        CHECK(cudaMemcpy(&res, out, sizeof(double), cudaMemcpyDeviceToHost));
    }
    printf("per-CTA flags, %s: grid %d: %.3f us per iteration, checksum "
        "%.6f\n", ONE_POLLER ? "warp 0 polls + bar.sync" : "every reader polls",
        grid, best * 1e3 / iters, res);
}

int main (int argc, char** argv)
{
    int const iters = 4000;
    int sms = 0;
    CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    int const grid = 2 * sms;
    unsigned int* counter; double *partials, *vec, *out;
    CHECK(cudaMalloc(&counter, sizeof(unsigned int) * MAXB));
    CHECK(cudaMalloc(&partials, sizeof(double) * 10 * MAXB));
    CHECK(cudaMalloc(&vec, sizeof(double) * 5 * grid * THREADS));
    CHECK(cudaMalloc(&out, sizeof(double)));
    CHECK(cudaMemset(partials, 0, sizeof(double) * 10 * MAXB));
    run<0, 0>(grid, iters, counter, partials, vec, out);
    run<1, 0>(grid, iters, counter, partials, vec, out);
    run<2, 0>(grid, iters, counter, partials, vec, out);
    run<0, 1>(grid, iters, counter, partials, vec, out);
    run<1, 1>(grid, iters, counter, partials, vec, out);
    run<2, 1>(grid, iters, counter, partials, vec, out);
    run_fused<false>(grid, iters, counter, partials, vec, out);
    run_fused<true>(grid, iters, counter, partials, vec, out);
    run_flags<false>(grid, iters, counter, partials, vec, out);
    run_flags<true>(grid, iters, counter, partials, vec, out);
    run<1, 1>(grid, iters, counter, partials, vec, out);
    run_flags<false>(grid, iters, counter, partials, vec, out);
    run<0, 0>(grid, iters, counter, partials, vec, out);
    return 0;
}
