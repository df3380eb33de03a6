// ubench_agg.cu — development microbenchmark (not part of the product):
// which update mechanism should the shared-memory hash aggregate use on H100?
// Input: gid[int32] + val[double] (12 B/row like config 2), N rows, G groups.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o ubench_agg ubench_agg.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint64_t mix64(uint64_t h) { h ^= h >> 33; h *= 0xff51afd7ed558ccdULL; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33; return h; }

__global__ void gen(int *gid, double *val, long long n, int G, int run)
{
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    for (; i < n; i += s) { gid[i] = (int) (mix64((uint64_t) (i / run) + 12345) % (uint64_t) G); val[i] = (double) (mix64(i) % 100000) / 100.0; }
}

// (a) global RED.ADD.F64 into R replicated dense tables {sum,cnt}
__global__ void k_global_red(const int *gid, const double *val, long long n, int G, int R, double *sum, unsigned long long *cnt, int do_cnt)
{
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    int rep = blockIdx.x % R;
    for (; i < n; i += s) {
        int g = gid[i]; double v = val[i];
        atomicAdd(&sum[(size_t) rep * G + g], v);
        if (do_cnt) atomicAdd(&cnt[(size_t) rep * G + g], 1ULL);
    }
}

// (b) CTA-shared dense table, CAS-loop fp64 atomicAdd in shared memory
__global__ void k_smem_cas(const int *gid, const double *val, long long n, int G, double *sum, unsigned long long *cnt, int do_cnt)
{
    extern __shared__ unsigned char sm[];
    double *ssum = (double *) sm; unsigned int *scnt = (unsigned int *) (ssum + G);
    for (int i = threadIdx.x; i < G; i += blockDim.x) { ssum[i] = 0; scnt[i] = 0; }
    __syncthreads();
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    for (; i < n; i += s) {
        int g = gid[i]; double v = val[i];
        atomicAdd(&ssum[g], v);
        if (do_cnt) atomicAdd(&scnt[g], 1u);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G; i += blockDim.x) { if (scnt[i] || ssum[i] != 0) { atomicAdd(&sum[i], ssum[i]); atomicAdd(&cnt[i], (unsigned long long) scnt[i]); } }
}

// (c) warp-private dense tables, no atomics: duplicates inside the warp are
// combined with match_any + shuffles, then one lane per distinct group does a
// plain read-modify-write.  Each thread keeps U rows in flight.
template <int U, int SLOTW>   // SLOTW: 1 = sum only (8 B), 2 = {sum,cnt} (16 B)
__global__ void k_warp_private(const int *gid, const double *val, long long n, int G, double *sum, unsigned long long *cnt)
{
    extern __shared__ unsigned char sm[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    double *tab = (double *) sm + (size_t) wid * G * SLOTW;
    for (int i = lane; i < G * SLOTW; i += 32) tab[i] = 0;
    __syncwarp();
    long long warp_global = (long long) blockIdx.x * nw + wid, nwarps = (long long) gridDim.x * nw;
    long long chunk = 32LL * U;
    for (long long base = warp_global * chunk; base < n; base += nwarps * chunk) {
        int g[U]; double v[U];
#pragma unroll
        for (int u = 0; u < U; u++) { long long i = base + u * 32 + lane; g[u] = i < n ? gid[i] : -1; v[u] = i < n ? val[i] : 0.0; }
#pragma unroll
        for (int u = 0; u < U; u++) {
            unsigned m = __match_any_sync(0xffffffffu, g[u]);
            double tot = v[u]; int c = 1;
            unsigned rest = m & ~((2u << lane) - 1);           // members above me
            bool leader = (m & ((1u << lane) - 1)) == 0;
            // leaders pull their followers one at a time (warp-uniform loop)
            while (__any_sync(0xffffffffu, leader && rest)) {
                int src = rest ? __ffs(rest) - 1 : lane;
                double x = __shfl_sync(0xffffffffu, v[u], src);
                if (leader && rest) { tot += x; c++; rest &= rest - 1; }
            }
            if (leader && g[u] >= 0) {
                if (SLOTW == 1) tab[g[u]] += tot;
                else { double2 t = *(double2 *) &tab[2 * g[u]]; t.x += tot; t.y = __longlong_as_double(__double_as_longlong(t.y) + c); *(double2 *) &tab[2 * g[u]] = t; }
            }
            __syncwarp();
        }
    }
    __syncwarp();
    for (int i = lane; i < G; i += 32) {
        if (SLOTW == 1) { if (tab[i] != 0) atomicAdd(&sum[i], tab[i]); }
        else { long long c = __double_as_longlong(tab[2 * i + 1]); if (c) { atomicAdd(&sum[i], tab[2 * i]); atomicAdd(&cnt[i], (unsigned long long) c); } }
    }
}

// (d) lane-private accumulators in shared memory for tiny G: slot [w][g][lane]
// -> bank == lane, conflict-free, no atomics, no matching.  W words per group.
template <int W>
__global__ void k_lane_private(const int *gid, const double *val, long long n, int G, double *sum)
{
    extern __shared__ unsigned char sm[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double *tab = (double *) sm + (size_t) wid * G * W * 32;
    for (int i = lane; i < G * W * 32; i += 32) tab[i] = 0;
    __syncwarp();
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    for (; i < n; i += s) {
        int g = gid[i]; double v = val[i];
#pragma unroll
        for (int w = 0; w < W; w++) tab[((size_t) w * G + g) * 32 + lane] += v * (w + 1);
    }
    __syncwarp();
    for (int k = lane; k < G * W; k += 32) { double t = 0; for (int l = 0; l < 32; l++) t += tab[(size_t) k * 32 + l]; atomicAdd(&sum[k], t); }
}

// (e) CTA-shared table, CAS loop, but adjacent equal keys are combined in the warp first
__global__ void k_smem_cas_combine(const int *gid, const double *val, long long n, int G, double *sum, unsigned long long *cnt)
{
    extern __shared__ unsigned char sm[];
    double *ssum = (double *) sm; unsigned int *scnt = (unsigned int *) (ssum + G);
    for (int i = threadIdx.x; i < G; i += blockDim.x) { ssum[i] = 0; scnt[i] = 0; }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    long long iters = (n + s - 1) / s;
    for (long long it = 0; it < iters; it++, i += s) {
        int g = i < n ? gid[i] : -1; double v = i < n ? val[i] : 0.0;
        unsigned m = __match_any_sync(0xffffffffu, g);
        double tot = v; int c = 1;
        unsigned rest = m & ~((2u << lane) - 1);
        bool leader = (m & ((1u << lane) - 1)) == 0;
        while (__any_sync(0xffffffffu, leader && rest)) {
            int src = rest ? __ffs(rest) - 1 : lane;
            double x = __shfl_sync(0xffffffffu, v, src);
            if (leader && rest) { tot += x; c++; rest &= rest - 1; }
        }
        if (leader && g >= 0) { atomicAdd(&ssum[g], tot); atomicAdd(&scnt[g], (unsigned) c); }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G; i += blockDim.x) { if (scnt[i]) { atomicAdd(&sum[i], ssum[i]); atomicAdd(&cnt[i], (unsigned long long) scnt[i]); } }
}

template <class F> static float time_it(F f, int reps = 5)
{
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    float best = 1e30f;
    for (int r = 0; r < reps; r++) { cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b)); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; }
    return best;
}

int main(int argc, char **argv)
{
    long long n = argc > 1 ? atoll(argv[1]) : 60000000LL;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    int *gid; double *val, *sum; unsigned long long *cnt;
    CK(cudaMalloc(&gid, n * 4)); CK(cudaMalloc(&val, n * 8));
    CK(cudaMalloc(&sum, 64 * 65536 * 8)); CK(cudaMalloc(&cnt, 64 * 65536 * 8));
    struct { int G, run; } cases[] = { { 2526, 1 }, { 2406, 4 }, { 6, 1 }, { 16384, 1 } };
    for (auto cs : cases) {
        int G = cs.G;
        gen<<<sms * 8, 256>>>(gid, val, n, G, cs.run); CK(cudaDeviceSynchronize());
        auto report = [&](const char *name, float ms) { printf("G=%d run=%d %-34s %8.3f ms %8.1f Grows/s %7.1f GB/s(12B/row)\n", G, cs.run, name, ms, n / ms / 1e6, n * 12.0 / ms / 1e6); fflush(stdout); };
        auto clear = [&]() { cudaMemset(sum, 0, 64 * 65536 * 8); cudaMemset(cnt, 0, 64 * 65536 * 8); };
        for (int R : { 1, 8, 64 }) {
            if ((size_t) R * G > 64 * 65536) continue;
            char nm[64];
            for (int dc = 0; dc < 2; dc++) { clear(); snprintf(nm, 64, "global_red R=%d cnt=%d", R, dc); report(nm, time_it([&] { k_global_red<<<sms * 8, 256>>>(gid, val, n, G, R, sum, cnt, dc); })); }
        }
        size_t smem_dense = (size_t) G * 12;
        if (smem_dense <= 200 * 1024) {
            cudaFuncSetAttribute(k_smem_cas, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
            cudaFuncSetAttribute(k_smem_cas_combine, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
            for (int dc = 0; dc < 2; dc++) {
                char nm[64];
                clear(); snprintf(nm, 64, "smem_cas 2x512 cnt=%d", dc); report(nm, time_it([&] { k_smem_cas<<<sms * 2, 512, smem_dense>>>(gid, val, n, G, sum, cnt, dc); }));
                clear(); snprintf(nm, 64, "smem_cas 1x1024 cnt=%d", dc); report(nm, time_it([&] { k_smem_cas<<<sms, 1024, smem_dense>>>(gid, val, n, G, sum, cnt, dc); }));
            }
            clear(); report("smem_cas_combine 2x512", time_it([&] { k_smem_cas_combine<<<sms * 2, 512, smem_dense>>>(gid, val, n, G, sum, cnt); }));
        }
        // warp-private: as many warps as fit in 220 KB
        for (int slotw = 1; slotw <= 2; slotw++) {
            size_t per_warp = (size_t) G * 8 * slotw;
            int nw = (int) ((220 * 1024) / per_warp); if (nw > 32) nw = 32; if (nw < 1) continue;
            char nm[64];
            if (slotw == 1) {
                cudaFuncSetAttribute(k_warp_private<8, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
                cudaFuncSetAttribute(k_warp_private<16, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
                clear(); snprintf(nm, 64, "warp_private sum U=8 warps=%d", nw); report(nm, time_it([&] { k_warp_private<8, 1><<<sms, nw * 32, per_warp * nw>>>(gid, val, n, G, sum, cnt); }));
                clear(); snprintf(nm, 64, "warp_private sum U=16 warps=%d", nw); report(nm, time_it([&] { k_warp_private<16, 1><<<sms, nw * 32, per_warp * nw>>>(gid, val, n, G, sum, cnt); }));
            } else {
                cudaFuncSetAttribute(k_warp_private<8, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
                cudaFuncSetAttribute(k_warp_private<16, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
                clear(); snprintf(nm, 64, "warp_private sum+cnt U=8 warps=%d", nw); report(nm, time_it([&] { k_warp_private<8, 2><<<sms, nw * 32, per_warp * nw>>>(gid, val, n, G, sum, cnt); }));
                clear(); snprintf(nm, 64, "warp_private sum+cnt U=16 warps=%d", nw); report(nm, time_it([&] { k_warp_private<16, 2><<<sms, nw * 32, per_warp * nw>>>(gid, val, n, G, sum, cnt); }));
            }
        }
        if (G <= 8) {
            cudaFuncSetAttribute(k_lane_private<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
            cudaFuncSetAttribute(k_lane_private<9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
            clear(); report("lane_private W=1 32 warps", time_it([&] { k_lane_private<1><<<sms, 1024, (size_t) 32 * G * 1 * 256>>>(gid, val, n, G, sum); }));
            int nw9 = (int) ((220 * 1024) / ((size_t) G * 9 * 256)); if (nw9 > 32) nw9 = 32;
            char nm[64]; snprintf(nm, 64, "lane_private W=9 warps=%d", nw9);
            clear(); report(nm, time_it([&] { k_lane_private<9><<<sms, nw9 * 32, (size_t) nw9 * G * 9 * 256>>>(gid, val, n, G, sum); }));
        }
    }
    // plain streaming read of the same bytes: the roofline reference for this input
    {
        float ms = time_it([&] { gen<<<sms * 8, 256>>>(gid, val, n, 100, 1); });
        printf("write 12B/row (gen kernel)              %8.3f ms %7.1f GB/s\n", ms, n * 12.0 / ms / 1e6);
    }
    return 0;
}
