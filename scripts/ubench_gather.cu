// ubench_gather.cu — development microbenchmark: random 16-byte gathers and
// random 64-bit CAS over tables of growing size (is the join table's random
// access bound by DRAM, by the TLB reach, or by the atomic units?).
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)
__device__ __forceinline__ uint64_t mix64(uint64_t h) { h ^= h >> 33; h *= 0xff51afd7ed558ccdULL; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ULL; h ^= h >> 33; return h; }

template <int U>
__global__ void k_gather(const ulonglong2 *tab, uint64_t mask, long long n, unsigned long long *sink, int run)
{
    long long i = ((long long) blockIdx.x * blockDim.x + threadIdx.x) * U, s = (long long) gridDim.x * blockDim.x * U;
    unsigned long long acc = 0;
    for (; i < n; i += s) {
        ulonglong2 v[U];
#pragma unroll
        for (int u = 0; u < U; u++) v[u] = tab[mix64((uint64_t) ((i + u) / run) * 0x9E3779B97F4A7C15ULL) & mask];
#pragma unroll
        for (int u = 0; u < U; u++) acc += v[u].x ^ v[u].y;
    }
    if (acc == 0x1234567) *sink = acc;
}
__global__ void k_cas(unsigned long long *tab, uint64_t mask, long long n, int do_store)
{
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    for (; i < n; i += s) {
        uint64_t slot = mix64((uint64_t) i * 0x9E3779B97F4A7C15ULL) & mask;
        unsigned long long old = atomicCAS(&tab[2 * slot], 0ULL, (unsigned long long) i + 1);
        if (do_store && old == 0) tab[2 * slot + 1] = (unsigned long long) i;
    }
}
// plain (non-atomic) random 16-byte stores
__global__ void k_store(ulonglong2 *tab, uint64_t mask, long long n)
{
    long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x, s = (long long) gridDim.x * blockDim.x;
    for (; i < n; i += s) { uint64_t slot = mix64((uint64_t) i * 0x9E3779B97F4A7C15ULL) & mask; tab[slot] = make_ulonglong2((unsigned long long) i, 7ULL); }
}
template <class F> static float time_it(F f, int reps = 3)
{
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); float best = 1e30f;
    for (int r = 0; r < reps; r++) { cudaEventRecord(a); f(); cudaEventRecord(b); CK(cudaEventSynchronize(b)); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; }
    return best;
}
int main()
{
    const long long n = 200000000LL;
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    unsigned long long *sink; CK(cudaMalloc(&sink, 8));
    for (long long mb : { 64LL, 256LL, 1024LL, 4096LL, 16384LL }) {
        size_t bytes = (size_t) mb << 20; uint64_t slots = bytes / 16;
        ulonglong2 *tab; CK(cudaMalloc(&tab, bytes)); CK(cudaMemset(tab, 0, bytes));
        auto rep = [&](const char *nm, float ms) { printf("table %6lld MB  %-28s %8.3f ms  %7.2f G acc/s  %7.1f GB/s @32B\n", mb, nm, ms, n / ms / 1e6, n * 32.0 / ms / 1e6); fflush(stdout); };
        rep("gather U=1 run=1 2048thr/SM", time_it([&] { k_gather<1><<<sms * 8, 256>>>(tab, slots - 1, n, sink, 1); }));
        rep("gather U=4 run=1", time_it([&] { k_gather<4><<<sms * 8, 256>>>(tab, slots - 1, n, sink, 1); }));
        rep("gather U=8 run=1", time_it([&] { k_gather<8><<<sms * 8, 256>>>(tab, slots - 1, n, sink, 1); }));
        rep("gather U=4 run=4", time_it([&] { k_gather<4><<<sms * 8, 256>>>(tab, slots - 1, n, sink, 4); }));
        rep("store 16B", time_it([&] { k_store<<<sms * 8, 256>>>(tab, slots - 1, n); }));
        CK(cudaMemset(tab, 0, bytes));
        rep("cas only", time_it([&] { k_cas<<<sms * 8, 256>>>((unsigned long long *) tab, slots - 1, n, 0); }, 1));
        CK(cudaMemset(tab, 0, bytes));
        rep("cas + payload store", time_it([&] { k_cas<<<sms * 8, 256>>>((unsigned long long *) tab, slots - 1, n, 1); }, 1));
        cudaFree(tab);
    }
    return 0;
}
