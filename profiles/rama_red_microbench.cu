// rama_red_microbench.cu — throughput of global reductions into a Ramachandran-sized count map ([512][512][4]), the operation that bounds
// k_rama_scatter (DESIGN.md §8c): 256 M keys computed in registers (no input read), 90 % in two 64 x 64-texel basins, 10 % uniform; one
// red.global.add per key into u32 or u64 counts, with and without merging equal keys of a warp (__match_any_sync) first.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/rama_red profiles/rama_red_microbench.cu && /tmp/rama_red
// Output of one run: profiles/rama_red_microbench.jsonl (H100 80GB HBM3 SXM, 400 W power limit).
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t hsh(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33; return (uint32_t)x; }
// key distribution: 90 % in two ~64x64 texel basins, 10 % uniform over 1M
__device__ __forceinline__ uint32_t key_of(uint64_t i) {
    uint32_t h = hsh(i), r = h % 100, a = hsh(i * 7 + 1);
    if (r < 90) { uint32_t bx = (r < 45) ? 150 : 80, by = (r < 45) ? 190 : 440; uint32_t x = bx + (a & 63), y = by + ((a >> 6) & 63); return ((x * 512 + (y & 511)) << 2) | (r & 3); }
    return a & ((1u << 20) - 1);
}
template <typename T> __global__ void k(uint64_t n, T* counts, int merge) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
        const uint64_t i = base + (threadIdx.x & 31); uint32_t key = i < n ? key_of(i) : 0xffffffffu;
        if (merge) { const uint32_t peers = __match_any_sync(0xffffffffu, key); if (key != 0xffffffffu && (threadIdx.x & 31) == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&counts[key], (T)__popc(peers)); }
        else if (key != 0xffffffffu) atomicAdd(&counts[key], (T)1);
    }
}
__global__ void knoatomic(uint64_t n, uint32_t* out) { uint32_t acc = 0; const uint64_t stride = (uint64_t)gridDim.x * blockDim.x; for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) acc ^= key_of(i); if (acc == 12345) out[0] = acc; }
int main() {
    const uint64_t n = 256000000ull; void* c; cudaMalloc(&c, 8u << 20); int sm; cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    for (int blocksPerSm : {8, 16}) for (int merge : {1, 0}) for (int w : {32, 64}) {
        float best = 1e9;
        for (int r = 0; r < 4; ++r) { cudaMemset(c, 0, 8u << 20); cudaEventRecord(a);
            if (w == 32) k<unsigned int><<<sm * blocksPerSm, 256>>>(n, (unsigned int*)c, merge); else k<unsigned long long><<<sm * blocksPerSm, 256>>>(n, (unsigned long long*)c, merge);
            cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); if (r && ms < best) best = ms; }
        printf("{\"blocks_per_sm\": %d, \"merge\": %d, \"bits\": %d, \"ms\": %.3f, \"reds_per_s\": %.3e}\n", blocksPerSm, merge, w, best, n / (best * 1e-3));
    }
    float best = 1e9; for (int r = 0; r < 3; ++r) { cudaEventRecord(a); knoatomic<<<sm * 8, 256>>>(n, (uint32_t*)c); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); if (ms < best) best = ms; }
    printf("{\"no_atomics_ms\": %.3f}\n", best);
    printf("err %s\n", cudaGetErrorString(cudaGetLastError()));
}
