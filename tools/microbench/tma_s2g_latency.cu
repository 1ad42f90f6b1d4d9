// Microbenchmark: latency of one cp.async.bulk shared -> global store of N bytes until the source may be reused
// (wait_group.read) and until the write is complete (wait_group), vs a lane-group copy with 128-bit stores.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 tma_s2g_latency.cu -o tma_s2g_latency
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void probe(int4* dst, int bytes, int lanes, long long* out, int iters) {
    extern __shared__ __align__(128) unsigned char sm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char* src = sm + (size_t)warp * 4096;
    for (int i = lane; i < 1024; i += 32) reinterpret_cast<int*>(src)[i] = i + warp;
    __syncwarp();
    int4* d = dst + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * 256 * 64;
    long long t_read = 0, t_full = 0, t_copy = 0;
    for (int it = 0; it < iters; it++) {
        int4* row = d + (size_t)(it & 63) * 256;
        __syncwarp();
        long long t0 = clock64();
        if (lane == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(row), "r"(smem_u32(src)), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        }
        __syncwarp();
        long long t1 = clock64();
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
        __syncwarp();
        long long t2 = clock64();
        const int4* s4 = reinterpret_cast<const int4*>(src);
        for (int i = lane; i < bytes / 16; i += lanes) if (lane < lanes) row[i] = s4[i];
        __syncwarp();
        long long t3 = clock64();
        t_read += t1 - t0; t_full += t2 - t0; t_copy += t3 - t2;
    }
    if (lane == 0 && warp == 0 && blockIdx.x == 0) { out[0] = t_read / iters; out[1] = t_full / iters; out[2] = t_copy / iters; }
}

int main() {
    int4* dst; long long* out; long long h[3];
    cudaMalloc(&dst, (size_t)148 * 8 * 256 * 64 * 16);
    cudaMalloc(&out, 24);
    for (int warps : {1, 8}) for (int bytes : {192, 896, 3072}) for (int lanes : {8, 32}) {
        probe<<<148, warps * 32, warps * 4096>>>(dst, bytes, lanes, out, 200);
        cudaDeviceSynchronize();
        cudaMemcpy(h, out, 24, cudaMemcpyDeviceToHost);
        printf("warps/SM %d bytes %4d copy-lanes %2d : tma source-free %lld cyc, tma complete %lld cyc, lane copy %lld cyc (%s)\n",
               warps, bytes, lanes, h[0], h[1], h[2], cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}
