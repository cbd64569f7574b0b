// lat_probe.cu -- micro-measurements behind the sampler's exchange design (run on an H100):
//   1. flag ping-pong between two CTAs (store -> visible -> load) : one-way exchange latency through L2
//   2. all-to-all round among G CTAs: each CTA publishes V {value,tag} pairs, every CTA collects all G*V pairs
//      variants: who polls (all threads / one warp), vector width, nanosleep backoff
//   3. atomic-counter grid barrier round
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o lat_probe tools/lat_probe.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <cooperative_groups.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ unsigned long long ld64(const unsigned long long* p) {
    unsigned long long w; asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w) : "l"(p) : "memory"); return w;
}
__device__ __forceinline__ void st64(unsigned long long* p, unsigned long long w) {
    asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" :: "l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ void ld64x2(const unsigned long long* p, unsigned long long& a, unsigned long long& b) {
    asm volatile("ld.relaxed.gpu.global.v2.b64 {%0,%1}, [%2];" : "=l"(a), "=l"(b) : "l"(p) : "memory");
}

// ---- 1. ping-pong
__global__ void pingpong(unsigned long long* flags, int iters, long long* cycles) {
    if (threadIdx.x != 0) return;
    unsigned long long* mine = flags + blockIdx.x * 32, *other = flags + (1 - blockIdx.x) * 32;
    long long t0 = clock64();
    for (int i = 1; i <= iters; ++i) {
        if (blockIdx.x == 0) { st64(mine, i); while (ld64(other) != (unsigned long long)i) {} }
        else { while (ld64(other) != (unsigned long long)i) {} st64(mine, i); }
    }
    if (blockIdx.x == 0) *cycles = clock64() - t0;
}

// ---- 2. all-to-all rounds.  buf[2][G*V] pairs (parity double buffered), tag = round+1
template <int MODE>   // 0: every thread polls pairs tid, tid+NT..; 1: same + nanosleep(40); 2: one warp polls, x2 vector; 3: all threads, x2 vector
__global__ void __launch_bounds__(256, 1) all2all(unsigned long long* buf, int V, int rounds, long long* cycles, float* sink) {
    const int G = gridDim.x, n = G * V, tid = threadIdx.x;
    __shared__ float vals[4096];
    float acc = 0.f;
    __syncthreads();
    long long t0 = clock64();
    for (int r = 0; r < rounds; ++r) {
        unsigned long long* b = buf + (size_t)(r & 1) * n;
        const unsigned long long tag = (unsigned long long)(r + 1) << 32;
        if (tid < V) st64(b + blockIdx.x * V + tid, tag | (unsigned)(r + tid));
        if (MODE == 0 || MODE == 1) {
            for (int i = tid; i < n; i += 256) {
                unsigned long long w = ld64(b + i);
                while ((w >> 32) != (unsigned long long)(r + 1)) { if (MODE == 1) __nanosleep(40); w = ld64(b + i); }
                vals[i] = __uint_as_float((unsigned)w);
            }
        } else if (MODE == 2) {
            if (tid < 32)
                for (int i = 2 * tid; i < n; i += 64) {
                    unsigned long long w0, w1;
                    do { ld64x2(b + i, w0, w1); } while ((w0 >> 32) != (unsigned long long)(r + 1) || (w1 >> 32) != (unsigned long long)(r + 1));
                    vals[i] = __uint_as_float((unsigned)w0); vals[i + 1] = __uint_as_float((unsigned)w1);
                }
        } else {
            for (int i = 2 * tid; i < n; i += 512) {
                unsigned long long w0, w1;
                do { ld64x2(b + i, w0, w1); } while ((w0 >> 32) != (unsigned long long)(r + 1) || (w1 >> 32) != (unsigned long long)(r + 1));
                vals[i] = __uint_as_float((unsigned)w0); vals[i + 1] = __uint_as_float((unsigned)w1);
            }
        }
        __syncthreads();
        acc += vals[(tid * 7) % n];
        __syncthreads();
    }
    if (blockIdx.x == 0 && tid == 0) *cycles = clock64() - t0;
    if (acc == 123.456f) *sink = acc;
}

// ---- 3. atomic grid barrier
__global__ void __launch_bounds__(256, 1) barrier_rounds(unsigned* ctr, int rounds, long long* cycles) {
    unsigned target = 0;
    __syncthreads();
    long long t0 = clock64();
    for (int r = 0; r < rounds; ++r) {
        __syncthreads();
        if (threadIdx.x == 0) {
            target += gridDim.x;
            __threadfence();
            atomicAdd(ctr, 1u);
            unsigned v;
            do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory"); } while ((int)(v - target) < 0);
        }
        __syncthreads();
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *cycles = clock64() - t0;
}

template <typename K, typename... A>
static double run_coop(K kern, int grid, int block, int rounds, long long* d_cyc, A... args) {
    void* params[] = {(void*)&args...};
    CK(cudaLaunchCooperativeKernel((const void*)kern, dim3(grid), dim3(block), params, 0, 0));
    CK(cudaDeviceSynchronize());
    long long c; CK(cudaMemcpy(&c, d_cyc, sizeof(c), cudaMemcpyDeviceToHost));
    return (double)c / rounds;
}

int main() {
    int clk_khz; CK(cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0));
    printf("SM clock (max) %.0f MHz\n", clk_khz / 1e3);
    unsigned long long* buf; long long* cyc; float* sink; unsigned* ctr;
    CK(cudaMalloc(&buf, 1 << 22)); CK(cudaMalloc(&cyc, 8)); CK(cudaMalloc(&sink, 4)); CK(cudaMalloc(&ctr, 4));
    int iters = 2000;
    CK(cudaMemset(buf, 0, 1 << 22));
    { void* params[] = {&buf, &iters, &cyc};
      CK(cudaLaunchCooperativeKernel((const void*)pingpong, dim3(2), dim3(32), params, 0, 0)); CK(cudaDeviceSynchronize());
      long long c; CK(cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost));
      printf("ping-pong round trip: %.0f cycles (one-way exchange ~%.0f)\n", (double)c / iters, (double)c / iters / 2); }
    int rounds = 2000;
    for (int G : {16, 64, 128, 148}) for (int V : {2, 4}) {
        double r[4];
        CK(cudaMemset(buf, 0, 1 << 22)); r[0] = run_coop(all2all<0>, G, 256, rounds, cyc, buf, V, rounds, cyc, sink);
        CK(cudaMemset(buf, 0, 1 << 22)); r[1] = run_coop(all2all<1>, G, 256, rounds, cyc, buf, V, rounds, cyc, sink);
        CK(cudaMemset(buf, 0, 1 << 22)); r[2] = run_coop(all2all<2>, G, 256, rounds, cyc, buf, V, rounds, cyc, sink);
        CK(cudaMemset(buf, 0, 1 << 22)); r[3] = run_coop(all2all<3>, G, 256, rounds, cyc, buf, V, rounds, cyc, sink);
        printf("all-to-all G=%3d V=%d (%4d pairs): all-threads %6.0f | +nanosleep %6.0f | one-warp x2 %6.0f | all-threads x2 %6.0f  cycles/round\n",
               G, V, G * V, r[0], r[1], r[2], r[3]);
    }
    for (int G : {16, 64, 128, 148}) {
        CK(cudaMemset(ctr, 0, 4));
        double c = run_coop(barrier_rounds, G, 256, rounds, cyc, ctr, rounds, cyc);
        printf("atomic grid barrier G=%3d: %6.0f cycles/round\n", G, c);
    }
    return 0;
}
