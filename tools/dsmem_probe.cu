// dsmem_probe.cu -- exchange latency inside one 16-CTA cluster (the sampler's per-stage all-to-all), per variant:
//   A  {value,tag} pairs by st.shared::cluster, every thread spins on the tags of the pairs it consumes (ld.volatile.shared)
//   B  same stores, ONE warp spins on the tags, the others wait at a CTA barrier
//   C  st.async (complete_tx on an mbarrier of the destination CTA), all threads mbarrier.try_wait
//   D  plain st.shared::cluster + barrier.cluster (arrive.release / wait.acquire)
//   E  like C with 8 streams of payload: 512 B per (source, destination) per round, v2 pieces (the batched sampler's pattern)
//   F  the payload of E staged in local shared memory, then ONE cp.async.bulk (shared::cta -> shared::cluster, 512 B,
//      complete_tx on the destination's mbarrier) per destination, issued by 16 lanes
//   G  like F with 1 KB per (source, destination)
//   H  the payload of F staged in local shared memory, then ONE warp reads it back (16 B per lane) and issues one
//      st.async.v4 per destination: a whole 512-byte block per instruction
//   I  like H with 64 B per destination (lanes 0-3 only): the payload of one live stream out of 8
//   J  like H with one mbarrier per source block; warp w reads blocks 4*(w/2)..+3, each as soon as its own barrier fires
//   K  I and J together: 64 B per destination, one mbarrier per source block
// Each round every CTA publishes V=16 values (x8 in E) to all 16 CTAs and needs all 256 values of the round before it may
// publish the next one.  Prints cycles per round.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o dsmem_probe tools/dsmem_probe.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)
constexpr int CL = 16, NT = 256, V = 16;

__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned mapa(unsigned a, unsigned d) { unsigned r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(d)); return r; }
__device__ __forceinline__ void csync() { asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ unsigned crank() { unsigned r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void st_pair_remote(unsigned raddr, float v, unsigned tag) {
    unsigned long long w = ((unsigned long long)tag << 32) | __float_as_uint(v);
    asm volatile("st.shared::cluster.b64 [%0], %1;" ::"r"(raddr), "l"(w) : "memory");
}
__device__ __forceinline__ void mbar_init(unsigned long long* b, unsigned c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(unsigned long long* b, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned par) {
    unsigned done;
    do { asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(s32(b)), "r"(par) : "memory"); } while (!done);
}
__device__ __forceinline__ void st_async1(unsigned raddr, float a, unsigned rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(raddr), "r"(__float_as_uint(a)), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async4(unsigned raddr, uint4 v, unsigned rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(raddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(rbar) : "memory");
}
__device__ __forceinline__ void st_async2(unsigned raddr, float a, float b, unsigned rbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.b32 [%0], {%1, %2}, [%3];" ::"r"(raddr), "r"(__float_as_uint(a)), "r"(__float_as_uint(b)), "r"(rbar) : "memory");
}

template <int MODE>
__global__ void __launch_bounds__(NT, 1) probe(int rounds, long long* cycles, float* sink) {
    __shared__ __align__(16) unsigned long long pairs[2][CL * V];      // A, B: {value, tag}
    __shared__ __align__(16) float vals[2][8][CL * V + 4];             // C, D, E: plain values ([stream][channel])
    __shared__ unsigned long long bar[2];
    __shared__ unsigned long long jbar[2][CL];                           // J, K: one barrier per source block
    __shared__ __align__(128) float stage[2][256];                       // F, G: this CTA's contribution, staged
    __shared__ __align__(128) float blocks[2][CL][256];                  // F, G: received contributions, one block per source
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, rank = (int)crank();
    for (int i = tid; i < 2 * CL * V; i += NT) (&pairs[0][0])[i] = 0ull;
    if (tid == 0) {
        mbar_init(bar, 1); mbar_init(bar + 1, 1);
        for (int i = 0; i < 2 * CL; ++i) mbar_init(&jbar[0][0] + i, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const unsigned bytes = (MODE == 4 || MODE == 5 || MODE == 7 || MODE == 9) ? 8 * CL * V * 4 : (MODE == 6) ? 16 * CL * V * 4 : CL * V * 4;
    const unsigned jbytes = (MODE == 9) ? 512 : 64;                      // J, K: bytes per source block
    if (tid == 0) {
        mbar_expect(bar, bytes); mbar_expect(bar + 1, bytes);
        for (int i = 0; i < 2 * CL; ++i) mbar_expect(&jbar[0][0] + i, jbytes);
    }
    csync();
    float acc = 0.f;
    unsigned par[2] = {0, 0};
    const long long t0 = clock64();
    for (int r = 0; r < rounds; ++r) {
        const int b = r & 1;
        const unsigned tag = (unsigned)r + 1u;
        const float myv = acc * 1e-30f + (float)(r + tid);
        if (MODE == 0 || MODE == 1) {
            if (tid < CL * V) st_pair_remote(mapa(s32(&pairs[b][rank * V + (tid >> 4)]), tid & 15), myv, tag);
            if (MODE == 0) {
                for (int i = tid; i < CL * V; i += NT) {           // one pair per thread
                    volatile unsigned long long* vp = &pairs[b][i];
                    unsigned long long w;
                    do { w = *vp; } while ((unsigned)(w >> 32) != tag);
                    acc += __uint_as_float((unsigned)w);
                }
            } else {
                if (warp == 0)
                    for (int i = lane; i < CL * V; i += 32) {
                        volatile unsigned long long* vp = &pairs[b][i];
                        unsigned long long w;
                        do { w = *vp; } while ((unsigned)(w >> 32) != tag);
                        acc += __uint_as_float((unsigned)w);
                    }
            }
            __syncthreads();
        } else if (MODE == 2) {
            if (tid < CL * V) {
                const unsigned d = tid & 15;
                st_async1(mapa(s32(&vals[b][0][rank * V + (tid >> 4)]), d), myv, mapa(s32(bar + b), d));
            }
            mbar_wait(bar + b, par[b]);
            par[b] ^= 1;
            if (tid == 0) mbar_expect(bar + b, bytes);
            acc += vals[b][0][tid];
            __syncthreads();
        } else if (MODE == 3) {
            if (tid < CL * V) {
                const unsigned ra = mapa(s32(&vals[b][0][rank * V + (tid >> 4)]), tid & 15);
                asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(ra), "f"(myv) : "memory");
            }
            csync();
            acc += vals[b][0][tid];
        } else if (MODE == 5 || MODE == 6) {
            const int nf = (MODE == 5) ? 128 : 256;              // floats per contribution
            if (tid < nf) stage[b][tid] = myv;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncthreads();
            if (tid < CL) {
                const unsigned dst = mapa(s32(&blocks[b][rank][0]), tid), rb = mapa(s32(bar + b), tid);
                asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(dst), "r"(s32(&stage[b][0])), "r"(nf * 4), "r"(rb) : "memory");
            }
            mbar_wait(bar + b, par[b]);
            par[b] ^= 1;
            if (tid == 0) mbar_expect(bar + b, bytes);
            acc += blocks[b][tid >> 4][tid & 15];
            __syncthreads();
        } else if (MODE == 9 || MODE == 10) {
            if (tid < 128) stage[b][tid] = myv;
            __syncthreads();
            if (warp == 0 && (MODE == 9 || lane < 4)) {
                const uint4 v = *reinterpret_cast<const uint4*>(&stage[b][lane * 4]);
                const unsigned la = s32(&blocks[b][rank][lane * 4]), lb = s32(&jbar[b][rank]);
#pragma unroll
                for (int d = 0; d < CL; ++d) st_async4(mapa(la, d), v, mapa(lb, d));
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int src = 4 * (warp >> 1) + i;
                mbar_wait(&jbar[b][src], par[b]);
                if ((warp & 1) == 0 && lane == 0) mbar_expect(&jbar[b][src], jbytes);
                acc += blocks[b][src][lane & 15];
            }
            par[b] ^= 1;
            __syncthreads();
        } else if (MODE == 7 || MODE == 8) {
            if (tid < 128) stage[b][tid] = myv;
            __syncthreads();
            if (warp == 0 && (MODE == 7 || lane < 4)) {
                const uint4 v = *reinterpret_cast<const uint4*>(&stage[b][lane * 4]);
                const unsigned la = s32(&blocks[b][rank][lane * 4]), lb = s32(bar + b);
#pragma unroll
                for (int d = 0; d < CL; ++d) st_async4(mapa(la, d), v, mapa(lb, d));
            }
            mbar_wait(bar + b, par[b]);
            par[b] ^= 1;
            if (tid == 0) mbar_expect(bar + b, bytes);
            acc += blocks[b][tid >> 4][tid & 15];
            __syncthreads();
        } else {                                                 // E: warp w publishes channels 2w,2w+1 of 8 streams as v2
            const int s = lane & 7;
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const unsigned d = (lane >> 3) + 4 * it;
                st_async2(mapa(s32(&vals[b][s][rank * V + 2 * warp]), d), myv, myv + 1.f, mapa(s32(bar + b), d));
            }
            mbar_wait(bar + b, par[b]);
            par[b] ^= 1;
            if (tid == 0) mbar_expect(bar + b, bytes);
            acc += vals[b][tid >> 5][tid & 31];
            __syncthreads();
        }
    }
    const long long t1 = clock64();
    csync();
    if (tid == 0 && blockIdx.x == 0) *cycles = t1 - t0;
    sink[blockIdx.x * NT + tid] = acc;
}

template <int MODE>
static void run(const char* name, int rounds, int clusters) {
    long long* cyc; float* sink;
    CK(cudaMalloc(&cyc, 8)); CK(cudaMalloc(&sink, 4 * NT * CL * clusters));
    CK(cudaFuncSetAttribute(probe<MODE>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(CL * clusters); cfg.blockDim = dim3(NT);
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    for (int rep = 0; rep < 2; ++rep) {
        CK(cudaLaunchKernelEx(&cfg, probe<MODE>, rounds, cyc, sink));
        CK(cudaDeviceSynchronize());
    }
    long long c; CK(cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost));
    printf("%-70s clusters=%d  %8.1f cycles/round\n", name, clusters, (double)c / rounds);
    cudaFree(cyc); cudaFree(sink);
}

int main() {
    const int rounds = 20000;
    for (int clusters : {1, 8}) {
        run<0>("A tagged pairs, every thread spins on its pair", rounds, clusters);
        run<1>("B tagged pairs, one warp spins, CTA barrier", rounds, clusters);
        run<2>("C st.async + mbarrier (1 KB per CTA per round)", rounds, clusters);
        run<3>("D plain remote stores + barrier.cluster", rounds, clusters);
        run<4>("E st.async v2, 8 streams (8 KB per CTA per round)", rounds, clusters);
        run<5>("F bulk copy smem->dsmem, 512 B x 16 destinations", rounds, clusters);
        run<6>("G bulk copy smem->dsmem, 1 KB x 16 destinations", rounds, clusters);
        run<7>("H one warp: LDS.128 + st.async.v4, 512 B per instruction per destination", rounds, clusters);
        run<8>("I like H, 64 B per destination (lanes 0-3: one live stream)", rounds, clusters);
        run<9>("J like H, one mbarrier per source block, read as they land", rounds, clusters);
        run<10>("K I + J: 64 B per destination, one mbarrier per source block", rounds, clusters);
    }
    return 0;
}
