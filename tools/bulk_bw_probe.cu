// bulk_bw_probe.cu -- what does one SM get out of cp.async.bulk (global -> shared) when every CTA streams its own weight images
// the way the batched sampler does?  112 CTAs; CTA b walks the regions of "rank" b % 16 (7 CTAs share every region, as the 7
// clusters of the sampler do) of a buffer of `footprint` MB, in images of `img` KB split into `chunk` KB copies, with `depth`
// images in flight.  Prints bytes per cycle per SM.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o bulk_bw_probe tools/bulk_bw_probe.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)
__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, unsigned c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void mbar_expect(unsigned long long* b, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned par) {
    unsigned done;
    do { asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(s32(b)), "r"(par) : "memory"); } while (!done);
}
__global__ void __launch_bounds__(64, 1) stream(const unsigned char* buf, size_t region_bytes, int n_regions, int img, int chunk, int depth,
                                                int n_imgs, long long* cycles, float* sink) {
    extern __shared__ __align__(128) unsigned char sm[];
    __shared__ unsigned long long full[4];
    const int tid = threadIdx.x;
    if (tid == 0) for (int i = 0; i < 4; ++i) mbar_init(full + i, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    const unsigned char* mine = buf + (size_t)(blockIdx.x % n_regions) * region_bytes;
    const int per_region = (int)(region_bytes / img);
    float acc = 0.f;
    const long long t0 = clock64();
    if (tid == 0) {
        // thread 0 is producer and consumer: keep `depth` images in flight
        int issued = 0;
        for (int done = 0; done < n_imgs; ++done) {
            while (issued < n_imgs && issued < done + depth) {
                const int slot = issued % depth;
                mbar_expect(full + slot, (unsigned)img);
                const unsigned char* src = mine + (size_t)(issued % per_region) * img;
                for (int o = 0; o < img; o += chunk)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(s32(sm + (size_t)slot * img + o)),
                                 "l"(src + o), "r"(chunk), "r"(s32(full + slot)) : "memory");
                ++issued;
            }
            const int slot = done % depth;
            mbar_wait(full + slot, (done / depth) & 1);
            acc += reinterpret_cast<float*>(sm + (size_t)slot * img)[done & 63];
        }
    }
    const long long t1 = clock64();
    if (tid == 0) { cycles[blockIdx.x] = t1 - t0; sink[blockIdx.x] = acc; }
}
int main() {
    const int G = 112;
    long long* cyc; float* sink; unsigned char* buf;
    const size_t cap = (size_t)96 << 20;
    CK(cudaMalloc(&cyc, 8 * G)); CK(cudaMalloc(&sink, 4 * G)); CK(cudaMalloc(&buf, cap)); CK(cudaMemset(buf, 1, cap));
    CK(cudaFuncSetAttribute(stream, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    printf("%-10s %-8s %-8s %-6s %-6s  B/cycle/SM   GB/s total (1.9 GHz)\n", "footprint", "img KB", "chunk KB", "depth", "CTAs");
    for (int ctas : {112, 16})
        for (int foot_mb : {8, 77})
            for (int img_kb : {64, 32})
                for (int chunk_kb : {img_kb, 8, 2})
                    for (int depth : {1, 2, 3}) {
                        if (depth * img_kb > 192) continue;
                        const size_t region = ((size_t)foot_mb << 20) / 16 / (img_kb << 10) * (img_kb << 10);
                        const int n_imgs = 600;
                        for (int rep = 0; rep < 2; ++rep) {
                            stream<<<ctas, 64, depth * img_kb * 1024>>>(buf, region, 16, img_kb << 10, chunk_kb << 10, depth, n_imgs, cyc, sink);
                            CK(cudaDeviceSynchronize());
                        }
                        long long h[G]; CK(cudaMemcpy(h, cyc, 8 * ctas, cudaMemcpyDeviceToHost));
                        double mean = 0; for (int i = 0; i < ctas; ++i) mean += (double)h[i]; mean /= ctas;
                        const double bpc = (double)n_imgs * (img_kb << 10) / mean;
                        printf("%-10d %-8d %-8d %-6d %-6d  %8.1f     %8.0f\n", foot_mb, img_kb, chunk_kb, depth, ctas, bpc, bpc * ctas * 1.9);
                    }
    return 0;
}
