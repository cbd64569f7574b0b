// cluster_occ.cu -- how many thread-block clusters of a given size are co-resident on this GPU when every CTA needs a
// whole SM's shared memory (the sampler kernels' situation)?
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o cluster_occ tools/cluster_occ.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void dummy(int* p) { extern __shared__ int s[]; if (p) p[0] = s[0]; }
int main() {
    cudaFuncSetAttribute(dummy, cudaFuncAttributeMaxDynamicSharedMemorySize, 215 * 1024);
    cudaFuncSetAttribute(dummy, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaDeviceProp pr; cudaGetDeviceProperties(&pr, 0);
    printf("%s: %d SMs\n", pr.name, pr.multiProcessorCount);
    for (int cs : {2, 4, 6, 8, 10, 12, 14, 16}) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(cs * 32); cfg.blockDim = dim3(288); cfg.dynamicSmemBytes = 215 * 1024;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        int n = -1;
        cudaError_t e = cudaOccupancyMaxActiveClusters(&n, dummy, &cfg);
        printf("cluster size %2d: max active clusters %d (%d CTAs)%s\n", cs, n, n * cs, e == cudaSuccess ? "" : cudaGetErrorString(e));
    }
    return 0;
}
