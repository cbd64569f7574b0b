// tc_ptx.cuh -- inline-PTX wrappers for the Hopper (sm_90a) tensor-core kernels (tc_gemm.cu, tc_block.cu, tc_bwd2.cu):
// mbarrier, TMA, warpgroup MMA (wgmma) with shared-memory descriptors, gate activations and bf16 pair splitting.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdint>

namespace wn {
namespace px {

constexpr unsigned SPIN_LIMIT = 1u << 28;     // a barrier that never completes traps instead of hanging the GPU

__device__ __forceinline__ unsigned s32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, unsigned n) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory");
}
__device__ __forceinline__ bool mbar_try(unsigned long long* b, unsigned parity) {
    unsigned done;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(s32(b)), "r"(parity) : "memory");
    return done != 0;
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity) {
    unsigned spins = 0;
    while (!mbar_try(b, parity)) if (++spins > SPIN_LIMIT) asm volatile("trap;");
}
// ---- TMA loads into this CTA's shared memory, completing on this CTA's barrier
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, unsigned long long* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(s32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, unsigned long long* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(s32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, unsigned long long* bar) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
                 ::"r"(s32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(s32(bar)) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier of one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---- wgmma (sm_90a): a warpgroup (4 consecutive warps) computes D[64 x 128] (+)= A[64 x K] * B[K x 128] from shared memory,
// fp32 accumulators in registers.  Fragment of thread i of the warpgroup (warp w = i / 32, lane l): d[4n + 2r + c] is row
// 16w + l/4 + 8r, column 8n + 2(l%4) + c.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_keep(float (&d)[N]) {       // the accumulators stay in place across the async MMAs
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// bf16 x bf16 -> fp32, K = 16; t<A><B>: 0 = K-major operand, 1 = MN-major (transposed) operand.  acc = 0 overwrites D.
__device__ __forceinline__ void wgmma_bf16_t00(float (&d)[64], unsigned long long a, unsigned long long b, unsigned acc) {
    asm volatile("{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0; }"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}
__device__ __forceinline__ void wgmma_bf16_t11(float (&d)[64], unsigned long long a, unsigned long long b, unsigned acc) {
    asm volatile("{ .reg .pred p; setp.ne.b32 p, %66, 0;\n"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 1, 1; }"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(acc) : "memory");
}

// shared-memory matrix descriptor (wgmma): start address, leading / stride byte offsets, layout (0 = no swizzle, 1 = 128B,
// 2 = 64B, 3 = 32B).  No swizzle, K-major: lbo = bytes between the 16-byte K chunks of a k-step, sbo = bytes between 8-row
// groups; no swizzle, MN-major: lbo = bytes between 8-deep K groups, sbo = bytes between 8-wide MN groups.  Swizzled K-major:
// lbo unused, sbo = bytes between 8-row atoms.
__device__ __forceinline__ unsigned long long wg_desc(unsigned saddr, unsigned lbo, unsigned sbo, unsigned layout = 0) {
    unsigned long long d = 0;
    d |= (unsigned long long)((saddr >> 4) & 0x3fff);
    d |= (unsigned long long)((lbo >> 4) & 0x3fff) << 16;
    d |= (unsigned long long)((sbo >> 4) & 0x3fff) << 32;
    d |= (unsigned long long)layout << 62;
    return d;
}

// ---- activations for the gate: ex2 / rcp approximations (relative error ~2e-7; the parity bar is 1e-4 on the logits)
__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcpf(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sigmoid_fast(float x) { return rcpf(1.f + ex2f(-1.4426950408889634f * x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 1.f - 2.f * rcpf(1.f + ex2f(2.8853900817779268f * x)); }

// fp32 -> bf16 (hi, lo) pair; packs two values per 32-bit word, first value in the low half
__device__ __forceinline__ void split2(float a, float b, unsigned& hi, unsigned& lo) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    const float2 hf = __bfloat1622float2(h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const unsigned*>(&h);
    lo = *reinterpret_cast<const unsigned*>(&l);
}
__device__ __forceinline__ float2 unpack_bf16x2(unsigned w) {
    return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}

}  // namespace px
}  // namespace wn
