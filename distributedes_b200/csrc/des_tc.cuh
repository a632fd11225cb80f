// Hopper tensor-core primitives (inline PTX, sm_90a): wgmma, mbarrier, TMA, cluster shared memory.
//
// Operand layouts used by the kernels:
//   * shared-memory operands are K-major SWIZZLE_128B: rows of 64 fp16 (128 B), 16-byte chunk c of row r stored at chunk
//     (c ^ (r & 7)); 8-row groups 1024 B apart (the descriptor's stride byte offset); a K-advance of 16 elements is +32 B
//     on the descriptor start address; the atom base must be 1024-byte aligned.
//   * wgmma m64nNk16 with fp32 accumulators: warp w of the warpgroup owns rows 16w + lane/4 and 16w + lane/4 + 8; for
//     every 8-column block j it holds d[4j + 0..1] = (row lane/4, columns 8j + 2(lane%4) + 0..1) and d[4j + 2..3] = the
//     same columns of row lane/4 + 8.  An fp16 A operand in registers (k16 step) has the same per-warp layout: a[0] =
//     row lane/4, k = 2(lane%4) + 0..1; a[1] = row lane/4 + 8; a[2], a[3] = the same rows at k + 8.  So the accumulator
//     columns [16s, 16s + 16) of one layer, packed to fp16, are the A operand of k-step s of the next layer.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace des {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(bar), "r"(parity), "r"(1000000u) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {
    }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// one arrival on the mbarrier at cluster address `cbar` (a peer CTA's, from map_cluster), default semantics: a consumer
// whose reads of a buffer have completed releases it to the peer's producer (no cluster-scope fence)
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cbar) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cbar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// generic-proxy writes to this CTA's shared memory -> visible to the async proxy (wgmma operand fetch, bulk copies)
__device__ __forceinline__ void fence_proxy_async_cta() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier `id` over the first `n` threads of the CTA (whole warps)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory");
}

// ---- TMA ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void *map, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar) : "memory");
}

// one lane of a fully converged warp
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- clusters ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// every CTA of the cluster has arrived (so runs), without ordering memory: a preceding fence.mbarrier_init publishes
// mbarrier initialisation to the peers (no GPU-scope fence, unlike the .release arrive)
__device__ __forceinline__ void cluster_sync_relaxed() {
    asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
}
// address of the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t map_cluster(uint32_t saddr, uint32_t rank) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(saddr), "r"(rank));
    return ra;
}
// bulk copy of `bytes` (a multiple of 16) from this CTA's shared memory at `src` to cluster address `cdst` (a peer's
// shared memory); completes `bytes` of transaction count on the mbarrier at cluster address `cbar` in the same CTA as cdst
__device__ __forceinline__ void bulk_copy_to_peer(uint32_t cdst, uint32_t src, uint32_t bytes, uint32_t cbar) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(cdst), "r"(src), "r"(bytes), "r"(cbar) : "memory");
}

// ---- warp specialisation: per-warpgroup register budgets (every warp of the warpgroup executes it) ----------------
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- wgmma --------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA descriptor):
// [0,14) start>>4 | [16,30) LBO>>4 (=1, unused for swizzled K-major) | [32,46) SBO>>4 (1024 B) | [62,64) layout=1 (128B)
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads/writes across an asynchronous wgmma
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

#define DES_F8(d, o) "+f"(d[o + 0]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3]), "+f"(d[o + 4]), "+f"(d[o + 5]), \
                     "+f"(d[o + 6]), "+f"(d[o + 7])

// D[64 x 64] (+)= A[64 x 16] (registers, fp16) * B[64 x 16]^T (shared memory, K-major), fp32 accumulate
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b_desc, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
        : DES_F8(d, 0), DES_F8(d, 8), DES_F8(d, 16), DES_F8(d, 24)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(acc));
}
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both in shared memory (K-major), fp32 accumulate
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : DES_F8(d, 0), DES_F8(d, 8), DES_F8(d, 16), DES_F8(d, 24), DES_F8(d, 32), DES_F8(d, 40), DES_F8(d, 48),
          DES_F8(d, 56)
        : "l"(a_desc), "l"(b_desc), "r"(acc));
}
#undef DES_F8

// ---- fp16 packing -------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {       // element k (even) low half, k+1 high half
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&h);
}
// hi = fp16(x), lo = fp16(x - hi): x ~= hi + lo to ~22 mantissa bits
__device__ __forceinline__ void split_h2(float a, float b, uint32_t &hi, uint32_t &lo) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 hf = __half22float2(h);
    const __half2 l = __floats2half2_rn(a - hf.x, b - hf.y);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    lo = *reinterpret_cast<const uint32_t *>(&l);
}

// tanh(v + b) with the bias pre-scaled: bs = b * 2 log2(e).
//   e = 2^(v * 2log2e + bs);  tanh = 1 - 2/(1 + e)      abs err ~2e-7; 2 MUFU + 3 FP32 ops
constexpr float kTwoLog2e = 2.8853900817779268f;
__device__ __forceinline__ float tanh_acc_b(float v, float bs) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(__fmaf_rn(v, kTwoLog2e, bs)));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return __fmaf_rn(-2.0f, r, 1.0f);
}

__device__ __forceinline__ float tanh_fast(float x) {       // MUFU.TANH, max rel err 2^-11
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

}  // namespace tc
}  // namespace des
