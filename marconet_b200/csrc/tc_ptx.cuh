// Inline-PTX wrappers for mbarrier / TMA / wgmma / ldmatrix / clusters (sm_90a), shared by the tensor-core kernels.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace tcptx {

// ------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done = 0;
    const long long t_start = clock64();
    for (uint32_t it = 0; !done; ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar), "r"(parity)
            : "memory");
        if (!done && (it & 1023u) == 1023u && clock64() - t_start > 4000000000ll) __trap();   // ~2 s: a broken pipeline must fail loudly, never hang the GPU
    }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

// K-major, 128B-swizzled shared-memory matrix descriptor of wgmma (rows of 128 B, 8-row groups 1024 B apart).
__device__ __forceinline__ uint64_t make_b_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);   // start address
    d |= (uint64_t)1 << 16;                      // leading byte offset (unused for swizzled K-major; canonical value 1)
    d |= (uint64_t)(1024 >> 4) << 32;            // stride byte offset: 8 rows x 128 B
    d |= (uint64_t)1 << 62;                      // SWIZZLE_128B
    return d;
}

__device__ __forceinline__ uint32_t pack_f16(float lo_elem, float hi_elem) {
    __half2 h = __floats2half2_rn(lo_elem, hi_elem);
    return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t pack_bf16(float lo_elem, float hi_elem) {
    __nv_bfloat162 h = __floats2bfloat162_rn(lo_elem, hi_elem);
    return *reinterpret_cast<uint32_t*>(&h);
}

// Four 8x8 16-bit matrices from shared memory; lane i supplies the address of row (i & 7) of matrix (i >> 3).  With lanes 0-15
// addressing rows 0-15 at k 0-7 and lanes 16-31 the same rows at k 8-15 the result is the A fragment of a 16 x 16 tile, which is
// what one warp holds of a wgmma A operand in registers.
__device__ __forceinline__ void ldsm_x4(uint32_t saddr, uint32_t* r) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(saddr));
}

// ---- wgmma (warpgroup-wide MMA, accumulators in registers) ----
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMA window
__device__ __forceinline__ void wg_fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x N] (+)= A[64 x 16, registers] * B[16 x N, shared-memory descriptor, K-major], N = 64 or 128; BF selects bf16 over fp16.
template <int N, bool BF>
__device__ __forceinline__ void wgmma_k16_rs(float* d, const uint32_t* a, uint64_t b_desc, uint32_t accumulate) {
#define MN_WG_D8(i) "+f"(d[i + 0]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define MN_WG_ASM64(TY)                                                                                                         \
    asm volatile(                                                                                                               \
        "{\n\t.reg .pred p;\n\t"                                                                                                \
        "setp.ne.b32 p, %38, 0;\n\t"                                                                                            \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " "                                                             \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                               \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "                                     \
        "{%32, %33, %34, %35}, %36, p, 1, 1, %37;\n\t}"                                                                         \
        : MN_WG_D8(0), MN_WG_D8(8), MN_WG_D8(16), MN_WG_D8(24)                                                                  \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "n"(0), "r"(accumulate)                                      \
        : "memory")
#define MN_WG_ASM128(TY)                                                                                                        \
    asm volatile(                                                                                                               \
        "{\n\t.reg .pred p;\n\t"                                                                                                \
        "setp.ne.b32 p, %70, 0;\n\t"                                                                                            \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " "                                                            \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                               \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "                                      \
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "                                      \
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "                                     \
        "{%64, %65, %66, %67}, %68, p, 1, 1, %69;\n\t}"                                                                         \
        : MN_WG_D8(0), MN_WG_D8(8), MN_WG_D8(16), MN_WG_D8(24), MN_WG_D8(32), MN_WG_D8(40), MN_WG_D8(48), MN_WG_D8(56)          \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "n"(0), "r"(accumulate)                                      \
        : "memory")
    static_assert(N == 64 || N == 128, "wgmma_k16_rs: N must be 64 or 128");
    if constexpr (N == 64) {
        if (BF) MN_WG_ASM64("bf16");
        else MN_WG_ASM64("f16");
    } else {
        if (BF) MN_WG_ASM128("bf16");
        else MN_WG_ASM128("f16");
    }
#undef MN_WG_ASM128
#undef MN_WG_ASM64
#undef MN_WG_D8
}

// Hand registers between warpgroups (every warp of the warpgroup executes it): dec returns them to the CTA's pool, inc waits for them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// One elected lane of a fully converged warp.  Code under `if (elect_one_sync())` inside warp-uniform control flow lets ptxas
// feed TMA uniform-register operands with plain R2UR instead of the loop it emits under a divergent `lane == 0` branch.
__device__ __forceinline__ uint32_t elect_one_sync() {
    uint32_t pred = 0, laneid = 0;
    asm volatile(
        "{\n\t.reg .b32 %%rx;\n\t.reg .pred %%px;\n\t"
        "elect.sync %%rx|%%px, %2;\n\t"
        "@%%px mov.s32 %1, 1;\n\t"
        "mov.s32 %0, %%rx;\n\t}"
        : "+r"(laneid), "+r"(pred)
        : "r"(0xFFFFFFFFu));
    return pred;
}

// ---- cluster / multicast variants ----
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void tma_load_3d_mc(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1, int c2, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
        ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "h"(mask)
        : "memory");
}
// shared::cluster address of `saddr` (a shared::cta address of THIS CTA) in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t mapa_u32(uint32_t saddr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(saddr), "r"(rank));
    return r;
}
// Arrive on an mbarrier of a CTA of the cluster, with the default semantics (release at CTA scope).  For a stage read only by
// wgmma that is enough: wgmma.wait_group has completed the reads before the arrive, so the peer's TMA refill cannot overtake
// them.  (.release.cluster compiles to MEMBAR.ALL.GPU before the arrive: a GPU-scope fence per tap in the releasing warps that also
// waits for their outstanding epilogue stores.)
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

}  // namespace tcptx
