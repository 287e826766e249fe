// sph_ptx.cuh -- every line of inline PTX the engine uses, in one place (sm_90a).
//
// tests/emu/cuda_emu.h provides host-side stand-ins with the same names, so that the kernel SOURCE in
// sph_kernels.cuh can also be compiled by g++ and run thread-for-thread under AddressSanitizer
// (tests/test_kernel_emulation.py); the product build never defines SPH_EMU.
#pragma once
#include <stdint.h>

// bare MUFU.RSQ / MUFU.RCP: rsqrtf() and __fdividef() without -ftz wrap the MUFU in a denormal
// rescue (FMUL 2^24, FSETP, FSEL, FMUL 2^12 -- four extra issue slots per pair); squared distances
// below 1.2e-38 m^2 do not occur and would flush to the r == 0 case, which is handled.
__device__ __forceinline__ float rsqrt_ftz(float x) {
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float rcp_ftz(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// one 32-byte record (32-byte aligned, so one sector) as two back-to-back 128-bit read-only loads
// (sm_90 has no 256-bit LDG; both LDG.E.128 are issued before either result is used)
__device__ __forceinline__ void ldg256(const float4 *p, float4 &a, float4 &b) {
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.v4.f32 {%4,%5,%6,%7}, [%8+16];"
                 : "=f"(a.x), "=f"(a.y), "=f"(a.z), "=f"(a.w), "=f"(b.x), "=f"(b.y), "=f"(b.z), "=f"(b.w)
                 : "l"(p));
}

// streamed-once 32-bit load that does not allocate in L1 (neighbour-list entries must not evict the
// gathered records)
__device__ __forceinline__ int ldg_stream(const int32_t *p) {
    int v;
    asm volatile("ld.global.nc.L1::no_allocate.b32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// ---- TMA / mbarrier primitives (sm_90 PTX; SASS UBLKCP.S.G, SYNCS.ARRIVE.TRANS64) ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra.uni WAIT_DONE;\n"
        "bra.uni WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// 1-D bulk copy global -> shared::cta; bytes multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void tma_bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// programmatic dependent launch: a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may be
// scheduled while its predecessor in the stream is still draining; everything it reads from the predecessor must
// come after this wait (a no-op for ordinary launches)
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
