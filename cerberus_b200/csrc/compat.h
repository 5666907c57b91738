// compat.h -- the handful of launch / qualifier macros the kernels are written against.
// Product build (nvcc, sm_90a): plain CUDA.  With -DCERB_CUSIM (tests/cusim, g++) the same kernel
// sources run on CPU threads so the non-GPU test tier can exercise the real kernel logic; that build
// is test infrastructure, is never linked into libcerberus_b200.so and is never a fallback.
#pragma once
#include <math.h>
#include <stdint.h>
#if defined(CERB_CUSIM)
#include "cusim.h"
#else
#include <cuda_runtime.h>
#define CERB_HD __host__ __device__ __forceinline__
#define CERB_D __device__ __forceinline__
#define CERB_GLOBAL __global__
// phase functions of the solve kernel are real calls: each gets its own register allocation (the kernel as one inlined
// body ran at the 255-register cap with spills in its hottest loops); the kernel parameter block stays addressable in place
#define CERB_NOINLINE __device__ __noinline__
#define CERB_GRID_CONSTANT const __grid_constant__
#define CERB_DYN_SMEM(T, name)                                   \
    extern __shared__ __align__(16) unsigned char name##_raw[]; \
    T *name = reinterpret_cast<T *>(name##_raw)
#define CERB_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
// named barrier among a subset of warps (bar.sync id, nthreads)
#define CERB_BAR_SYNC(id, nthreads) asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory")
// asynchronous global -> shared copy of one double (LDGSTS): the data lands in shared memory without passing through
// registers and without stalling the issuing thread; CERB_CP_ASYNC_WAIT() makes this thread's copies complete
#define CERB_CP_ASYNC8(dst_smem, src_global) asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src_global) : "memory")
#define CERB_CP_ASYNC_WAIT() asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory")
// 1-D bulk copy global -> shared through the TMA unit (cp.async.bulk, SASS UBLKCP): ONE thread issues the whole region, completion is
// signalled on an mbarrier in shared memory (transaction bytes), every consumer waits on the barrier's phase parity.  Addresses and size
// must be multiples of 16 bytes.  The issuing thread fences the async proxy first (the destination was last touched by generic accesses).
#define CERB_SMEM_U32(p) ((unsigned)__cvta_generic_to_shared(p))
#define CERB_MBAR_INIT(bar) do { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(CERB_SMEM_U32(bar))); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); } while (0)
#define CERB_BULK_G2S(dst_smem, src_global, bytes, bar) do {                                                                                        \
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");                                                                                 \
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(CERB_SMEM_U32(bar)), "r"((unsigned)(bytes)) : "memory");         \
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"                                      \
                     ::"r"(CERB_SMEM_U32(dst_smem)), "l"(src_global), "r"((unsigned)(bytes)), "r"(CERB_SMEM_U32(bar)) : "memory");                   \
    } while (0)
#define CERB_MBAR_WAIT(bar, parity) do {                                                                                                             \
        unsigned done_ = 0;                                                                                                                          \
        while (!done_) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"                 \
                                    : "=r"(done_) : "r"(CERB_SMEM_U32(bar)), "r"((unsigned)(parity)) : "memory");                                    \
    } while (0)
// producer / consumer hand-over through a shared-memory flag: release store by the producer (after a __syncwarp that orders the other
// lanes' writes before it), acquire load in the consumer's spin loop
#define CERB_ST_RELEASE_S32(p, v) asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(CERB_SMEM_U32(p)), "r"((int)(v)) : "memory")
#define CERB_LD_ACQUIRE_S32(p) ({ int v_; asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v_) : "r"(CERB_SMEM_U32(p)) : "memory"); v_; })
// body of a spin-wait on a shared-memory flag (a short sleep keeps the polling warps out of the producer's issue slots)
#define CERB_SPIN_PAUSE() __nanosleep(20)
// non-blocking arrival at a named barrier (producer / consumer hand-over: one side arrives, the other side syncs)
#define CERB_BAR_ARRIVE(id, nthreads) asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory")
// fp64 tensor-core MMA, D(8x8) = A(8x4, row) * B(4x8, col) + C.  Fragment layout (PTX ISA, m8n8k4 .f64):
//   a = A[lane / 4][lane % 4], b = B[lane % 4][lane / 4], c/d{0,1} = C[lane / 4][2 * (lane % 4) + {0,1}]
#define CERB_DMMA(d0, d1, a, b, c0, c1) \
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%4,%5};" : "=d"(d0), "=d"(d1) : "d"(a), "d"(b), "d"(c0), "d"(c1))
#endif
