// fm_ptx.cuh -- thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma,
// scoped acquire/release accesses used by the cross-CTA and cross-GPU flag protocol.
// Hand-written for this project (no CUTLASS/CuTe on the hot path -- BASELINE.json north_star).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace fm {

// ----------------------------------------------------------------------------------------------------------------
// bounded spinning: every wait in the kernel gives up after `timeout_ns`, records why in a host-mapped debug record
// and traps, so a protocol bug or a dead peer ends the launch with an error instead of hanging the GPU.
// ----------------------------------------------------------------------------------------------------------------
struct DebugRecord {          // lives in pinned, device-mapped host memory (readable after a trap)
    unsigned int code;        // FM_TRAP_* below (0 = none)
    unsigned int block;
    unsigned int thread;
    unsigned int info0;
    unsigned int info1;
    unsigned int info2;
    unsigned long long waited_ns;
};

enum : unsigned int {
    FM_TRAP_NONE = 0,
    FM_TRAP_MBAR = 1,   // info0 = the barrier's id in the kernel's mbarrier table (fm_kernel.cuh), info1 = the parity
    // 2-6 and 12: no longer used
    FM_TRAP_GRID_BARRIER = 7,
    FM_TRAP_RECV_FLAG = 8,
    FM_TRAP_G0_DONE = 9,
    FM_TRAP_RET_FLAG = 10,
    FM_TRAP_RECV_ROWS = 11,
    // not a trap: the launch read a token count outside [0, S] from device memory and ran on 0 tokens (info0 = the
    // count, info1 = S).  The host reports it once and clears the record; the context stays usable.
    FM_STATUS_BAD_COUNT = 13,
    // not a trap: a routed launch read an expert index outside [-1, E) and treated that pick as -1 (info0 = the token,
    // info1 = the pick, info2 = the index).  Reported once like FM_STATUS_BAD_COUNT.
    FM_STATUS_BAD_EXPERT = 14,
};

// plain stores to pinned host memory (no PCIe atomics needed); first writer wins loosely
__device__ __forceinline__ void fm_record(DebugRecord* dbg, unsigned int code, unsigned int i0, unsigned int i1,
                                          unsigned int i2, unsigned long long waited) {
    if (dbg != nullptr) {
        volatile DebugRecord* d = dbg;
        if (d->code == 0u) {
            d->block = blockIdx.x;
            d->thread = threadIdx.x;
            d->info0 = i0;
            d->info1 = i1;
            d->info2 = i2;
            d->waited_ns = waited;
            d->code = code;
            __threadfence_system();
        }
    }
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __noinline__ void fm_trap(DebugRecord* dbg, unsigned int code, unsigned int i0, unsigned int i1,
                                     unsigned int i2, unsigned long long waited) {
    fm_record(dbg, code, i0, i1, i2, waited);
    __trap();
}

struct SpinGuard {  // cheap: reads %globaltimer only every 256 polls
    unsigned long long t0 = 0;
    unsigned int polls = 0;
    __device__ __forceinline__ void tick(DebugRecord* dbg, unsigned long long timeout_ns, unsigned int code,
                                         unsigned int i0, unsigned int i1, unsigned int i2) {
        if ((++polls & 255u) == 0u) {
            const unsigned long long now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > timeout_ns) fm_trap(dbg, code, i0, i1, i2, now - t0);
        }
    }
};

// ----------------------------------------------------------------------------------------------------------------
// shared-memory addressing + mbarrier
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// `id` only names the barrier in a timeout record
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, DebugRecord* dbg,
                                          unsigned long long timeout_ns, unsigned int id) {
    SpinGuard g;
    while (!mbar_try_wait(bar, parity)) g.tick(dbg, timeout_ns, FM_TRAP_MBAR, id, parity, 0);
}

// named CTA barriers (id 0 is __syncthreads): the N threads that take part, whole warps, either wait (sync) or only
// signal (arrive); id and count are immediates
template <int ID, int N>
__device__ __forceinline__ void named_sync() {
    static_assert(ID > 0 && ID < 16 && N % 32 == 0, "named barrier id 1-15, whole warps");
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(N) : "memory");
}
template <int ID, int N>
__device__ __forceinline__ void named_arrive() {
    static_assert(ID > 0 && ID < 16 && N % 32 == 0, "named barrier id 1-15, whole warps");
    asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------------------------
// proxy / memory fences
// ----------------------------------------------------------------------------------------------------------------
// generic-proxy global writes <-> async-proxy (TMA) global reads
__device__ __forceinline__ void fence_proxy_async_global() {
    asm volatile("fence.proxy.async.global;" ::: "memory");
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------------------------
// scoped loads/stores/reductions for flags and counters
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys_u32(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_sys_add_u32(unsigned int* p, unsigned int v) {  // also on peer-mapped addresses
    asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_gpu_u32(const unsigned int* p) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_acquire_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_release_gpu_add_u32(unsigned int* p, unsigned int v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int atom_acq_rel_gpu_add_u32(unsigned int* p, unsigned int v) {
    unsigned int old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ unsigned long long atom_acq_rel_gpu_add_u64(unsigned long long* p,
                                                                       unsigned long long v) {
    unsigned long long old;
    asm volatile("atom.acq_rel.gpu.global.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(p), "l"(v) : "memory");
    return old;
}

// 16-byte global accesses (coalesced row copies, also valid on NVLink peer-mapped addresses)
__device__ __forceinline__ uint4 ld_global_nc_v4(const void* p) {
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ld_global_v4(const void* p) {  // coherent path (data written during this launch)
    uint4 v;
    asm volatile("ld.global.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(p)
                 : "memory");
    return v;
}
__device__ __forceinline__ int4 ld_global_cg_i4(const void* p) {   // L2-coherent (data written by other SMs in this launch)
    int4 v;
    asm volatile("ld.global.cg.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_global_v4(void* p, const uint4& v) {
    asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}

// 8 x bf16 element-wise add into global memory (REDG.E.ADD.BF16x8.RN): round-to-nearest-even like a bf16 atomicAdd,
// no return value; valid on peer-mapped addresses (NVLink atomics)
__device__ __forceinline__ void red_add_bf16x8(void* p, const uint4& v) {
    asm volatile("red.relaxed.sys.global.add.noftz.v4.bf16x2 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
}

// ----------------------------------------------------------------------------------------------------------------
// TMA: 2-D tiled bulk tensor load, global -> shared, completion on an mbarrier (complete_tx::bytes)
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}
// 1-D bulk copies through the TMA engine (no tensor map): contiguous global -> shared with mbarrier completion, and
// shared -> global (also peer-mapped) tracked with bulk async-groups
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void bulk_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// until at most N committed bulk groups of this thread still have to read their smem source
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
// shared-memory only: generic-proxy accesses to smem <-> async-proxy (TMA) accesses to the same smem; does not wait for
// the thread's outstanding global stores
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// L2 prefetch of a tensor tile (no smem destination, no barrier): hides HBM latency for k-blocks the pipeline will
// request a few steps later
__device__ __forceinline__ void tma_prefetch_l2_2d(const void* tmap, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, int32_t c0, int32_t c1,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// 2-D tiled bulk tensor store, shared -> global, tracked with bulk async-groups (bulk_commit_group / bulk_wait_group*).
// The smem source must hold the box in the tensor map's swizzled layout; rows outside the tensor are not written.
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int32_t c0, int32_t c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(tmap), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}

// ----------------------------------------------------------------------------------------------------------------
// wgmma: warpgroup MMA (four consecutive warps), both operands in shared memory, fp32 accumulators in registers
// ----------------------------------------------------------------------------------------------------------------
// accumulator registers written by other instructions -> visible to the following wgmma.mma_async
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed groups of this thread are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// per-warp register budget (every warp of a warpgroup must request the same count; multiples of 8 in [24, 256]).
// An increase waits until other warps of the CTA have released enough registers with a decrease.
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// D[64 x N] += A[64 x 16] * B[N x 16]^T, bf16 inputs (both K-major), fp32 accumulation.  Thread t of the warpgroup
// holds, per 8-column group j, d[4j + 0..1] = row 16*(t/32) + (t%32)/4, columns 8j + 2*(t%4) + {0, 1}, and d[4j + 2..3]
// = the same columns of row + 8.
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(1));
}
// the same fragment layout with 32 eight-column groups: d[4j + 0..3] for columns 8j .. 8j + 7 (j < 32)
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[128], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(1));
}
__device__ __forceinline__ void wgmma_m64n64k16_bf16(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// Shared-memory matrix descriptor (PTX ISA "Matrix Descriptor Format" for wgmma) for a K-major bf16 operand tile
// stored as rows of 128 bytes (64 bf16) with the 128-byte swizzle TMA writes (CU_TENSOR_MAP_SWIZZLE_128B):
//   bits  0-13  start address >> 4            bits 16-29  leading-dim byte offset >> 4 (unused for swizzled K-major)
//   bits 32-45  stride-dim byte offset >> 4 = 1024 B (8 rows x 128 B swizzle atom) >> 4
//   bits 62-63  layout: 1 = SWIZZLE_128B
// Advancing K by 16 elements inside the swizzle row adds 32 bytes (2 in the address field).
__device__ __forceinline__ uint64_t gmma_smem_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
    d |= static_cast<uint64_t>(1) << 16;
    d |= static_cast<uint64_t>(1024u >> 4) << 32;
    d |= static_cast<uint64_t>(1) << 62;
    return d;
}

// ----------------------------------------------------------------------------------------------------------------
// small numeric helpers
// ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ex2_approx_ftz(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// the reference's __expf under --use_fast_math: ex2.approx.ftz(x * log2(e))  (moe/gate.cuh:580-583)
__device__ __forceinline__ float fast_expf(float x) { return ex2_approx_ftz(x * 1.4426950408889634f); }

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);  // RNE, like cutlass::NumericConverter
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float bf16_bits_to_f32(uint32_t bits16) { return __uint_as_float(bits16 << 16); }
// a ^ b that the compiler cannot hoist or fold into precomputed values (keeps swizzled smem addresses out of registers
// across loops)
__device__ __forceinline__ uint32_t xor_u32(uint32_t a, uint32_t b) {
    uint32_t r;
    asm volatile("xor.b32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ float rne_bf16(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

}  // namespace fm
