// Peer-write bandwidth probe (2 GPUs, one process): how fast can SM-side code push rows into another GPU's memory over
// NVLink, by method and transfer size?  Feeds the dispatch design (DESIGN.md section 4, item 3).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o scripts/bin/peer_bw_probe scripts/peer_bw_probe.cu
//   scripts/bin/peer_bw_probe            (needs >= 2 GPUs with peer access)
// Methods: bulk = cp.async.bulk shared -> peer global of `chunk` bytes per operation (one issuing lane per operation, 32
// lanes of one warp per CTA, everything in flight, like the dispatch's remote mover); st = 16-byte st.global from all
// threads (coalesced 512 B per warp instruction); red = red.global.add.noftz.bf16x2 x4 (the return path's operation).
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__global__ void __launch_bounds__(256, 1) k_bulk(uint8_t* dst, size_t bytes_per_cta, int chunk, int row_stride_chunks) {
    extern __shared__ __align__(128) uint8_t sm[];
    // fill the staging (content irrelevant)
    for (int i = threadIdx.x * 16; i < 32 * 1024; i += blockDim.x * 16) *reinterpret_cast<uint4*>(sm + i) = make_uint4(1, 2, 3, 4);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (threadIdx.x < 32) {
        const size_t n = bytes_per_cta / chunk;
        uint8_t* base = dst + (size_t)blockIdx.x * bytes_per_cta * row_stride_chunks;
        for (size_t i = threadIdx.x; i < n; i += 32) {
            const uint32_t src = (uint32_t)__cvta_generic_to_shared(sm + ((i * chunk) & (32 * 1024 - 1) & ~(size_t)(chunk - 1)));
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(base + i * (size_t)chunk * row_stride_chunks), "r"(src), "r"(chunk) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
}

__global__ void __launch_bounds__(256, 1) k_st(uint4* dst, size_t vec_per_cta, int warps_active) {
    if ((int)(threadIdx.x >> 5) >= warps_active) return;
    uint4* base = dst + (size_t)blockIdx.x * vec_per_cta;
    const int nt = warps_active * 32;
    const uint4 v = make_uint4(threadIdx.x, 2, 3, 4);
    for (size_t i = threadIdx.x; i < vec_per_cta; i += nt)
        asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(base + i), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__global__ void __launch_bounds__(256, 1) k_red(uint4* dst, size_t vec_per_cta, int warps_active) {
    if ((int)(threadIdx.x >> 5) >= warps_active) return;
    uint4* base = dst + (size_t)blockIdx.x * vec_per_cta;
    const int nt = warps_active * 32;
    const uint32_t one = 0x3f803f80u;
    for (size_t i = threadIdx.x; i < vec_per_cta; i += nt)
        asm volatile("red.global.add.noftz.v4.bf16x2 [%0], {%1, %2, %3, %4};" ::"l"(base + i), "r"(one), "r"(one), "r"(one), "r"(one) : "memory");
}

struct Side { int dev; cudaStream_t st; cudaEvent_t e0, e1; uint8_t* buf; };

int main() {
    int nd = 0;
    CK(cudaGetDeviceCount(&nd));
    if (nd < 2) { printf("needs 2 GPUs\n"); return 0; }
    const size_t total = 64u << 20;   // bytes per direction per launch
    Side s[2];
    for (int d = 0; d < 2; ++d) {
        s[d].dev = d;
        CK(cudaSetDevice(d));
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, d, 1 - d));
        if (!can) { printf("no peer access\n"); return 0; }
        CK(cudaDeviceEnablePeerAccess(1 - d, 0));
        CK(cudaStreamCreate(&s[d].st));
        CK(cudaEventCreate(&s[d].e0));
        CK(cudaEventCreate(&s[d].e1));
        CK(cudaMalloc(&s[d].buf, total * 2));
        CK(cudaMemset(s[d].buf, 0, total * 2));
        CK(cudaFuncSetAttribute(k_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, 32 * 1024));
    }
    int G = 0;   // one CTA per SM
    CK(cudaDeviceGetAttribute(&G, cudaDevAttrMultiProcessorCount, 0));
    const int iters = 10;
    auto run = [&](const char* name, int dirs, auto launch) {
        // dirs = 1: GPU 0 writes to GPU 1; dirs = 2: both write to each other at the same time
        float ms[2] = {0, 0};
        size_t sent = 0;
        for (int rep = 0; rep < 2; ++rep) {   // rep 0 = warm-up
            for (int d = 0; d < dirs; ++d) {
                CK(cudaSetDevice(d));
                CK(cudaEventRecord(s[d].e0, s[d].st));
                for (int it = 0; it < iters; ++it) sent = launch(d, s[1 - d].buf, s[d].st);
                CK(cudaEventRecord(s[d].e1, s[d].st));
            }
            for (int d = 0; d < dirs; ++d) {
                CK(cudaSetDevice(d));
                CK(cudaStreamSynchronize(s[d].st));
                CK(cudaEventElapsedTime(&ms[d], s[d].e0, s[d].e1));
            }
        }
        const double gbs0 = (double)sent * iters / (ms[0] * 1e-3) / 1e9;
        if (dirs == 2) printf("%-44s bidir  %7.1f / %7.1f GB/s per direction (%.1f us per launch of %.1f MB)\n", name, gbs0, (double)sent * iters / (ms[1] * 1e-3) / 1e9, ms[0] * 1e3 / iters, sent / 1e6);
        else printf("%-44s unidir %7.1f GB/s (%.1f us per launch of %.1f MB)\n", name, gbs0, ms[0] * 1e3 / iters, sent / 1e6);
        fflush(stdout);
    };
    char name[128];
    for (int dirs = 1; dirs <= 2; ++dirs) {
        for (int chunk : {512, 2048, 4096, 8192, 16384, 32768}) {
            snprintf(name, sizeof name, "bulk store %5d B, contiguous", chunk);
            run(name, dirs, [&](int, uint8_t* dst, cudaStream_t st) { const size_t b = total / G / 32768 * 32768; k_bulk<<<G, 256, 32 * 1024, st>>>(dst, b, chunk, 1); return b * G; });
        }
        // rows scattered with a stride of 2 chunks (like rows of different packets)
        snprintf(name, sizeof name, "bulk store  2048 B, stride 4096");
        run(name, dirs, [&](int, uint8_t* dst, cudaStream_t st) { const size_t b = total / G / 32768 * 32768; k_bulk<<<G, 256, 32 * 1024, st>>>(dst, b, 2048, 2); return b * G; });
        for (int w : {1, 2, 4, 8}) {
            snprintf(name, sizeof name, "st.global.v4, %d warps per CTA", w);
            run(name, dirs, [&](int, uint8_t* dst, cudaStream_t st) { const size_t v = total / G / 16; k_st<<<G, 256, 0, st>>>(reinterpret_cast<uint4*>(dst), v, w); return v * 16 * G; });
        }
        for (int w : {4, 8}) {
            snprintf(name, sizeof name, "red.add.v4.bf16x2, %d warps per CTA", w);
            run(name, dirs, [&](int, uint8_t* dst, cudaStream_t st) { const size_t v = total / G / 16; k_red<<<G, 256, 0, st>>>(reinterpret_cast<uint4*>(dst), v, w); return v * 16 * G; });
        }
        // fewer CTAs: is the limit per SM or per link?
        for (int g : {16, 37, 74}) {
            snprintf(name, sizeof name, "bulk store 2048 B, %d CTAs", g);
            run(name, dirs, [&](int, uint8_t* dst, cudaStream_t st) { const size_t b = total / g / 32768 * 32768; k_bulk<<<g, 256, 32 * 1024, st>>>(dst, b, 2048, 1); return b * g; });
        }
    }
    // small-transfer regime of the kernel: 8.4 MB per direction in one launch (launch overhead included)
    {
        const size_t small = 8u << 20;
        for (int dirs = 1; dirs <= 2; ++dirs) {
            float ms[2];
            for (int rep = 0; rep < 3; ++rep) {
                for (int d = 0; d < dirs; ++d) {
                    CK(cudaSetDevice(d));
                    CK(cudaEventRecord(s[d].e0, s[d].st));
                    k_bulk<<<G, 256, 32 * 1024, s[d].st>>>(s[1 - d].buf, small / G / 2048 * 2048, 2048, 1);
                    CK(cudaEventRecord(s[d].e1, s[d].st));
                }
                for (int d = 0; d < dirs; ++d) { CK(cudaSetDevice(d)); CK(cudaStreamSynchronize(s[d].st)); CK(cudaEventElapsedTime(&ms[d], s[d].e0, s[d].e1)); }
            }
            printf("one launch, 8 MiB per direction, 2 KiB bulk stores, dirs=%d: %.1f us (%.1f GB/s incl. launch)\n", dirs, ms[0] * 1e3, small / (ms[0] * 1e-3) / 1e9);
        }
    }
    // reference: cudaMemcpyPeerAsync
    {
        CK(cudaSetDevice(0));
        float ms;
        for (int rep = 0; rep < 2; ++rep) {
            CK(cudaEventRecord(s[0].e0, s[0].st));
            for (int it = 0; it < iters; ++it) CK(cudaMemcpyPeerAsync(s[1].buf, 1, s[0].buf + total, 0, total, s[0].st));
            CK(cudaEventRecord(s[0].e1, s[0].st));
            CK(cudaStreamSynchronize(s[0].st));
            CK(cudaEventElapsedTime(&ms, s[0].e0, s[0].e1));
        }
        printf("cudaMemcpyPeerAsync 64 MiB: %.1f GB/s\n", (double)total * iters / (ms * 1e-3) / 1e9);
    }
    return 0;
}
