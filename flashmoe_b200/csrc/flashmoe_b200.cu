// flashmoe_b200.cu -- host runtime + C-ABI (include/flashmoe_b200.h) around the fused sm_90a kernel.
//
// Replaces the used slice of the reference's host runtime: bootstrap.cuh:278-512 (symmetric heap + bookkeeping
// allocation, peer pointer tables), moe.cuh:146-205 (launch) and python_bindings.cu:17-151 (argument checks) --
// without NVSHMEM (peer mapping is CUDA IPC or caller-provided pointers), without per-call weight copies
// (python_bindings.cu:76-120 re-uploads every weight on every call) and without exit() on errors.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "fm_kernel.cuh"

// ---- compile-time configuration surface: csrc/flashmoe_config.json -> -DFM_CFG_* (build script) -------------
#ifndef FM_CFG_CAPACITY_FACTOR
#define FM_CFG_CAPACITY_FACTOR 1
#define FM_CFG_DROP_TOKENS 1
#define FM_CFG_EXPERT_TOP_K 2
#define FM_CFG_GLOBAL_BATCH 256
#define FM_CFG_IS_TRAINING 0
#define FM_CFG_HIDDEN_ACT 0
#define FM_CFG_HIDDEN_SIZE 1024
#define FM_CFG_INTERMEDIATE_SIZE 4096
#define FM_CFG_MINI_BATCH 1
#define FM_CFG_MOE_FREQUENCY 1
#define FM_CFG_NUM_EXPERTS 8
#define FM_CFG_NUM_LAYERS 1
#define FM_CFG_SEQUENCE_LEN 4096
#define FM_CFG_TORCH_DTYPE 2
#define FM_CFG_VOCAB_SIZE 32000
#endif

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define FM_CUDA(expr)                                                                                         \
    do {                                                                                                      \
        cudaError_t _e = (expr);                                                                              \
        if (_e != cudaSuccess)                                                                                \
            return fail(FM_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

// A tensor map and the base and shape it was encoded for (its box is fixed per cache).
struct TmapCache {
    const void* base = nullptr;
    uint64_t rows = 0, cols = 0;
    CUtensorMap map = {};
};

// 2-D row-major bf16 tensor [rows, cols], tile box [box_rows, 64 cols], 128-byte swizzle (matches the wgmma smem
// descriptors built in fm_ptx.cuh), out-of-bounds elements read as zero.  Re-encoded only when the base or the shape
// differs from the cached map's; a failed encode leaves the cache as it was.
int cached_tmap(TmapCache* tc, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    if (tc->base == base && tc->rows == rows && tc->cols == cols) return FM_OK;
    EncodeTiledFn fn = get_encode_fn();
    if (fn == nullptr) return fail(FM_ECUDA, "cuTensorMapEncodeTiled entry point not available");
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {cols * 2};
    const cuuint32_t box[2] = {(cuuint32_t)fm::BLOCK_K, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    CUtensorMap m;
    CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(FM_ECUDA, "cuTensorMapEncodeTiled failed with CUresult %d (base=%p rows=%llu cols=%llu)", (int)r,
                    base, (unsigned long long)rows, (unsigned long long)cols);
    *tc = {base, rows, cols, m};
    return FM_OK;
}

}  // namespace

struct fm_ctx {
    fm_config_t cfg;
    fm_dims_t d;
    int device = 0;
    int grid = 0;
    int tpc = 0;
    int TN1 = 0, num_pkts = 0, num_blocks = 0;
    int dbg_flags = 0;
    // in-kernel waits give up after this long (fm_set_timeout_ms): generous by default so that ordinary rank skew (a peer
    // still loading data, compiling, paused in a debugger) is not turned into a trap -- see fm_ptx.cuh SpinGuard
    unsigned long long timeout_ns = 120ull * 1000ull * 1000ull * 1000ull;
    uint64_t launches = 0;   // launches issued through the API (graph replays are not counted; fm_last_launch counts them)
    // device buffers
    int* topk_idx = nullptr;
    __nv_bfloat16* topk_w = nullptr;
    float* mcw = nullptr;
    int* slot = nullptr;
    int* counts = nullptr;
    __nv_bfloat16* gate_out = nullptr;
    int* chunk_counts = nullptr;
    // [0] unused, [1] claim, [2..3] grid barrier (u64), [4..5] launch counter (u64), [6] token count of the last launch,
    // [7] epoch of the last routed launch that reported a bad expert index (FmParams::status_word)
    unsigned int* ctrl = nullptr;
    unsigned int* g0_done = nullptr;
    unsigned int* g1_done = nullptr;
    int* recv_cnt = nullptr;
    fm::TileBlock* blocks = nullptr;
    __nv_bfloat16* hidden = nullptr;
    // host-buffer path (fm_host_submit / fm_host_wait): FM_HOST_SLOTS staging pairs, three streams, so the H2D copy of
    // step i+1 and the D2H copy of step i-1 run under the kernel of step i (PCIe is full duplex; steps are independent)
    __nv_bfloat16* x_stage[FM_HOST_SLOTS] = {};
    __nv_bfloat16* out_stage[FM_HOST_SLOTS] = {};
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t ev_h2d[FM_HOST_SLOTS] = {}, ev_kernel[FM_HOST_SLOTS] = {}, ev_d2h[FM_HOST_SLOTS] = {};
    bool host_ready = false;
    uint64_t host_submitted = 0, host_waited = 0;
    // symmetric slab
    void* symm = nullptr;
    bool symm_external = false;
    size_t symm_bytes = 0, off_recv_x = 0, off_ret_y = 0, off_recv_flag = 0, off_ret_flag = 0;
    size_t off_recv_meta = 0, off_out_acc = 0, off_done_flag = 0, off_recv_rows = 0;
    bool fused = false;   // GEMM1 epilogue adds straight into the source rank's output (no return buffer / gather)
    bool dense = false;   // E == 1: GEMM0 reads x in place, no router GEMV, no dispatch copy (reference fffn.cuh:31-167)
    float* aux = nullptr; // is_training: [2][2E+1] {gML, gMeC, loss} by epoch parity
    bool tc_gate = false;               // router logits on the tensor cores (E <= 256)
    unsigned int* pkt_done = nullptr;
    void* peer_base[FM_MAX_WORLD] = {};
    bool peer_opened[FM_MAX_WORLD] = {};
    bool attached = false;
    fm::DebugRecord* dbg_host = nullptr;
    fm::DebugRecord* dbg_dev = nullptr;
    unsigned long long* trace = nullptr;
    bool trace_on = false;
    bool weight_on_input = false;   // fm_set_weight_on_input (caller and gated routes)
    TmapCache tm[fm::NUM_TMAPS];   // FmParams::tm (fm_symm_use_external moves recv_x's base)
    // shared expert (fm_shared_reserve): staging h_s [S, shared_max] and y_s [S, H], row-block counters [S / 128]
    int shared_max = 0;
    int shared_ps = 0;   // Ps of the last launch enqueued (or captured) with a shared expert: h_s's row stride
    __nv_bfloat16* h_s = nullptr;
    __nv_bfloat16* y_s = nullptr;
    unsigned int* s0_done = nullptr;
    unsigned int* s1_done = nullptr;
};

namespace {

// expert capacity of n tokens in token-expert pairs per (source rank, expert) packet (reference types.cuh:497)
long long expert_capacity(const fm_config_t& c, long long n) {
    return (c.drop_tokens ? (n + c.num_experts - 1) / c.num_experts : n) * c.capacity_factor * c.expert_top_k;
}

int validate_config(const fm_config_t& c, int world, fm_dims_t* d) {
    if (c.torch_dtype != 2) return fail(FM_EINVAL, "torch_dtype=%d: this build computes in bf16 only (2)", c.torch_dtype);
    if (c.is_training != 0 && c.is_training != 1) return fail(FM_EINVAL, "is_training must be 0 or 1");
    if (c.hidden_act < 0 || c.hidden_act > 2)
        return fail(FM_EINVAL, "hidden_act must be 0 (relu), 1 (gelu) or 2 (swiglu)");
    if (c.drop_tokens != 0 && c.drop_tokens != 1) return fail(FM_EINVAL, "drop_tokens must be 0 or 1");
    if (c.capacity_factor < 1) return fail(FM_EINVAL, "capacity_factor must be >= 1");
    if (c.hidden_size <= 0 || c.hidden_size % 64) return fail(FM_EINVAL, "hidden_size must be a positive multiple of 64");
    if (c.intermediate_size <= 0 || c.intermediate_size % 64)
        return fail(FM_EINVAL, "intermediate_size must be a positive multiple of 64");
    if (c.hidden_size > 32768) return fail(FM_EINVAL, "hidden_size > 32768 is not supported (row staging)");
    if (c.mini_batch < 1 || c.sequence_len < 1) return fail(FM_EINVAL, "mini_batch and sequence_len must be >= 1");
    const long long S = (long long)c.sequence_len * c.mini_batch;
    if (S % 128) return fail(FM_EINVAL, "S = sequence_len*mini_batch = %lld must be a multiple of 128", S);
    if (S > (1ll << 24)) return fail(FM_EINVAL, "S = %lld too large", S);
    if (c.num_experts < 1 || c.num_experts > fm::MAX_EXPERTS)
        return fail(FM_EINVAL, "num_experts must be in [1, %d]", fm::MAX_EXPERTS);
    if (c.expert_top_k < 1 || c.expert_top_k > c.num_experts || c.expert_top_k > 8)
        return fail(FM_EINVAL, "expert_top_k must be in [1, min(num_experts, 8)]");
    if (world < 1 || world > FM_MAX_WORLD) return fail(FM_EINVAL, "world size %d not in [1, %d]", world, FM_MAX_WORLD);
    if (c.num_experts % world) return fail(FM_EINVAL, "num_experts=%d not divisible by world=%d", c.num_experts, world);
    d->S = (int)S;
    d->H = c.hidden_size;
    d->E = c.num_experts;
    d->P = c.intermediate_size;
    d->PX = ceil_div(c.num_experts, 64) * 64;
    d->element_size = 2;
    d->k = c.expert_top_k;
    const long long ec = expert_capacity(c, S);
    if (ec > (1ll << 24)) return fail(FM_EINVAL, "expert capacity %lld too large", ec);
    d->EC = (int)ec;
    d->pEC = ceil_div(d->EC, 128) * 128;
    d->TCM = d->pEC / 128;
    d->world = world;
    d->num_local_experts = c.num_experts / world;
    return FM_OK;
}

template <typename T>
int dev_alloc(T** p, size_t count, bool zero = true) {
    void* q = nullptr;
    const size_t bytes = count * sizeof(T);
    cudaError_t e = cudaMalloc(&q, bytes ? bytes : 16);
    if (e != cudaSuccess) return fail(FM_ENOMEM, "cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
    if (zero) {
        e = cudaMemset(q, 0, bytes ? bytes : 16);
        if (e != cudaSuccess) return fail(FM_ECUDA, "cudaMemset failed: %s", cudaGetErrorString(e));
    }
    *p = static_cast<T*>(q);
    return FM_OK;
}

void set_peer_pointers(const fm_ctx* c, fm::FmParams& p) {
    for (int r = 0; r < c->d.world; ++r) {
        char* b = static_cast<char*>(c->peer_base[r]);
        p.peer_recv_x[r] = reinterpret_cast<__nv_bfloat16*>(b + c->off_recv_x);
        p.peer_ret_y[r] = reinterpret_cast<__nv_bfloat16*>(b + c->off_ret_y);
        p.peer_recv_flag[r] = reinterpret_cast<unsigned long long*>(b + c->off_recv_flag);
        p.peer_recv_rows[r] = reinterpret_cast<unsigned int*>(b + c->off_recv_rows);
        p.peer_ret_flag[r] = reinterpret_cast<unsigned long long*>(b + c->off_ret_flag);
        p.peer_recv_meta[r] = reinterpret_cast<uint4*>(b + c->off_recv_meta);
        p.peer_done_flag[r] = reinterpret_cast<unsigned long long*>(b + c->off_done_flag);
        p.peer_out_acc[r] = reinterpret_cast<__nv_bfloat16*>(b + c->off_out_acc);
    }
}

int check_kernel_status(fm_ctx* c) {
    if (c->dbg_host != nullptr && c->dbg_host->code == fm::FM_STATUS_BAD_COUNT) {
        // not a fault: reported once, then the record is cleared and the context stays usable
        const int n = (int)c->dbg_host->info0, S = (int)c->dbg_host->info1;
        memset(c->dbg_host, 0, sizeof(fm::DebugRecord));
        return fail(FM_EINVAL, "device token count n_tokens = %d not in [0, S = %d]: that launch ran on 0 tokens", n, S);
    }
    if (c->dbg_host != nullptr && c->dbg_host->code == fm::FM_STATUS_BAD_EXPERT) {   // (not a fault either)
        const int t = (int)c->dbg_host->info0, j = (int)c->dbg_host->info1, e = (int)c->dbg_host->info2;
        memset(c->dbg_host, 0, sizeof(fm::DebugRecord));
        return fail(FM_EINVAL, "topk_idx[%d, %d] = %d not in [-1, E = %d): a routed launch treated that pick as -1", t, j, e,
                    c->d.E);
    }
    if (c->dbg_host != nullptr && c->dbg_host->code == fm::FM_TRAP_MBAR) {
        const fm::DebugRecord r = *c->dbg_host;
        const fm::MbarName b = fm::mbar_name((int)r.info0);
        return fail(FM_EKERNEL,
                    "kernel wait timed out on mbarrier %s[%d], parity %u (block %u, warp %u): waited %.1f ms (rank %d, "
                    "launch %llu)",
                    b.group != nullptr ? b.group : "unknown", b.index, r.info1, r.block, r.thread / 32,
                    (double)r.waited_ns * 1e-6, c->d.rank, (unsigned long long)c->launches);
    }
    if (c->dbg_host != nullptr && c->dbg_host->code != 0) {
        static const char* names[] = {"none", "mbarrier", "(unused)", "(unused)", "(unused)", "(unused)", "(unused)",
                                      "grid barrier", "dispatch flag (packet never arrived)", "GEMM0 row-block counter",
                                      "return flag (expert output never arrived)",
                                      "dispatch row acknowledgement (rows of a packet never arrived)"};
        const fm::DebugRecord r = *c->dbg_host;
        const char* nm = r.code < sizeof(names) / sizeof(names[0]) ? names[r.code] : "unknown";
        return fail(FM_EKERNEL,
                    "kernel wait timed out on %s: block %u thread %u info=(%u,%u,%u) waited %.1f ms (rank %d, launch %llu)",
                    nm, r.block, r.thread, r.info0, r.info1, r.info2, (double)r.waited_ns * 1e-6, c->d.rank,
                    (unsigned long long)c->launches);
    }
    return FM_OK;
}

// What a forward entry point received.  n_tok is the host count; with n_dev the kernel reads the count from *n_dev when
// it starts, and n_tok is then S (the rows of x, out and the routing arrays).  A routed call (fm::ROUTE_CALLER) has
// topk_idx / topk_w [n, k] and no gate weights; a gated one (ROUTE_GATED) has the rule `router` and score_bias [E].
struct ForwardCall {
    const void* x;
    int n_tok;
    const int32_t* n_dev;
    const void *gate_w, *expert_w, *bias_up, *bias_down;
    void *out, *stream;   // stream: a cudaStream_t
    bool count_on_device = false;   // fm_moe_forward_tokens_dev: the count exists only in device memory, n_dev is required
    int route = fm::ROUTE_ROUTER;
    const int32_t* topk_idx = nullptr;
    const float* topk_w = nullptr;
    const fm_router_t* router = nullptr;
    const float* score_bias = nullptr;
    bool with_shared = false;   // fm_moe_forward_shared: `shared` is required
    const fm_shared_expert_t* shared = nullptr;
};

// The conditions on a gated call's rule that the header lists (flashmoe_b200.router.RouterSpec mirrors them).
int check_router(const fm_dims_t& d, const fm_router_t& r) {
    const int E = d.E;
    if (r.scoring != 0 && r.scoring != 1)
        return fail(FM_EINVAL, "router.scoring = %d: 0 (softmax) or 1 (sigmoid)", r.scoring);
    if (r.n_group < 1 || r.n_group > fm::MAX_GROUPS || E % r.n_group != 0)
        return fail(FM_EINVAL, "router.n_group = %d: must be in [1, %d] and divide E = %d", r.n_group, fm::MAX_GROUPS, E);
    if (r.topk_group < 1 || r.topk_group > r.n_group)
        return fail(FM_EINVAL, "router.topk_group = %d not in [1, n_group = %d]", r.topk_group, r.n_group);
    if (r.n_group > 1 && ((r.group_top != 1 && r.group_top != 2) || r.group_top > E / r.n_group))
        return fail(FM_EINVAL, "router.group_top = %d: 1 or 2, and at most the group size E / n_group = %d",
                    r.group_top, E / r.n_group);
    if (d.k > r.topk_group * (E / r.n_group))
        return fail(FM_EINVAL, "k = %d picks need at least k experts in the topk_group = %d kept groups of %d", d.k,
                    r.topk_group, E / r.n_group);
    if (r.renormalize != 0 && r.renormalize != 1)
        return fail(FM_EINVAL, "router.renormalize = %d: 0 or 1", r.renormalize);
    if (!std::isfinite(r.scale) || !(r.scale > 0.0f))
        return fail(FM_EINVAL, "router.scale = %g: must be finite and > 0", (double)r.scale);
    return FM_OK;
}

// Every argument check of a forward call; issues no CUDA call.  The pointers only some entry points take are checked
// before any field of the context is read.
int check_call(const fm_ctx* c, const ForwardCall& f) {
    if (f.count_on_device && f.n_dev == nullptr) return fail(FM_EINVAL, "n_tokens_dev must point to an int32");
    if (f.route == fm::ROUTE_GATED && f.router == nullptr) return fail(FM_EINVAL, "router must point to an fm_router_t");
    if (f.with_shared && f.shared == nullptr) return fail(FM_EINVAL, "shared must point to an fm_shared_expert_t");
    // fm_moe_forward_shared picks the route from gate_w and router: the other route's arguments must be absent
    if (f.route != fm::ROUTE_CALLER && (f.topk_idx != nullptr || f.topk_w != nullptr))
        return fail(FM_EINVAL, "topk_idx / topk_w are the caller's routing: gate_w must be NULL with them");
    if (f.route == fm::ROUTE_CALLER && f.router != nullptr)
        return fail(FM_EINVAL, "router needs gate_w (a rule applies to the router's logits)");
    if (f.route != fm::ROUTE_GATED && f.score_bias != nullptr)
        return fail(FM_EINVAL, "score_bias needs gate_w and router (it steers a rule's selection)");
    const fm_dims_t& d = c->d;
    if (f.n_tok < 0 || f.n_tok > d.S) return fail(FM_EINVAL, "n_tokens = %d not in [0, S = %d]", f.n_tok, d.S);
    if (f.n_dev != nullptr && f.n_tok != d.S)
        return fail(FM_EINVAL, "with n_tokens_dev, n_tokens must be S = %d (the rows of x, out and the routing arrays); "
                               "got %d", d.S, f.n_tok);
    // both replace the router's softmax top-k: an E = 1 context has no router, and the auxiliary loss of a training one
    // is defined on the router's probabilities
    if (f.route != fm::ROUTE_ROUTER && (d.E == 1 || c->aux != nullptr))
        return fail(FM_EINVAL, "%s needs num_experts > 1 and is_training = 0; this context has E = %d, is_training = %d",
                    f.route == fm::ROUTE_CALLER ? "caller routing" : "a gated call", d.E, c->cfg.is_training);
    int rc;
    if (f.route == fm::ROUTE_GATED && (rc = check_router(d, *f.router))) return rc;
    const fm_shared_expert_t none = {};
    const fm_shared_expert_t& sh = f.shared != nullptr ? *f.shared : none;
    if (f.with_shared) {
        if (d.E == 1)
            return fail(FM_EINVAL, "a shared expert needs num_experts > 1 (an E = 1 context is one dense expert already)");
        if (sh.inter <= 0 || sh.inter % 64)
            return fail(FM_EINVAL, "shared->inter = %d must be a positive multiple of 64", sh.inter);
        if (c->shared_max == 0)
            return fail(FM_ESTATE, "no shared-expert staging: call fm_shared_reserve on this context first");
        if (sh.inter > c->shared_max)
            return fail(FM_EINVAL, "shared->inter = %d is above the reserved %d (fm_shared_reserve)", sh.inter,
                        c->shared_max);
    }
    // Nothing reads the per-token rows of a call on no tokens.  TMA tensor maps, cp.async.bulk row copies and the
    // 16-byte vector accesses all need 16-byte aligned bases.
    const bool rows = f.n_tok > 0, routed = f.route == fm::ROUTE_CALLER;
    const struct { const void* ptr; const char* name; bool required; } args[] = {
        {f.x, "x", rows}, {f.gate_w, "gate_w", !routed}, {f.expert_w, "expert_w", true}, {f.bias_up, "bias_up", false},
        {f.bias_down, "bias_down", false}, {f.out, "out", rows}, {f.topk_idx, "topk_idx", routed && rows},
        {f.topk_w, "topk_w", routed && rows}, {f.score_bias, "score_bias", false},
        {sh.w, "shared->w", f.with_shared}, {sh.bias_up, "shared->bias_up", false},
        {sh.bias_down, "shared->bias_down", false}};
    for (const auto& a : args)
        if (a.required && a.ptr == nullptr) return fail(FM_EINVAL, "%s must be a non-null device pointer", a.name);
    for (const auto& a : args)
        if (reinterpret_cast<uintptr_t>(a.ptr) % 16)
            return fail(FM_EINVAL, "%s must be 16-byte aligned (got %p)", a.name, a.ptr);
    if (reinterpret_cast<uintptr_t>(f.n_dev) % alignof(int32_t))
        return fail(FM_EINVAL, "n_tokens_dev must be 4-byte aligned (got %p)", static_cast<const void*>(f.n_dev));
    if (!c->attached) return fail(FM_ESTATE, "peers not attached: call fm_symm_attach_ipc/ptrs before fm_moe_forward");
    return FM_OK;
}

// One forward of n tokens (0 <= n <= S): the call computes exactly what a context created for n tokens would --
// capacity EC(n), tokens per CTA ceil(n / grid) -- while every buffer keeps its create-time (maximum) size and stride.
// The kernel derives everything that depends on n and on the launch's place in the context's sequence of launches
// itself (fm_kernel.cuh, struct Launch), so the parameters built here are valid for every replay of a captured launch,
// and this function issues nothing that stream capture forbids.
int launch(fm_ctx* c, const ForwardCall& f) {
    int rc;
    if ((rc = check_call(c, f))) return rc;
    FM_CUDA(cudaSetDevice(c->device));
    const fm_dims_t& d = c->d;
    const int nLx = d.num_local_experts;
    // The maps over x have exactly n_tok rows (a box taller than that reads the missing rows as zero); with no tokens
    // nothing reads x, and no map over it is encoded.  GEMM0's A operand is x itself when dense (E == 1), otherwise the
    // rows dispatched into recv_x.
    const uint64_t n = (uint64_t)f.n_tok, pkt_rows = (uint64_t)c->num_pkts * d.pEC;
    const void* a0 = c->dense ? f.x : static_cast<const char*>(c->symm) + c->off_recv_x;
    const uint64_t a0_rows = c->dense ? n : pkt_rows;
    // router on tensor cores: x as [n_tok, H] in 32-row boxes, Wg_eff = the [H, E] tensor read flat as [E, H]
    // (python_bindings.cu:93-99, moe.cuh:107-109) in boxes of min(128, E rounded up to 64) rows; rows past E read as
    // zero.  A routed launch has no router maps.
    const bool gate_maps = c->tc_gate && f.route != fm::ROUTE_CALLER;
    const uint32_t e64 = (uint32_t)((d.E + 63) / 64 * 64);
    const fm_shared_expert_t* sh = f.shared;
    const uint64_t Ps = sh != nullptr ? (uint64_t)sh->inter : 0;
    const char* ws = sh != nullptr ? static_cast<const char*>(sh->w) : nullptr;
    // expert_weights [nLx, 2, P, H]: [i,0] is W_up [P,H]; [i,1] is the same P*H block viewed as W_down [H,P]
    // (python_bindings.cu:104-119).  One tensor map per GEMM over the whole tensor with a per-expert row stride
    // of 2*P (resp. 2*H) rows is not expressible in 2-D, so rows are addressed as [nLx*2*P, H] / [nLx*2*H, P]:
    // expert i's W_up starts at row i*2*P, its W_down at row (i*2+1)*H of the [.,P] view.  The shared expert's
    // w [2, Ps, H] is one such expert: W_up_s [Ps, H] and W_down_s [H, Ps].
    // SwiGLU (hidden_act 2): [nLx, 3, P, H] = W_gate, W_up, W_down per expert, so mats = 3 matrices per expert; GEMM0's
    // maps load 128-row boxes, a gate half and an up half per tile, and W_down is matrix 2.
    const bool glu = c->cfg.hidden_act == 2;
    const uint64_t mats = glu ? 3 : 2;
    const uint32_t box0 = glu ? fm::BLOCK_N / 2 : fm::BLOCK_N;
    struct MapSpec { const void* base; uint64_t rows, cols; uint32_t box_rows; bool needed; };
    const MapSpec maps[fm::NUM_TMAPS] = {
        {a0, a0_rows, (uint64_t)d.H, fm::BLOCK_M, a0_rows > 0},                            // TM_A0
        {f.expert_w, nLx * mats * d.P, (uint64_t)d.H, box0, true},                         // TM_B0
        {c->hidden, pkt_rows, (uint64_t)d.P, fm::BLOCK_M, true},                           // TM_A1
        {f.expert_w, nLx * mats * d.H, (uint64_t)d.P, fm::BLOCK_N, true},                  // TM_B1
        {f.x, n, (uint64_t)d.H, 32, gate_maps && n > 0},                                   // TM_GX
        {f.gate_w, (uint64_t)d.E, (uint64_t)d.H, std::min(128u, e64), gate_maps},          // TM_GW
        {f.x, n, (uint64_t)d.H, fm::BLOCK_M, sh != nullptr && n > 0},                      // TM_XS
        {ws, glu ? 3 * Ps : Ps, (uint64_t)d.H, box0, sh != nullptr},                       // TM_WS0
        {ws + (mats - 1) * Ps * d.H * 2, (uint64_t)d.H, Ps, fm::BLOCK_N, sh != nullptr},   // TM_WS1
        {c->h_s, (uint64_t)d.S, Ps, fm::BLOCK_M, sh != nullptr},                           // TM_HS
    };

    fm::FmParams p;
    memset(&p, 0, sizeof(p));
    for (int i = 0; i < fm::NUM_TMAPS; ++i) {
        const MapSpec& m = maps[i];
        if (!m.needed) continue;
        if ((rc = cached_tmap(&c->tm[i], m.base, m.rows, m.cols, m.box_rows))) return rc;
        p.tm[i] = c->tm[i].map;
    }
    // the GEMMs' operands, fields in fm::GemmOp's order: {A map, B map, A rows per packet, B row of expert 0,
    // B rows per expert, k-blocks, output columns, column tiles, rows from a packet, bias per expert, done counters per
    // packet, destination, bias, done counters}.  SwiGLU: the bias is [gate; up] per expert, and a GEMM0 tile is
    // tile_cols = 128 columns of h from its gate rows and the up rows glu_rows below them (column tiles ceil(n / 128)).
    const int from_packet = c->dense ? 0 : 1, m = (int)mats;
    using bf16p = const __nv_bfloat16*;
    p.gemm[fm::GEMM_UP] = {fm::TM_A0, fm::TM_B0, d.pEC, 0, m * d.P, d.H / fm::BLOCK_K, d.P, ceil_div(d.P, fm::BLOCK_N),
                           from_packet, (m - 1) * d.P, d.TCM, 0, static_cast<bf16p>(f.bias_up), c->g0_done};
    if (glu) { p.gemm[fm::GEMM_UP].glu_rows = d.P; p.gemm[fm::GEMM_UP].tn = ceil_div(d.P, (int)box0); }
    p.gemm[fm::GEMM_DOWN] = {fm::TM_A1, fm::TM_B1, d.pEC, (m - 1) * d.H, m * d.H, d.P / fm::BLOCK_K, d.H, c->TN1,
                             from_packet, d.H, 0, c->fused ? fm::DEST_FUSED : fm::DEST_RETURN,
                             static_cast<bf16p>(f.bias_down), nullptr};
    if (sh != nullptr) {   // rows are the call's tokens
        p.shared = 1;
        p.y_s = c->y_s; p.s0_done = c->s0_done; p.s1_done = c->s1_done;
        const int ps = (int)Ps;
        p.gemm[fm::GEMM_S_UP] = {fm::TM_XS, fm::TM_WS0, 0, 0, 0, d.H / fm::BLOCK_K, ps, ceil_div(ps, fm::BLOCK_N), 0, 0,
                                 0, 0, static_cast<bf16p>(sh->bias_up), c->s0_done};
        if (glu) { p.gemm[fm::GEMM_S_UP].glu_rows = ps; p.gemm[fm::GEMM_S_UP].tn = ceil_div(ps, (int)box0); }
        p.gemm[fm::GEMM_S_DOWN] = {fm::TM_HS, fm::TM_WS1, 0, 0, 0, ps / fm::BLOCK_K, d.H, c->TN1, 0, 0, 0, fm::DEST_Y_S,
                                   static_cast<bf16p>(sh->bias_down), nullptr};
    }
    p.tc_gate = c->tc_gate ? 1 : 0;
    p.n_tokens = f.n_tok; p.n_tokens_dev = f.n_dev;
    p.H = d.H; p.P = d.P; p.E = d.E; p.k = d.k; p.W = d.world; p.rank = d.rank; p.nLx = nLx;
    p.pEC = d.pEC; p.TCM = d.TCM; p.act = c->cfg.hidden_act;
    p.TN1 = c->TN1; p.num_pkts = c->num_pkts; p.num_blocks = c->num_blocks;
    p.drop_tokens = c->cfg.drop_tokens; p.ec_mult = c->cfg.capacity_factor * d.k;   // EC(n), as expert_capacity
    p.dbg_flags = c->dbg_flags;
    p.timeout_ns = c->timeout_ns;
    p.launch_ctr = reinterpret_cast<unsigned long long*>(c->ctrl + 4);
    p.launch_tokens = reinterpret_cast<int*>(c->ctrl + 6);
    p.x = static_cast<const __nv_bfloat16*>(f.x);
    p.wg = static_cast<const __nv_bfloat16*>(f.gate_w);
    p.out = static_cast<__nv_bfloat16*>(f.out);
    p.topk_idx = c->topk_idx; p.topk_w = c->topk_w; p.mcw = c->mcw; p.slot = c->slot; p.counts = c->counts;
    p.gate_out = c->gate_out; p.chunk_counts = c->chunk_counts;
    p.claim = c->ctrl + 1;
    p.grid_bar = reinterpret_cast<unsigned long long*>(c->ctrl + 2);
    p.g0_done = c->g0_done; p.g1_done = c->g1_done; p.recv_cnt = c->recv_cnt; p.blocks = c->blocks;
    p.hidden = c->hidden;
    char* sb = static_cast<char*>(c->symm);
    p.recv_x = reinterpret_cast<__nv_bfloat16*>(sb + c->off_recv_x);
    p.ret_y = reinterpret_cast<__nv_bfloat16*>(sb + c->off_ret_y);
    p.recv_flag = reinterpret_cast<unsigned long long*>(sb + c->off_recv_flag);
    p.recv_rows = reinterpret_cast<unsigned int*>(sb + c->off_recv_rows);
    p.ret_flag = reinterpret_cast<unsigned long long*>(sb + c->off_ret_flag);
    set_peer_pointers(c, p);
    p.fused = c->fused ? 1 : 0;
    p.pkt_done = c->pkt_done;
    p.recv_meta = reinterpret_cast<uint4*>(sb + c->off_recv_meta);
    p.done_flag = reinterpret_cast<unsigned long long*>(sb + c->off_done_flag);
    // single rank: accumulate straight into the caller's tensor; otherwise into the peer-mapped accumulator
    p.out_acc = d.world == 1 ? p.out : reinterpret_cast<__nv_bfloat16*>(sb + c->off_out_acc);
    if (d.world == 1) p.peer_out_acc[0] = p.out;
    p.aux = c->aux;
    p.dense = c->dense ? 1 : 0;
    p.route = f.route;
    p.routed_idx = f.topk_idx;
    p.routed_w = f.topk_w;
    p.status_word = c->ctrl + 7;
    if (f.route == fm::ROUTE_GATED) {
        p.scoring = f.router->scoring; p.n_group = f.router->n_group; p.topk_group = f.router->topk_group;
        p.group_top = f.router->group_top; p.renormalize = f.router->renormalize; p.route_scale = f.router->scale;
        p.score_bias = f.score_bias;
    }
    p.dbg = c->dbg_dev;
    p.trace = c->trace_on ? c->trace : nullptr;
    p.weight_on_input = c->weight_on_input && f.route != fm::ROUTE_ROUTER ? 1 : 0;   // (the router route copies y unscaled)

    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3(c->grid);
    lc.blockDim = dim3(fm::NUM_THREADS);
    lc.dynamicSmemBytes = (size_t)fm::SMEM_BYTES;
    lc.stream = static_cast<cudaStream_t>(f.stream);
    // The persistent grid spins on flags, counters and one grid barrier, so every CTA must be resident: the launch is
    // cooperative (the driver then refuses to start it unless the whole grid fits, also next to other work on the GPU).
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeCooperative;
    attr.val.cooperative = 1;
    lc.attrs = &attr;
    lc.numAttrs = 1;
    FM_CUDA(cudaLaunchKernelEx(&lc, fm::fm_moe_forward_kernel, p));
    c->launches += 1;
    if (sh != nullptr) c->shared_ps = (int)Ps;
    return FM_OK;
}

// the device's launch record: launches run so far (replays included) and the token count of the last one.  Synchronises.
int read_launch_record(fm_ctx* c, uint64_t* launches, int32_t* n_tokens) {
    FM_CUDA(cudaSetDevice(c->device));
    FM_CUDA(cudaDeviceSynchronize());
    unsigned int w[3];
    FM_CUDA(cudaMemcpy(w, c->ctrl + 4, sizeof(w), cudaMemcpyDeviceToHost));
    if (launches != nullptr) *launches = (uint64_t)w[0] | ((uint64_t)w[1] << 32);
    if (n_tokens != nullptr) *n_tokens = (int32_t)w[2];
    return FM_OK;
}

}  // namespace

// =================================================================================================================
extern "C" {

FM_API const char* fm_last_error(void) { return g_err.c_str(); }
FM_API const char* fm_version(void) { return "flashmoe_b200 0.1.0 (sm_90a, wgmma/TMA)"; }

FM_API int fm_compiled_config(fm_config_t* out) {
    if (out == nullptr) return fail(FM_EINVAL, "null output");
    out->capacity_factor = FM_CFG_CAPACITY_FACTOR;
    out->drop_tokens = FM_CFG_DROP_TOKENS;
    out->expert_top_k = FM_CFG_EXPERT_TOP_K;
    out->global_batch = FM_CFG_GLOBAL_BATCH;
    out->is_training = FM_CFG_IS_TRAINING;
    out->hidden_act = FM_CFG_HIDDEN_ACT;
    out->hidden_size = FM_CFG_HIDDEN_SIZE;
    out->intermediate_size = FM_CFG_INTERMEDIATE_SIZE;
    out->mini_batch = FM_CFG_MINI_BATCH;
    out->moe_frequency = FM_CFG_MOE_FREQUENCY;
    out->num_experts = FM_CFG_NUM_EXPERTS;
    out->num_layers = FM_CFG_NUM_LAYERS;
    out->sequence_len = FM_CFG_SEQUENCE_LEN;
    out->torch_dtype = FM_CFG_TORCH_DTYPE;
    out->vocab_size = FM_CFG_VOCAB_SIZE;
    return FM_OK;
}

FM_API int fm_create(const fm_config_t* cfg, int rank, int world, int device, fm_ctx_t** out) {
    if (out == nullptr) return fail(FM_EINVAL, "null output");
    *out = nullptr;
    fm_config_t c;
    if (cfg != nullptr) c = *cfg;
    else fm_compiled_config(&c);
    fm_dims_t d;
    memset(&d, 0, sizeof(d));
    int rc = validate_config(c, world, &d);
    if (rc) return rc;
    if (rank < 0 || rank >= world) return fail(FM_EINVAL, "rank %d not in [0, %d)", rank, world);
    d.rank = rank;

    int ndev = 0;
    FM_CUDA(cudaGetDeviceCount(&ndev));
    if (device < 0 || device >= ndev) return fail(FM_EINVAL, "device %d not in [0, %d)", device, ndev);
    FM_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    FM_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(FM_ECUDA, "device %d is sm_%d%d; this library contains sm_90a code only (wgmma/TMA)", device,
                    prop.major, prop.minor);
    int coop = 0;
    FM_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
    if (!coop) return fail(FM_ECUDA, "device does not support cooperative launch");
    d.num_sms = prop.multiProcessorCount;
    d.smem_bytes = fm::SMEM_BYTES;
    d.grid = prop.multiProcessorCount;

    FM_CUDA(cudaFuncSetAttribute(reinterpret_cast<const void*>(&fm::fm_moe_forward_kernel),
                                 cudaFuncAttributeMaxDynamicSharedMemorySize, fm::SMEM_BYTES));
    int occ = 0;
    FM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fm::fm_moe_forward_kernel, fm::NUM_THREADS,
                                                          (size_t)fm::SMEM_BYTES));
    if (occ < 1) return fail(FM_ECUDA, "kernel does not fit on an SM (smem %d B)", fm::SMEM_BYTES);

    fm_ctx* ctx = new fm_ctx();
    ctx->cfg = c;
    ctx->d = d;
    ctx->device = device;
    // path choices (combine, dense E = 1, router, work order); environment overrides are for tests and experiments
    auto env_int = [](const char* name, int dflt) {
        const char* v = getenv(name);
        return (v != nullptr && *v) ? atoi(v) : dflt;
    };
    ctx->grid = d.num_sms;  // one persistent CTA per SM; all co-resident (spin waits + grid barrier)
    {
        // fused GEMM1 -> combine (REDG into the token's output row): only for k <= 2, where bf16 accumulation is
        // order-independent (0 + a exact, a + b commutative) and therefore bit-identical to the deterministic gather;
        // k > 2 keeps the gather so results do not depend on arrival order
        const char* f = getenv("FM_FUSED_COMBINE");
        ctx->fused = ((f != nullptr && *f) ? atoi(f) != 0 : true) && d.k <= 2;
        ctx->dense = d.E == 1 && world == 1 && env_int("FM_DENSE_E1", 1) != 0;
        // router logits by wgmma instead of the CUDA-core GEMV (2*S*H*E flops: 4.3 GFLOP per rank at E = 128,
        // d_model 2048, 8192 tokens); up to 256 experts, 128 per pass over d_model.  Default: from 17 experts up (at a
        // handful of experts the GEMV is latency-, not flop-bound).
        ctx->tc_gate = !ctx->dense && d.E <= 256 && env_int("FM_TC_GATE", d.E > 16 ? 1 : 0) != 0;
        ctx->d.grid = ctx->grid;
    }
    ctx->tpc = ceil_div(d.S, ctx->grid);
    if ((long long)ctx->tpc * d.k > fm::G_SEL_MAX) {
        delete ctx;
        return fail(FM_EINVAL, "tokens-per-CTA * k = %d exceeds the router scratch (%d)", ctx->tpc * d.k, fm::G_SEL_MAX);
    }
    const int nLx = d.num_local_experts;
    ctx->dbg_flags = env_int("FM_DBG_FLAGS", 0);
    ctx->TN1 = ceil_div(d.H, fm::BLOCK_N);
    ctx->num_pkts = world * nLx;

    // Work list.  Sources in the order own rank, rank+1, ... (local rows need no NVLink hop, so they are ready first).
    // A work item is one 128 x 256 output tile of one packet.  The table stores, per block, how many blocks of each GEMM
    // precede it; the kernel derives the block's first item from the call's row blocks per packet (fm::block_start).
    struct Unit { int pkt; bool local; };
    std::vector<Unit> units;
    for (int j = 0; j < world; ++j)
        for (int le = 0; le < nLx; ++le) units.push_back({((rank + j) % world) * nLx + le, j == 0});
    std::vector<fm::TileBlock> blocks;
    auto push = [&](int gemm, const Unit& u) { blocks.push_back({{}, gemm, u.pkt}); };
    // GEMM0: local sources first (their rows are acknowledged first), then rank+1, rank+2, ...  GEMM1: REMOTE sources
    // first, local last -- the outputs of remote packets cross NVLink as reductions and their done flags have a link round
    // trip ahead of them, so they should not be what every rank finishes with; the local packets' adds are cheap and
    // nobody but this rank waits for them.  FM_G1_LAG interleaves GEMM1 of a unit `lag` units after its GEMM0 instead.
    std::vector<Unit> g1_units;
    for (const Unit& u : units) if (!u.local) g1_units.push_back(u);
    for (const Unit& u : units) if (u.local) g1_units.push_back(u);
    // FM_G1_LAG: -1 (default) = the orders described here; n >= 1 = GEMM1 of a unit n units after its GEMM0.
    //   one rank:    all GEMM0, then all GEMM1;
    //   two ranks:   GEMM0 local, GEMM0 remote, GEMM1 remote, GEMM1 local (the remote rows land while the local packets
    //                run; the local adds, which nobody else waits for, come last);
    //   four+ ranks: GEMM0 local, GEMM1 local, then the remote units with GEMM1 one unit behind GEMM0 -- the local
    //                packets are the only work available until the remote rows have crossed NVLink, and starting the
    //                remote units' GEMM1 early spreads the return traffic (reductions over NVLink, which would otherwise
    //                pile up behind the last tiles) over the whole phase.
    const int lag = env_int("FM_G1_LAG", -1);
    if (lag >= 1 && lag < (int)units.size()) {
        for (size_t i = 0; i < units.size(); ++i) {
            push(0, units[i]);
            if ((int)i >= lag) push(1, units[i - lag]);
        }
        for (size_t i = units.size() - lag; i < units.size(); ++i) push(1, units[i]);
    } else if (world >= 4 && lag < 0) {
        std::vector<Unit> loc, rem;
        for (const Unit& u : units) (u.local ? loc : rem).push_back(u);
        for (const Unit& u : loc) push(0, u);
        for (const Unit& u : loc) push(1, u);
        // remote units grouped by source rank (nLx units per source): GEMM1 one source behind GEMM0
        const size_t per_src = (size_t)nLx;
        for (size_t g0 = 0; g0 < rem.size(); g0 += per_src) {
            for (size_t i = g0; i < std::min(g0 + per_src, rem.size()); ++i) push(0, rem[i]);
            if (g0 >= per_src)
                for (size_t i = g0 - per_src; i < g0; ++i) push(1, rem[i]);
        }
        for (size_t i = rem.size() >= per_src ? rem.size() - per_src : 0; i < rem.size(); ++i) push(1, rem[i]);
    } else {
        for (const Unit& u : units) push(0, u);
        for (const Unit& u : g1_units) push(1, u);
    }
    // The shared expert's blocks, empty in a launch without one.  Its GEMM0 comes first: it needs nothing but x, which is
    // in memory when the kernel starts, so it fills the time the routed packets' rows take to land.  Its GEMM1 follows
    // the leading local routed GEMM0 blocks: by then its h rows are complete, and it fills the time until the routed
    // GEMM1 dependencies resolve.
    size_t split = 0;
    while (split < blocks.size() && blocks[split].gemm == fm::GEMM_UP && blocks[split].pkt / nLx == rank) ++split;
    blocks.insert(blocks.begin() + split, {{}, fm::GEMM_S_DOWN, rank * nLx});
    blocks.insert(blocks.begin(), {{}, fm::GEMM_S_UP, rank * nLx});
    ctx->num_blocks = (int)blocks.size();
    blocks.push_back({{}, -1, 0});   // the sentinel: its block_start is the launch's item count
    int n_g[fm::NUM_GEMMS] = {};
    for (fm::TileBlock& b : blocks) {
        std::copy(n_g, n_g + fm::NUM_GEMMS, b.g);
        if (b.gemm >= 0) ++n_g[b.gemm];
    }

#define FM_TRY(expr)          \
    do {                      \
        rc = (expr);          \
        if (rc) {             \
            fm_destroy(ctx);  \
            return rc;        \
        }                     \
    } while (0)
#define FM_TRY_CUDA(expr)                                                                             \
    do {                                                                                              \
        cudaError_t _e = (expr);                                                                      \
        if (_e != cudaSuccess) {                                                                      \
            fm_destroy(ctx);                                                                          \
            return fail(FM_ECUDA, "%s failed: %s", #expr, cudaGetErrorString(_e));                    \
        }                                                                                             \
    } while (0)

    FM_TRY(dev_alloc(&ctx->topk_idx, (size_t)d.S * d.k));
    FM_TRY(dev_alloc(&ctx->topk_w, (size_t)d.S * d.k));
    FM_TRY(dev_alloc(&ctx->mcw, (size_t)d.S));
    FM_TRY(dev_alloc(&ctx->slot, (size_t)d.S * d.k));
    FM_TRY(dev_alloc(&ctx->counts, (size_t)d.E));
    FM_TRY(dev_alloc(&ctx->gate_out, (size_t)d.S * d.E));
    FM_TRY(dev_alloc(&ctx->chunk_counts, (size_t)ctx->grid * d.E));
    FM_TRY(dev_alloc(&ctx->ctrl, 8));
    FM_TRY(dev_alloc(&ctx->g0_done, (size_t)ctx->num_pkts * d.TCM));
    FM_TRY(dev_alloc(&ctx->g1_done, (size_t)ctx->num_pkts * d.TCM));
    FM_TRY(dev_alloc(&ctx->recv_cnt, (size_t)ctx->num_pkts));
    FM_TRY(dev_alloc(&ctx->pkt_done, (size_t)ctx->num_pkts));
    FM_TRY(dev_alloc(&ctx->blocks, blocks.size(), false));
    FM_TRY_CUDA(cudaMemcpy(ctx->blocks, blocks.data(), blocks.size() * sizeof(fm::TileBlock), cudaMemcpyHostToDevice));
    FM_TRY(dev_alloc(&ctx->hidden, (size_t)ctx->num_pkts * d.pEC * d.P));
    FM_TRY(dev_alloc(&ctx->trace, (size_t)ctx->grid * fm::TRACE_SLOTS));
    if (c.is_training) FM_TRY(dev_alloc(&ctx->aux, (size_t)2 * (2 * d.E + 1)));

    // symmetric slab: [recv_x | ret_y | recv_flag | ret_flag]  (reference heap + flags, bootstrap.cuh:348-362)
    size_t off = 0;
    // the return buffer + per-row-block return flags exist only on the gather-combine path (the fused path adds
    // straight into the token's output row)
    ctx->off_recv_x = off; off = align_up(off + (size_t)ctx->num_pkts * d.pEC * d.H * 2, 1024);
    ctx->off_ret_y = off;  off = align_up(off + (ctx->fused ? 0 : (size_t)d.E * d.pEC * d.H * 2), 1024);
    ctx->off_recv_flag = off; off = align_up(off + (size_t)ctx->num_pkts * 8, 1024);
    ctx->off_recv_rows = off; off = align_up(off + (size_t)2 * ctx->num_pkts * d.TCM * 4, 1024);
    ctx->off_ret_flag = off;  off = align_up(off + (ctx->fused ? 0 : (size_t)d.E * d.TCM * 8), 1024);
    ctx->off_recv_meta = off; off = align_up(off + (size_t)ctx->num_pkts * d.pEC * 16, 1024);
    ctx->off_done_flag = off; off = align_up(off + (size_t)d.E * 8, 1024);
    ctx->off_out_acc = off;   off = align_up(off + (world > 1 ? (size_t)d.S * d.H * 2 : 0), 1024);
    ctx->symm_bytes = off;
    {
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, ctx->symm_bytes);
        if (e != cudaSuccess) {
            fm_destroy(ctx);
            return fail(FM_ENOMEM, "cudaMalloc(symmetric slab, %zu bytes) failed: %s", ctx->symm_bytes, cudaGetErrorString(e));
        }
        ctx->symm = q;
        FM_TRY_CUDA(cudaMemset(q, 0, ctx->symm_bytes));
    }
    FM_TRY_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&ctx->dbg_host), sizeof(fm::DebugRecord), cudaHostAllocMapped));
    memset(ctx->dbg_host, 0, sizeof(fm::DebugRecord));
    FM_TRY_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&ctx->dbg_dev), ctx->dbg_host, 0));
    FM_TRY_CUDA(cudaDeviceSynchronize());
    if (world == 1) {
        ctx->peer_base[0] = ctx->symm;
        ctx->attached = true;
    }
#undef FM_TRY
#undef FM_TRY_CUDA
    *out = ctx;
    return FM_OK;
}

FM_API int fm_destroy(fm_ctx_t* ctx) {
    if (ctx == nullptr) return FM_OK;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (int r = 0; r < ctx->d.world; ++r)
        if (ctx->peer_opened[r] && ctx->peer_base[r] != nullptr) cudaIpcCloseMemHandle(ctx->peer_base[r]);
    void* bufs[] = {ctx->topk_idx, ctx->topk_w, ctx->mcw, ctx->slot, ctx->counts, ctx->gate_out, ctx->chunk_counts,
                    ctx->ctrl, ctx->g0_done, ctx->g1_done, ctx->pkt_done, ctx->recv_cnt, ctx->blocks, ctx->hidden, ctx->trace,
                    ctx->aux, ctx->h_s, ctx->y_s, ctx->s0_done, ctx->s1_done};
    for (void* b : bufs)
        if (b != nullptr) cudaFree(b);
    for (int i = 0; i < FM_HOST_SLOTS; ++i) {
        if (ctx->x_stage[i] != nullptr) cudaFree(ctx->x_stage[i]);
        if (ctx->out_stage[i] != nullptr) cudaFree(ctx->out_stage[i]);
        if (ctx->ev_h2d[i] != nullptr) cudaEventDestroy(ctx->ev_h2d[i]);
        if (ctx->ev_kernel[i] != nullptr) cudaEventDestroy(ctx->ev_kernel[i]);
        if (ctx->ev_d2h[i] != nullptr) cudaEventDestroy(ctx->ev_d2h[i]);
    }
    if (ctx->s_h2d != nullptr) cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_d2h != nullptr) cudaStreamDestroy(ctx->s_d2h);
    if (ctx->symm != nullptr && !ctx->symm_external) cudaFree(ctx->symm);
    if (ctx->dbg_host != nullptr) cudaFreeHost(ctx->dbg_host);
    delete ctx;
    return FM_OK;
}

FM_API int fm_get_dims(const fm_ctx_t* ctx, fm_dims_t* out) {
    if (ctx == nullptr || out == nullptr) return fail(FM_EINVAL, "null argument");
    *out = ctx->d;
    return FM_OK;
}

FM_API int fm_num_local_experts(const fm_ctx_t* ctx) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    return ctx->d.num_local_experts;
}

FM_API int fm_symm_size(const fm_ctx_t* ctx, size_t* bytes) {
    if (ctx == nullptr || bytes == nullptr) return fail(FM_EINVAL, "null argument");
    *bytes = ctx->symm_bytes;
    return FM_OK;
}

FM_API int fm_symm_local_ptr(const fm_ctx_t* ctx, void** base) {
    if (ctx == nullptr || base == nullptr) return fail(FM_EINVAL, "null argument");
    *base = ctx->symm;
    return FM_OK;
}

FM_API int fm_output_buffer(const fm_ctx_t* ctx, void** ptr, size_t* bytes) {
    if (ctx == nullptr || ptr == nullptr || bytes == nullptr) return fail(FM_EINVAL, "null argument");
    const bool has = ctx->d.world > 1;   // the accumulation target peers add into; single rank: the caller's tensor
    *ptr = has ? static_cast<char*>(ctx->symm) + ctx->off_out_acc : nullptr;
    *bytes = has ? (size_t)ctx->d.S * ctx->d.H * 2 : 0;
    return FM_OK;
}

FM_API int fm_symm_use_external(fm_ctx_t* ctx, void* base, size_t bytes) {
    if (ctx == nullptr || base == nullptr) return fail(FM_EINVAL, "null argument");
    if (ctx->attached && ctx->d.world > 1) return fail(FM_ESTATE, "already attached");
    if (bytes < ctx->symm_bytes) return fail(FM_EINVAL, "external slab too small: %zu < %zu", bytes, ctx->symm_bytes);
    if (reinterpret_cast<uintptr_t>(base) % 1024) return fail(FM_EINVAL, "external slab must be 1 KiB aligned");
    FM_CUDA(cudaSetDevice(ctx->device));
    if (ctx->symm != nullptr && !ctx->symm_external) FM_CUDA(cudaFree(ctx->symm));
    ctx->symm = base;
    ctx->symm_external = true;
    if (ctx->d.world == 1) ctx->peer_base[0] = base;
    return FM_OK;
}

FM_API int fm_symm_export(fm_ctx_t* ctx, void* handle_out) {
    if (ctx == nullptr || handle_out == nullptr) return fail(FM_EINVAL, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == FM_IPC_HANDLE_BYTES, "IPC handle size");
    FM_CUDA(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    FM_CUDA(cudaIpcGetMemHandle(&h, ctx->symm));
    memcpy(handle_out, &h, sizeof(h));
    return FM_OK;
}

FM_API int fm_symm_attach_ipc(fm_ctx_t* ctx, const void* all_handles) {
    if (ctx == nullptr || all_handles == nullptr) return fail(FM_EINVAL, "null argument");
    if (ctx->attached && ctx->d.world > 1) return fail(FM_ESTATE, "already attached");
    FM_CUDA(cudaSetDevice(ctx->device));
    const char* hs = static_cast<const char*>(all_handles);
    for (int r = 0; r < ctx->d.world; ++r) {
        if (r == ctx->d.rank) {
            ctx->peer_base[r] = ctx->symm;
            continue;
        }
        cudaIpcMemHandle_t h;
        memcpy(&h, hs + (size_t)r * FM_IPC_HANDLE_BYTES, sizeof(h));
        void* ptr = nullptr;
        FM_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        ctx->peer_base[r] = ptr;
        ctx->peer_opened[r] = true;
    }
    ctx->attached = true;
    return FM_OK;
}

FM_API int fm_symm_attach_ptrs(fm_ctx_t* ctx, void* const* peer_bases) {
    if (ctx == nullptr || peer_bases == nullptr) return fail(FM_EINVAL, "null argument");
    for (int r = 0; r < ctx->d.world; ++r) {
        if (peer_bases[r] == nullptr) return fail(FM_EINVAL, "peer base %d is null", r);
        ctx->peer_base[r] = (r == ctx->d.rank) ? ctx->symm : peer_bases[r];
    }
    ctx->attached = true;
    return FM_OK;
}

FM_API int fm_moe_forward_tokens(fm_ctx_t* ctx, const void* x, int n_tokens, const void* gate_w, const void* expert_w,
                                 const void* bias_up, const void* bias_down, void* out, void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    return launch(ctx, {x, n_tokens, nullptr, gate_w, expert_w, bias_up, bias_down, out, stream});
}

FM_API int fm_moe_forward_tokens_dev(fm_ctx_t* ctx, const void* x, const int32_t* n_tokens_dev, const void* gate_w,
                                     const void* expert_w, const void* bias_up, const void* bias_down, void* out,
                                     void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    // x and out hold S rows; a null count pointer is rejected before the context is read
    const int rows = n_tokens_dev != nullptr ? ctx->d.S : 0;
    ForwardCall f = {x, rows, n_tokens_dev, gate_w, expert_w, bias_up, bias_down, out, stream};
    f.count_on_device = true;
    return launch(ctx, f);
}

FM_API int fm_moe_forward_routed(fm_ctx_t* ctx, const void* x, int n_tokens, const int32_t* n_tokens_dev,
                                 const int32_t* topk_idx, const float* topk_w, const void* expert_w,
                                 const void* bias_up, const void* bias_down, void* out, void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    ForwardCall f = {x, n_tokens, n_tokens_dev, nullptr /* no gate weights */, expert_w, bias_up, bias_down, out, stream};
    f.route = fm::ROUTE_CALLER;
    f.topk_idx = topk_idx;
    f.topk_w = topk_w;
    return launch(ctx, f);
}

FM_API int fm_moe_forward_gated(fm_ctx_t* ctx, const void* x, int n_tokens, const int32_t* n_tokens_dev,
                                const void* gate_w, const fm_router_t* router, const float* score_bias,
                                const void* expert_w, const void* bias_up, const void* bias_down, void* out,
                                void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    ForwardCall f = {x, n_tokens, n_tokens_dev, gate_w, expert_w, bias_up, bias_down, out, stream};
    f.route = fm::ROUTE_GATED;
    f.router = router;
    f.score_bias = score_bias;
    return launch(ctx, f);
}

FM_API int fm_shared_reserve(fm_ctx_t* ctx, int32_t max_inter) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    if (max_inter <= 0 || max_inter % 64)
        return fail(FM_EINVAL, "max_inter = %d must be a positive multiple of 64", max_inter);
    if (ctx->d.E == 1)
        return fail(FM_EINVAL, "a shared expert needs num_experts > 1 (an E = 1 context is one dense expert already)");
    if (ctx->shared_max != 0)
        return fail(FM_ESTATE, "the shared-expert staging is already reserved (max_inter = %d)", ctx->shared_max);
    FM_CUDA(cudaSetDevice(ctx->device));
    const size_t S = (size_t)ctx->d.S;
    int rc;
    if ((rc = dev_alloc(&ctx->h_s, S * max_inter)) || (rc = dev_alloc(&ctx->y_s, S * ctx->d.H)) ||
        (rc = dev_alloc(&ctx->s0_done, S / fm::BLOCK_M)) || (rc = dev_alloc(&ctx->s1_done, S / fm::BLOCK_M))) {
        void* bufs[] = {ctx->h_s, ctx->y_s, ctx->s0_done, ctx->s1_done};
        for (void* b : bufs)
            if (b != nullptr) cudaFree(b);
        ctx->h_s = ctx->y_s = nullptr;
        ctx->s0_done = ctx->s1_done = nullptr;
        return rc;
    }
    ctx->shared_max = max_inter;
    return FM_OK;
}

FM_API int fm_moe_forward_shared(fm_ctx_t* ctx, const void* x, int n_tokens, const int32_t* n_tokens_dev,
                                 const void* gate_w, const fm_router_t* router, const float* score_bias,
                                 const int32_t* topk_idx, const float* topk_w,
                                 const void* expert_w, const void* bias_up, const void* bias_down,
                                 const fm_shared_expert_t* shared, void* out, void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    ForwardCall f = {x, n_tokens, n_tokens_dev, gate_w, expert_w, bias_up, bias_down, out, stream};
    f.route = gate_w == nullptr ? fm::ROUTE_CALLER : router == nullptr ? fm::ROUTE_ROUTER : fm::ROUTE_GATED;
    f.topk_idx = topk_idx;
    f.topk_w = topk_w;
    f.router = router;
    f.score_bias = score_bias;
    f.with_shared = true;
    f.shared = shared;
    return launch(ctx, f);
}

FM_API int fm_last_launch(fm_ctx_t* ctx, uint64_t* launches, int32_t* n_tokens) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    return read_launch_record(ctx, launches, n_tokens);
}

FM_API int fm_moe_forward(fm_ctx_t* ctx, const void* x, const void* gate_w, const void* expert_w, const void* bias_up,
                          const void* bias_down, void* out, void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    return launch(ctx, {x, ctx->d.S, nullptr, gate_w, expert_w, bias_up, bias_down, out, stream});
}

// ---- host-buffer entry points -----------------------------------------------------------------------------------
static int host_setup(fm_ctx* c) {
    if (c->host_ready) return FM_OK;
    const size_t elems = (size_t)c->d.S * c->d.H;
    int rc;
    for (int i = 0; i < FM_HOST_SLOTS; ++i) {
        if ((rc = dev_alloc(&c->x_stage[i], elems, false))) return rc;
        if ((rc = dev_alloc(&c->out_stage[i], elems, false))) return rc;
        FM_CUDA(cudaEventCreateWithFlags(&c->ev_h2d[i], cudaEventDisableTiming));
        FM_CUDA(cudaEventCreateWithFlags(&c->ev_kernel[i], cudaEventDisableTiming));
        FM_CUDA(cudaEventCreateWithFlags(&c->ev_d2h[i], cudaEventDisableTiming));
    }
    FM_CUDA(cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking));
    FM_CUDA(cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking));
    c->host_ready = true;
    return FM_OK;
}

FM_API int fm_host_submit(fm_ctx_t* ctx, const void* x_host, const void* gate_w, const void* expert_w, const void* bias_up,
                          const void* bias_down, void* out_host, void* stream, uint64_t* ticket) {
    if (ctx == nullptr || x_host == nullptr || out_host == nullptr || ticket == nullptr) return fail(FM_EINVAL, "null argument");
    FM_CUDA(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = host_setup(ctx))) return rc;
    if (ctx->host_submitted - ctx->host_waited >= FM_HOST_SLOTS)
        return fail(FM_ESTATE, "%d steps in flight: call fm_host_wait on the oldest ticket first", FM_HOST_SLOTS);
    const size_t bytes = (size_t)ctx->d.S * ctx->d.H * 2;
    const int slot = (int)(ctx->host_submitted % FM_HOST_SLOTS);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // x_stage[slot] was last read by the kernel of step (submitted - SLOTS): the H2D copy waits for that kernel
    // (out_stage[slot]'s previous D2H has been waited for on the host already, see the in-flight bound above)
    if (ctx->host_submitted >= FM_HOST_SLOTS) FM_CUDA(cudaStreamWaitEvent(ctx->s_h2d, ctx->ev_kernel[slot], 0));
    FM_CUDA(cudaMemcpyAsync(ctx->x_stage[slot], x_host, bytes, cudaMemcpyHostToDevice, ctx->s_h2d));
    FM_CUDA(cudaEventRecord(ctx->ev_h2d[slot], ctx->s_h2d));
    FM_CUDA(cudaStreamWaitEvent(s, ctx->ev_h2d[slot], 0));
    if ((rc = launch(ctx, {ctx->x_stage[slot], ctx->d.S, nullptr, gate_w, expert_w, bias_up, bias_down,
                           ctx->out_stage[slot], stream}))) return rc;
    FM_CUDA(cudaEventRecord(ctx->ev_kernel[slot], s));
    FM_CUDA(cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_kernel[slot], 0));
    FM_CUDA(cudaMemcpyAsync(out_host, ctx->out_stage[slot], bytes, cudaMemcpyDeviceToHost, ctx->s_d2h));
    FM_CUDA(cudaEventRecord(ctx->ev_d2h[slot], ctx->s_d2h));
    *ticket = ctx->host_submitted++;
    return FM_OK;
}

FM_API int fm_host_wait(fm_ctx_t* ctx, uint64_t ticket) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    if (ticket >= ctx->host_submitted) return fail(FM_EINVAL, "ticket %llu was never issued", (unsigned long long)ticket);
    if (ticket < ctx->host_waited) return FM_OK;   // already complete
    if (ticket != ctx->host_waited) return fail(FM_ESTATE, "tickets must be waited for in submission order (oldest is %llu)",
                                                (unsigned long long)ctx->host_waited);
    FM_CUDA(cudaSetDevice(ctx->device));
    cudaError_t e = cudaEventSynchronize(ctx->ev_d2h[ticket % FM_HOST_SLOTS]);
    int rc;
    if ((rc = check_kernel_status(ctx))) return rc;
    if (e != cudaSuccess) return fail(FM_ECUDA, "cudaEventSynchronize failed: %s", cudaGetErrorString(e));
    ctx->host_waited = ticket + 1;
    return FM_OK;
}

FM_API int fm_moe_forward_host(fm_ctx_t* ctx, const void* x_host, const void* gate_w, const void* expert_w,
                               const void* bias_up, const void* bias_down, void* out_host, void* stream) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    int rc;
    while (ctx->host_waited < ctx->host_submitted)   // drain earlier asynchronous steps first
        if ((rc = fm_host_wait(ctx, ctx->host_waited))) return rc;
    uint64_t t = 0;
    if ((rc = fm_host_submit(ctx, x_host, gate_w, expert_w, bias_up, bias_down, out_host, stream, &t))) return rc;
    return fm_host_wait(ctx, t);
}

FM_API int fm_check(fm_ctx_t* ctx) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    return check_kernel_status(ctx);
}

FM_API int fm_set_timeout_ms(fm_ctx_t* ctx, uint32_t ms) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    ctx->timeout_ns = (unsigned long long)ms * 1000000ull;
    return FM_OK;
}

FM_API int fm_set_trace(fm_ctx_t* ctx, int enable) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    ctx->trace_on = enable != 0;
    return FM_OK;
}

FM_API int fm_set_weight_on_input(fm_ctx_t* ctx, int enable) {
    if (ctx == nullptr) return fail(FM_EINVAL, "null context");
    if (enable != 0 && enable != 1) return fail(FM_EINVAL, "enable must be 0 or 1, got %d", enable);
    if (enable && ctx->d.k != 1)
        return fail(FM_EINVAL, "the router weight on the input needs k = 1 (each pick would need its own copy of the "
                               "row); this context has k = %d", ctx->d.k);
    if (enable && ctx->d.E == 1) return fail(FM_EINVAL, "the router weight on the input needs E > 1 (no routing at E = 1)");
    ctx->weight_on_input = enable == 1;
    return FM_OK;
}

FM_API uint64_t fm_launch_count(const fm_ctx_t* ctx) { return ctx ? ctx->launches : 0; }

static int buffer_desc(const fm_ctx_t* c, int which, const void** ptr, size_t* bytes) {
    const fm_dims_t& d = c->d;
    const char* sb = static_cast<const char*>(c->symm);
    switch (which) {
        case FM_BUF_TOPK_IDX: *ptr = c->topk_idx; *bytes = (size_t)d.S * d.k * 4; break;
        case FM_BUF_TOPK_W: *ptr = c->topk_w; *bytes = (size_t)d.S * d.k * 2; break;
        case FM_BUF_MCW: *ptr = c->mcw; *bytes = (size_t)d.S * 4; break;
        case FM_BUF_SLOT: *ptr = c->slot; *bytes = (size_t)d.S * d.k * 4; break;
        case FM_BUF_COUNTS: *ptr = c->counts; *bytes = (size_t)d.E * 4; break;
        case FM_BUF_RECV_X: *ptr = sb + c->off_recv_x; *bytes = (size_t)c->num_pkts * d.pEC * d.H * 2; break;
        case FM_BUF_HIDDEN: *ptr = c->hidden; *bytes = (size_t)c->num_pkts * d.pEC * d.P * 2; break;
        case FM_BUF_RET_Y:
            if (c->fused) return fail(FM_EINVAL, "the return buffer does not exist on the fused-combine path (FM_FUSED_COMBINE=0 keeps it)");
            *ptr = sb + c->off_ret_y; *bytes = (size_t)d.E * d.pEC * d.H * 2; break;
        case FM_BUF_GATE_OUT: *ptr = c->gate_out; *bytes = (size_t)d.S * d.E * 2; break;
        case FM_BUF_RECV_CNT: *ptr = c->recv_cnt; *bytes = (size_t)c->num_pkts * 4; break;
        case FM_BUF_TRACE: *ptr = c->trace; *bytes = (size_t)c->grid * fm::TRACE_SLOTS * 8; break;
        case FM_BUF_AUX_LOSS:
            if (c->aux == nullptr) return fail(FM_EINVAL, "the auxiliary loss exists only with is_training = 1");
            // the last launch's half of the [2][2E+1] buffer: fm_read_buffer adds its offset from the device's launch count
            *ptr = c->aux; *bytes = (size_t)(2 * d.E + 1) * 4; break;
        case FM_BUF_SHARED_Y:
            if (c->y_s == nullptr) return fail(FM_EINVAL, "the shared expert's outputs exist only after fm_shared_reserve");
            *ptr = c->y_s; *bytes = (size_t)d.S * d.H * 2; break;
        case FM_BUF_SHARED_HIDDEN:   // [S, Ps] at the stride of the last shared launch's tensor map (TM_HS)
            if (c->shared_ps == 0) return fail(FM_EINVAL, "the shared expert's h_s exists only after a launch with one");
            *ptr = c->h_s; *bytes = (size_t)d.S * c->shared_ps * 2; break;
        default: return fail(FM_EINVAL, "unknown buffer id %d", which);
    }
    return FM_OK;
}

FM_API int fm_buffer_bytes(const fm_ctx_t* ctx, int which, size_t* bytes) {
    if (ctx == nullptr || bytes == nullptr) return fail(FM_EINVAL, "null argument");
    const void* p = nullptr;
    return buffer_desc(ctx, which, &p, bytes);
}

FM_API int fm_read_buffer(fm_ctx_t* ctx, int which, void* host_dst, size_t bytes) {
    if (ctx == nullptr || host_dst == nullptr) return fail(FM_EINVAL, "null argument");
    const void* p = nullptr;
    size_t n = 0;
    int rc = buffer_desc(ctx, which, &p, &n);
    if (rc) return rc;
    if (bytes != n) return fail(FM_EINVAL, "buffer %d holds %zu bytes, caller asked for %zu", which, n, bytes);
    FM_CUDA(cudaSetDevice(ctx->device));
    cudaError_t e = cudaDeviceSynchronize();
    if ((rc = check_kernel_status(ctx))) return rc;
    if (e != cudaSuccess) return fail(FM_ECUDA, "cudaDeviceSynchronize failed: %s", cudaGetErrorString(e));
    if (which == FM_BUF_AUX_LOSS) {   // launch L wrote parity L & 1
        uint64_t launches = 0;
        if ((rc = read_launch_record(ctx, &launches, nullptr))) return rc;
        p = static_cast<const float*>(p) + (size_t)(launches & 1u) * (2 * ctx->d.E + 1);
    }
    FM_CUDA(cudaMemcpy(host_dst, p, n, cudaMemcpyDeviceToHost));
    return FM_OK;
}

}  // extern "C"
