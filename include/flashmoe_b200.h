/*
 * flashmoe_b200.h -- C-ABI of the H100-native (sm_90a) fused distributed-MoE forward path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch types.  It replaces what the reference binds
 * through pybind in csrc/python_bindings.cu (reference paths below are relative to osayamenja/FlashMoE):
 *
 *   reference interface                                   replaced by
 *   ---------------------------------------------------   ------------------------------------------------------
 *   _C.initialize()        python_bindings.cu:157-159     fm_create + fm_symm_* (explicit rank/world, no NVSHMEM PMI)
 *                          bootstrap.cuh:532-547
 *   _C.finalize()          python_bindings.cu:164-166     fm_destroy
 *                          bootstrap.cuh:561-588
 *   _C.moe_forward(...)    python_bindings.cu:17-151      fm_moe_forward (device buffers, caller's weights used in
 *                          moe.cuh:146-205                place) / fm_moe_forward_host (host activations in/out)
 *   _C.get_compiled_config python_bindings.cu:170-179     fm_compiled_config + fm_get_dims
 *   _C.get_bookkeeping /   python_bindings.cu:181-189     fm_num_local_experts
 *   get_num_local_experts
 *   csrc/flashmoe_config.json -> -D macros -> ACC         fm_config_t (the same 15 keys); the JSON is baked into the
 *                          CMakeLists.txt:114-237         library at build time and returned by fm_compiled_config
 *                          types.cuh:441-512
 *
 * Error convention: every function returns 0 on success or a negative FM_E* code; fm_last_error() returns a
 * thread-local human-readable message.  The library never calls exit() (the reference does: debug.cuh:19-43).
 *
 * Threading: a context is used by one host thread at a time; one context (= one process) per GPU; work is enqueued
 * on the stream passed by the caller (the reference uses cudaStreamPerThread and blocks, python_bindings.cu:145).
 */
#ifndef FLASHMOE_B200_H
#define FLASHMOE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FM_API __attribute__((visibility("default")))

#define FM_OK 0
#define FM_EINVAL (-1)   /* bad argument / config violates a hot-path constraint */
#define FM_ECUDA (-2)    /* a CUDA runtime/driver call failed */
#define FM_ESTATE (-3)   /* call made in the wrong state (e.g. forward before peers are attached) */
#define FM_EKERNEL (-4)  /* the kernel reported a protocol timeout (see fm_last_error) */
#define FM_ENOMEM (-5)

#define FM_MAX_WORLD 16
#define FM_IPC_HANDLE_BYTES 64

/* The 15 keys of csrc/flashmoe_config.json (reference csrc/flashmoe_config.json:1-16), same names. */
typedef struct fm_config {
    int32_t capacity_factor;
    int32_t drop_tokens;
    int32_t expert_top_k;
    int32_t global_batch;
    int32_t is_training;
    int32_t hidden_act; /* 0 relu, 1 gelu, 2 swiglu (expert_w [nLx, 3, P, H]) */
    int32_t hidden_size;
    int32_t intermediate_size;
    int32_t mini_batch;
    int32_t moe_frequency;
    int32_t num_experts;
    int32_t num_layers;
    int32_t sequence_len;
    int32_t torch_dtype; /* 2 = bf16 is the only compute type of this build */
    int32_t vocab_size;
} fm_config_t;

/* Derived dimensions, the reference's get_compiled_config() keys plus the capacity figures (types.cuh:470-504). */
typedef struct fm_dims {
    int32_t S, H, E, P, PX, element_size;
    int32_t k, EC, pEC, TCM;
    int32_t world, rank, num_local_experts;
    int32_t num_sms, smem_bytes;
    int32_t grid; /* CTAs of the persistent kernel (= num_sms); rows of FM_BUF_TRACE */
} fm_dims_t;

typedef struct fm_ctx fm_ctx_t;

/* Config baked into the library at build time from csrc/flashmoe_config.json. */
FM_API int fm_compiled_config(fm_config_t* out);

/* Create a context on CUDA device `device` for rank `rank` of `world` expert-parallel ranks.
 * cfg == NULL uses the compiled config.  Allocates all workspaces, including this rank's symmetric slab
 * (receive buffers + flags that peers write into over NVLink). */
FM_API int fm_create(const fm_config_t* cfg, int rank, int world, int device, fm_ctx_t** out);
FM_API int fm_destroy(fm_ctx_t* ctx);

FM_API int fm_get_dims(const fm_ctx_t* ctx, fm_dims_t* out);
FM_API int fm_num_local_experts(const fm_ctx_t* ctx);

/* ---- symmetric memory plumbing (replaces nvshmem_malloc/nvshmem_ptr, bootstrap.cuh:359-360,442-443) ----
 * world == 1: nothing to do.  Otherwise the host exchanges either CUDA IPC handles (any out-of-band channel,
 * e.g. torch.distributed all_gather) or already-mapped peer base pointers (e.g. torch symmetric memory). */
FM_API int fm_symm_size(const fm_ctx_t* ctx, size_t* bytes);
FM_API int fm_symm_local_ptr(const fm_ctx_t* ctx, void** base);
FM_API int fm_symm_export(fm_ctx_t* ctx, void* handle_out /* FM_IPC_HANDLE_BYTES */);
FM_API int fm_symm_attach_ipc(fm_ctx_t* ctx, const void* all_handles /* world x FM_IPC_HANDLE_BYTES, rank order */);
FM_API int fm_symm_attach_ptrs(fm_ctx_t* ctx, void* const* peer_bases /* world pointers, rank order */);
/* Use a caller-provided slab (size >= fm_symm_size, 1 KiB aligned, zero-filled) instead of the internal one;
 * must be called before attach.  For torch symmetric memory / NVSHMEM allocations. */
FM_API int fm_symm_use_external(fm_ctx_t* ctx, void* base, size_t bytes);

/* ---- the hot path ----
 * All pointers are DEVICE pointers to contiguous bf16 tensors:
 *   x            [S, H]                     activations of this rank's tokens        (input.view(S,H))
 *   gate_w       [H, E]                     consumed REINTERPRETED flat as [E, H]    (python_bindings.cu:93-99)
 *   expert_w     [nLx, 2, P, H]             [i,0] = W_up [P,H]; [i,1] flat-viewed as W_down [H,P] (:104-119)
 *   bias_up      [nLx, P] or NULL (zero)    bias_down [nLx, H] or NULL (zero)        (moe.cuh:117-124)
 *   out          [S, H]                     written in full
 * With hidden_act = 2 (SwiGLU, y = W_down (silu(W_gate x + b_g) * (W_up x + b_u)) + b_down):
 *   expert_w     [nLx, 3, P, H]             [i,0] = W_gate [P,H]; [i,1] = W_up [P,H]; [i,2] flat-viewed as W_down [H,P]
 *                                           (per expert vLLM's w13, gate then up, followed by w2).  From Hugging Face
 *                                           tensors, once at load time: torch.stack([w_gate, w_up,
 *                                           w_down.reshape(nLx, P, H)], 1)
 *   bias_up      [nLx, 2, P] or NULL        [i,0] = gate bias, [i,1] = up bias
 *   h = rne_bf16(fl(fl(g * sigmoid(g)) * u)), g = fl(W_gate x + b_g), u = fl(W_up x + b_u), all in fp32 with the one
 *   final rounding (Hugging Face rounds W_gate x, silu and the product to bf16 separately; this does not).
 * Enqueues one fused persistent kernel on `stream` (cudaStream_t); collective across the world: every rank must
 * call it the same number of times.  Does not synchronise. */
FM_API int fm_moe_forward(fm_ctx_t* ctx, const void* x, const void* gate_w, const void* expert_w,
                          const void* bias_up, const void* bias_down, void* out, void* stream);

/* Same, on n_tokens tokens (0 <= n_tokens <= S; any count, not only multiples of 128): x and out are [n_tokens, H] and
 * may be exactly that long.  The context's S is the maximum; the call computes exactly what a context created with
 * sequence_len * mini_batch = n_tokens computes -- routing, capacity EC(n) = (drop_tokens ? ceil(n/E) : n) * CF * k,
 * slots, drops, outputs, and with is_training = 1 the auxiliary loss averaged over n (all zero at n = 0).  Nothing is
 * written to out at or beyond row n_tokens.  With n_tokens = 0, x and out may be NULL; the call still launches and takes
 * part in the collective.  With world > 1 every rank passes its own count (counts may differ between ranks and between
 * calls; every rank still calls the same number of times).  fm_moe_forward(...) is fm_moe_forward_tokens(..., S, ...).
 * FM_EINVAL for n_tokens < 0 or > S.  The routing tables read back with fm_read_buffer hold n_tokens valid rows.  A row
 * below n_tokens that holds a NaN routes all k of its picks to expert 0, as the reference does; they take capacity of
 * expert 0 like any other pick. */
FM_API int fm_moe_forward_tokens(fm_ctx_t* ctx, const void* x, int n_tokens, const void* gate_w, const void* expert_w,
                                 const void* bias_up, const void* bias_down, void* out, void* stream);

/* Same, with the token count in DEVICE memory: the kernel reads n = *n_tokens_dev (one int32) when it starts, so the
 * count may be produced on the GPU (no host synchronisation) and one captured CUDA graph serves every count.  x and out
 * are buffers of S rows; the result is bit-identical to fm_moe_forward_tokens(ctx, x, n, ...) -- routing tables and
 * auxiliary loss included.  Rows n and above of x may hold anything (NaN included) and affect no result; rows n and
 * above of out are never written.  A count outside [0, S] does not fault: that launch runs on 0 tokens (it still takes
 * part in the collective) and the next fm_check / fm_read_buffer / fm_host_wait returns FM_EINVAL once, naming the
 * count; the context stays usable.  fm_last_launch returns the count a launch ran with. */
FM_API int fm_moe_forward_tokens_dev(fm_ctx_t* ctx, const void* x, const int32_t* n_tokens_dev, const void* gate_w,
                                     const void* expert_w, const void* bias_up, const void* bias_down, void* out,
                                     void* stream);

/* Same, on the caller's routing instead of the built-in router (no gate weights): topk_idx int32 [n, k] and topk_w fp32
 * [n, k], DEVICE memory, contiguous and 16-byte aligned, name the experts of each token's k picks and their weights;
 * -1 means "no expert" (the pick takes no capacity, is not counted and moves no row).  The token count follows
 * fm_moe_forward_tokens (n_tokens_dev == NULL: x, out and the routing arrays hold n_tokens rows) or
 * fm_moe_forward_tokens_dev (n_tokens_dev != NULL: n is read from the device when the kernel starts, the arrays hold S
 * rows and n_tokens must be S); rows at or past n are never read, rows of out at or past n are never written.
 * Capacity EC(n) and slots (ascending (token, pick) order among the picks of one expert; kept = slot < EC) are the
 * router path's.  Result: out[t] = bf16 accumulation, in ascending pick order from +0, of rne(w~_j * y_j) over the kept
 * picks j, with w~_j = rne_bf16(topk_w[t, j]) and y_j the bf16 output of expert topk_idx[t, j] on row t (bias
 * included) -- the router path's combine with p~ = w~ and mCw = 1.  k = 1 is scaled too (the router path copies y
 * unscaled; pass w = 1 for that).  A token may name one expert twice (each pick is its own row); weights are not checked
 * (a NaN propagates).  An index outside [-1, E) does not fault: it is treated as -1 and the next fm_check /
 * fm_read_buffer / fm_host_wait returns FM_EINVAL once, naming the token, the pick and the value; the context stays
 * usable.  FM_EINVAL for an E = 1 context (no router to replace) and an is_training = 1 context (the auxiliary loss
 * needs router probabilities).  With world > 1 each rank passes its own routing, in global expert ids, and its own
 * count; the kind of call (routed or not) may differ between ranks, the number of calls may not.  May be captured in a
 * CUDA graph like the other entry points: the pointers are fixed at capture, the arrays' contents (and *n_tokens_dev)
 * are read when the launch starts. */
FM_API int fm_moe_forward_routed(fm_ctx_t* ctx, const void* x, int n_tokens, const int32_t* n_tokens_dev,
                                 const int32_t* topk_idx, const float* topk_w, const void* expert_w,
                                 const void* bias_up, const void* bias_down, void* out, void* stream);

/* A router rule for fm_moe_forward_gated (DeepSeek-V2/V3, Kimi K2, GLM-4.5, Qwen-MoE, OLMoE and Llama 4 style routers;
 * Llama 4 also needs fm_set_weight_on_input, since it scales the expert's input row by the weight, not its output). */
typedef struct fm_router {
    int32_t scoring;      /* 0 softmax (the router's own recurrence), 1 sigmoid */
    int32_t n_group;      /* experts split into n_group contiguous groups of E / n_group; 1 = no group limit */
    int32_t topk_group;   /* groups kept per token */
    int32_t group_top;    /* group score = sum of the group's 1 (max) or 2 largest biased scores */
    int32_t renormalize;  /* 0 / 1 */
    float scale;          /* route scale applied to every weight */
} fm_router_t;

/* Same as fm_moe_forward_routed, but the routing is computed in the kernel from the gate weights by the rule *router:
 * the router's logits l (the same GEMV / tensor-core product as fm_moe_forward_tokens), then per token t
 *   1. scores s_e: scoring 0 = the router's softmax probability (the bits of gate_out of an fm_moe_forward_tokens
 *      launch); scoring 1 = sigmoid, computed as __frcp_rn(1 + ex2.approx.ftz(fl(-l * log2e))), relative error at most
 *      2^-21 + 2^-24 * (1.25 |l| + 2) against 1 / (1 + e^-l) while the score is normal; exactly 1.0 for l >= 17.34,
 *      subnormal for l in about [-88.7, -87.4], +0 from l = -88.73 (the power overflows);
 *   2. choice values c_e = fl(s_e + score_bias[e]) (c = s without a bias); the bias steers selection only;
 *   3. n_group > 1: group score G_g = the largest c of the group (group_top 1) or fl(largest + second largest)
 *      (group_top 2); the topk_group groups with the largest G are kept, the experts of the others cannot be picked
 *      (DeepSeek's own Gate.forward; not the 0.0 mask of the Hugging Face DeepseekV3TopkRouter);
 *   4. k picks by c among the allowed experts, k rounds of a strict '>': an equal value goes to the lower index, NaN
 *      never compares greater, a round in which nothing compares greater than -inf takes index 0 (groups likewise);
 *   5. weights w_j = s_{e_j} (unbiased); renormalize: W = fp32 sum of the w_j in pick order from +0,
 *      w_j = W > 0 ? w_j / W (rounded) : 0 (capacity-dropped picks count in W); then w_j = fl(w_j * scale).
 * The launch stores topk_idx, topk_w = rne_bf16(w), mcw = 1 and gate_out = rne_bf16(s) (the unbiased scores), and from
 * there runs exactly as fm_moe_forward_routed on that routing: capacity, slots, the mCw = 1 combine, k = 1 scaled.
 * The token count follows fm_moe_forward_routed.  score_bias: fp32 [E] device memory, 16-byte aligned, or NULL; its
 * contents are read when each launch starts.  FM_EINVAL for router == NULL, scoring not 0 / 1, n_group not in [1, 32]
 * or not dividing E, topk_group not in [1, n_group], n_group > 1 with group_top not 1 / 2 or above E / n_group,
 * k > topk_group * E / n_group, renormalize not 0 / 1, scale not finite or <= 0, a misaligned score_bias, an E = 1
 * context and an is_training = 1 context.  With world > 1 each rank passes its own gate weights and bias (global expert
 * ids). */
FM_API int fm_moe_forward_gated(fm_ctx_t* ctx, const void* x, int n_tokens, const int32_t* n_tokens_dev,
                                const void* gate_w, const fm_router_t* router, const float* score_bias /* [E] or NULL */,
                                const void* expert_w, const void* bias_up, const void* bias_down, void* out,
                                void* stream);

/* ---- shared expert (DeepSeek-V2/V3 and Kimi K2 n_shared_experts, Qwen-MoE shared_expert_intermediate_size, Llama 4
 * with fm_set_weight_on_input, GLM-4.5, DeepSpeed Residual-MoE) ----
 * A dense FFN every token passes through, its output added to the routed combine:
 *   w          bf16 [2, Ps, H], contiguous: exactly one routed expert's slice of expert_w -- [0] is W_up [Ps, H], [1] is the
 *              same Ps*H block flat-viewed as W_down [H, Ps]
 *   bias_up    bf16 [Ps] or NULL (zero)     bias_down  bf16 [H] or NULL (zero)
 *   inter      Ps, a positive multiple of 64, at most the context's reserved size (fm_shared_reserve)
 * In a hidden_act = 2 (SwiGLU) context w is [3, Ps, H] (W_gate, W_up, W_down flat-viewed) and bias_up [2, Ps].
 * For every token t < n: s[t] = the bf16 output of that FFN on x[t], with a routed expert's arithmetic (GEMM0 + bias_up ->
 * the context's hidden_act -> bf16 h -> GEMM1 + bias_down -> one bf16 RNE), and
 *   out[t] = rne_bf16(fl32(r[t]) + fl32(s[t]))   (the sum in fp32, then one RNE)
 * where r[t] is, bit for bit, the row the same call without a shared expert writes -- on every route (router, caller,
 * gated), for every k, on both the fused and the gather combine, the router path's unscaled k = 1 copy included.  s is
 * not added into the output row beside the routed terms (with k <= 2 the fused combine is order-independent only because
 * it adds two bf16 terms onto +0; a third add would depend on arrival order): it is staged and added once, after the
 * row's routed contributions are complete.  Everything else -- topk_idx, topk_w, mcw, slot, counts, recv_cnt, gate_out
 * and, with is_training = 1, FM_BUF_AUX_LOSS -- is exactly the call without a shared expert.  The shared tiles run in the
 * same persistent kernel as the routed ones: they need only x, so they fill the time the routed rows take to arrive. */
typedef struct fm_shared_expert {
    const void* w;          /* bf16 [2, Ps, H]; SwiGLU: [3, Ps, H] */
    const void* bias_up;    /* bf16 [Ps] or NULL */
    const void* bias_down;  /* bf16 [H] or NULL */
    int32_t inter;          /* Ps */
} fm_shared_expert_t;

/* Allocate the shared expert's staging (h_s [S, max_inter], y_s [S, H], row-block counters); once per context,
 * before any forward that passes a shared expert (and before any capture).  FM_EINVAL for max_inter not a positive
 * multiple of 64, or an E = 1 context; FM_ESTATE on a second call. */
FM_API int fm_shared_reserve(fm_ctx_t* ctx, int32_t max_inter);

/* One forward with a shared expert, on any of the three routes:
 *   gate_w == NULL            caller routing: topk_idx / topk_w as fm_moe_forward_routed (router must be NULL)
 *   gate_w, router == NULL    the built-in router, as fm_moe_forward_tokens (topk_idx, topk_w and score_bias NULL)
 *   gate_w and router         the rule *router with score_bias, as fm_moe_forward_gated (topk_idx and topk_w NULL)
 * The token count follows fm_moe_forward_routed: a host n_tokens, or n_tokens_dev with n_tokens = S (rows n and above of
 * x may then hold anything, NaN included, and affect no result).  Every condition of the chosen route applies, and
 * FM_EINVAL for shared == NULL, shared->w == NULL, inter not a positive multiple of 64 or above the reserved size, a
 * misaligned (not 16-byte) w, bias_up or bias_down, an E = 1 context, gate_w with topk_idx / topk_w, router without
 * gate_w, and score_bias without router; FM_ESTATE without fm_shared_reserve.  Training contexts are accepted on the
 * router route.  May be captured in a CUDA graph like the other entry points (the shared expert's pointers and inter
 * are fixed at capture, the weights' contents are read at every replay).  With world > 1 each rank passes its own
 * shared expert, or calls an entry point without one: the kind of call may differ between ranks. */
FM_API int fm_moe_forward_shared(fm_ctx_t* ctx, const void* x, int n_tokens, const int32_t* n_tokens_dev,
                                 const void* gate_w, const fm_router_t* router, const float* score_bias,
                                 const int32_t* topk_idx, const float* topk_w,
                                 const void* expert_w, const void* bias_up, const void* bias_down,
                                 const fm_shared_expert_t* shared, void* out, void* stream);

/* ---- CUDA graphs ----
 * Every forward entry point on device buffers (fm_moe_forward, fm_moe_forward_tokens, fm_moe_forward_tokens_dev,
 * fm_moe_forward_routed, fm_moe_forward_gated, fm_moe_forward_shared) may
 * be captured into a CUDA graph and the graph replayed any number of times, interleaved with eager calls on the same
 * context.  A launch keeps no per-launch state in its parameters: the kernel takes its epoch, grid-barrier target and
 * token-dependent sizes from the context's device-side launch counter (and the device-side count) when it starts.
 * What is fixed at capture: the pointers (x, out, weights, biases, score_bias, n_tokens_dev), a host-side n_tokens, a
 * gated call's fm_router_t values, and the fm_set_trace, fm_set_weight_on_input and fm_set_timeout_ms settings (the contents of score_bias are
 * read at every replay, so a graph follows in-place bias updates).  Replays of launches on one context must run in stream order, one at a
 * time, like eager calls.  With world > 1 every rank issues the same number of launches, eager calls and replays
 * together, in the same order.  The host-buffer entry points (fm_moe_forward_host, fm_host_submit) cannot be captured.
 *
 * fm_last_launch synchronises the device and returns the number of launches the context has run (graph replays
 * included) and the token count the last one ran with (0 for an out-of-range device count).  Either pointer may be
 * NULL. */
FM_API int fm_last_launch(fm_ctx_t* ctx, uint64_t* launches, int32_t* n_tokens);

/* world > 1: the [S,H] bf16 region of this rank's symmetric slab into which the experts (local and remote) accumulate
 * this rank's output rows.  Passing exactly this pointer as `out` to fm_moe_forward leaves the result there and skips
 * the final copy into a caller tensor (zero-copy output, like registering a user buffer with NVSHMEM); it is
 * overwritten by the next forward.  world == 1: *ptr = NULL, *bytes = 0 (the kernel accumulates straight into `out`). */
FM_API int fm_output_buffer(const fm_ctx_t* ctx, void** ptr, size_t* bytes);

/* Same, with the activations in HOST memory (pinned for full PCIe speed): copies x host->device, runs the layer,
 * copies out device->host, then waits for the result (the reference's blocking behaviour,
 * python_bindings.cu:131-148).  Equivalent to fm_host_submit + fm_host_wait. */
FM_API int fm_moe_forward_host(fm_ctx_t* ctx, const void* x_host, const void* gate_w, const void* expert_w,
                               const void* bias_up, const void* bias_down, void* out_host, void* stream);

/* Pipelined form of the host-buffer call: fm_host_submit enqueues H2D copy -> layer -> D2H copy for one step and
 * returns a ticket at once; up to FM_HOST_SLOTS steps may be in flight, so the copies of neighbouring steps overlap
 * the kernel (separate copy streams, PCIe full duplex).  The kernel runs on `stream`; weights must be ready there.
 * fm_host_wait blocks until that step's out_host is complete; tickets are waited for in submission order.
 * x_host must stay valid until its H2D copy has run (i.e. until the step's ticket has been waited for). */
#define FM_HOST_SLOTS 3
FM_API int fm_host_submit(fm_ctx_t* ctx, const void* x_host, const void* gate_w, const void* expert_w,
                          const void* bias_up, const void* bias_down, void* out_host, void* stream, uint64_t* ticket);
FM_API int fm_host_wait(fm_ctx_t* ctx, uint64_t ticket);

/* Check the kernel's host-mapped status record after a synchronise; FM_EKERNEL + message if a wait timed out. */
FM_API int fm_check(fm_ctx_t* ctx);
FM_API int fm_set_timeout_ms(fm_ctx_t* ctx, uint32_t ms);
/* Launches issued through this API (a captured launch counts once, at capture; graph replays are not counted). */
FM_API uint64_t fm_launch_count(const fm_ctx_t* ctx);
/* Per-CTA phase / tile time stamps into FM_BUF_TRACE (profiling aid; off by default). */
FM_API int fm_set_trace(fm_ctx_t* ctx, int enable);
/* Apply the router weight to each routed token's INPUT row instead of its expert output (Llama 4's Llama4TextMoe, vLLM's
 * apply_router_weight_on_input); enable 0 / 1, default 0.  With it on, the caller route (fm_moe_forward_routed) and the
 * gated route (fm_moe_forward_gated), directly or through fm_moe_forward_shared, change as follows:
 *   - a kept pick of token t dispatches rne_bf16(fl32(x[t]) * fl32(w~)) instead of x[t], w~ = the stored topk_w entry
 *     (rne_bf16 of the caller's weight or of the rule's w); the fp32 product of two bf16 numbers is exact, so this is
 *     bit for bit torch's bf16 x * w;
 *   - the combine takes weight 1: out[t] is the expert's output row y (bias included); with a shared expert
 *     out[t] = rne_bf16(fl32(y) + fl32(s)), s computed from the unscaled x[t].
 * So out is bit for bit what a context with the setting off returns from fm_moe_forward_routed(x', topk_idx, ones), x'
 * the scaled rows, on the fused and the gather combine.  topk_idx, topk_w = rne_bf16(w), mcw = 1, slot, counts and
 * gate_out are those of the same call with the setting off; FM_BUF_RECV_X holds the scaled rows.  The router route
 * (fm_moe_forward, _tokens[_dev], the host entry points) is unchanged: its k = 1 combine copies y unscaled.  FM_EINVAL
 * for a null context, enable not 0 / 1, and enable = 1 on a context with k != 1 (each pick would need its own copy of the
 * row) or E = 1.  Fixed at capture, like fm_set_trace.  With world > 1 each rank's own setting governs the rows it
 * sends (the sender picks the combine weight), so ranks may differ. */
FM_API int fm_set_weight_on_input(fm_ctx_t* ctx, int enable);

/* ---- inspection (tests / debugging): copy an internal device buffer to host memory after synchronising ---- */
enum fm_buffer {
    FM_BUF_TOPK_IDX = 0, /* int32 [S,k]   expert index per pick (bit-exact parity target); routed: the caller's, invalid
                            ones replaced by -1 */
    FM_BUF_TOPK_W = 1,   /* bf16  [S,k]   gateOut[t, e_j] (bf16-rounded probability); routed: rne_bf16(topk_w); gated:
                            rne_bf16(w_j), the renormalised and scaled weight */
    FM_BUF_MCW = 2,      /* f32   [S]     sum of the k selected fp32 probabilities; routed and gated: 1.0 */
    FM_BUF_SLOT = 3,     /* int32 [S,k]   slot in the (this rank, expert) packet; >= EC means dropped; routed: INT32_MAX
                            for a -1 pick */
    FM_BUF_COUNTS = 4,   /* int32 [E]     selections per expert on this rank (incl. dropped) */
    FM_BUF_RECV_X = 5,   /* bf16  [W, nLx, pEC, H]  dispatched rows received by this rank */
    FM_BUF_HIDDEN = 6,   /* bf16  [W, nLx, pEC, P]  h = act(x W_up^T + b) staging; SwiGLU: h = silu(g)*u */
    FM_BUF_RET_Y = 7,    /* bf16  [E, pEC, H]       expert outputs returned to this rank */
    FM_BUF_GATE_OUT = 8, /* bf16  [S, E]  full softmax row (reference gateOut[S,PX] without the padding columns); not
                            written by a routed launch; gated: rne_bf16(s), the full unbiased score row */
    FM_BUF_RECV_CNT = 9, /* int32 [W, nLx] rows received per (source rank, local expert) in the last forward */
    FM_BUF_TRACE = 10,   /* u64   [grid, 128] %globaltimer stamps of the last forward (fm_set_trace) */
    FM_BUF_AUX_LOSS = 11, /* f32  [2E+1] is_training = 1 only: gML[E] (mean gate probability per expert), gMeC[E] (mean
                            routed fraction per expert), loss = sum_e gML*gMeC / E  (moe/gate.cuh:608-635,698-706,763-773) */
    FM_BUF_SHARED_Y = 12, /* bf16 [S,H]   the shared expert's s rows of the last launch that had one (rows < n valid);
                            after fm_shared_reserve only */
    FM_BUF_SHARED_HIDDEN = 13 /* bf16 [S,Ps] the shared expert's h_s rows of the last launch that had one (rows < n
                            valid), Ps that launch's (a captured launch's, recorded at capture); FM_EINVAL before any */
};
FM_API int fm_buffer_bytes(const fm_ctx_t* ctx, int which, size_t* bytes);
FM_API int fm_read_buffer(fm_ctx_t* ctx, int which, void* host_dst, size_t bytes);

FM_API const char* fm_last_error(void);
FM_API const char* fm_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FLASHMOE_B200_H */
