// fm_kernel.cuh -- the fused persistent MoE-forward kernel for sm_90a.
//
// One launch = one MoE layer forward on this rank (reference: flashmoe::moe::forward, csrc/include/flashmoe/moe/moe.cuh:77-144):
//
//   prologue  mbarriers for the later phases (off the critical path)
//   phase G   router    x.Wg^T -> online softmax -> top-k -> capacity slots         (reference moe/gate.cuh:473-720)
//             (or the caller's top-k ids and weights -> capacity slots: fm_moe_forward_routed;
//              or x.Wg^T -> softmax / sigmoid scores, bias, group limit, top-k, scaled weights: fm_moe_forward_gated)
//             grid barrier (the only one, like the reference's gate.cuh:761)
//   phase D   dispatch  token rows -> owner rank's receive buffer over NVLink (TMA bulk copies) + one flag per expert
//                                                                                    (reference os/packet.cuh:21-286)
//   phase F   expert FFN  persistent wgmma tile loop: GEMM0(+bias+act) -> h, GEMM1(+bias) -> for k <= 2
//             scaled and ADDED straight into the token's output row on the source rank (REDG.BF16x8 over peer memory),
//             otherwise stored to the source rank's return buffer + per-row-block flag
//                                                                                    (reference os/processor/processor.cuh:340-468,
//                                                                                    685-750; the OS CTA of os/os.cuh, scheduler.cuh,
//                                                                                    subscriber.cuh is replaced by an atomic tile
//                                                                                    claim + flag waits in one warp per CTA)
//   phase C   completion: wait for the experts' done flags (fused path) or gather-combine the k returned rows per token
//                                                                                    (reference processor.cuh:27-205)
//
// CTA = 384 threads, one CTA per SM, all co-resident (cooperative launch).  After the grid barrier the warps specialise:
// warp 0 = TMA producer, warp 3 = tile scheduler, warps 2 and 4-11 = dispatch, then warps 4-11 = two consumer warpgroups
// (wgmma into register accumulators, warpgroup g owns rows [64g, 64g + 64) of the 128 x 256 tile, then the epilogue:
// bias/activation/combine scaling -> bf16 -> swizzled smem transpose -> 16-byte global / peer stores or adds) and
// warp 2 = publisher (the release fence + counter / flag traffic of every finished tile, off the consumer warps'
// critical path).  Warp 1 has no role in phase F.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/flashmoe_b200.h"
#include "fm_ptx.cuh"

namespace fm {

constexpr int BLOCK_M = 128;   // token rows per tile (= reference BLOCK_M)
constexpr int BLOCK_N = 256;   // output columns per tile: 128 fp32 accumulators per consumer thread
constexpr int BLOCK_K = 64;    // 64 bf16 = 128 B = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int NSCHED = 4;
constexpr int CLAIM_AHEAD_KB = 16;   // the scheduler claims the next tile when this many k-blocks of the current one remain
constexpr int NUM_THREADS = 384;
constexpr int NUM_WARPS = NUM_THREADS / 32;
constexpr int EPI_WARP0 = 4;   // warps 4..11: warpgroup (warp - 4) / 4 owns tile rows [64g, 64g + 64), warp % 4 its 16-row slice
constexpr int NUM_EPI_WARPS = 8;

// Trace stamps (%globaltimer, FmParams::trace): TRACE_SLOTS per CTA, phase slots 0-15, then per-tile slots base + i for
// the first TRACE_TILES tiles of the CTA.  scripts/trace_gantt.py and scripts/trace_multi.py read them through
// flashmoe_b200/trace_slots.py, which keeps the same names (tests/test_trace_slots.py checks that the two agree).
constexpr int TRACE_SLOTS = 128;
constexpr int TRACE_TILES = 16;
enum TraceSlot : int {
    TRACE_START = 0,             // kernel entry
    TRACE_GATE_DONE = 1,         // router done, before the grid barrier
    TRACE_BARRIER = 2,           // past the grid barrier
    TRACE_DISPATCH_END = 3,      // warp 2 done with dispatch
    TRACE_FFN_START = 4,         // warp 4 enters the expert FFN
    TRACE_FFN_END = 5,           // every FFN role done
    TRACE_KERNEL_END = 6,
    TRACE_FIRST_TMA = 7,         // producer: first loads of the first tile issued
    TRACE_DISP_PREFIX = 8,       // dispatch: prefix over the chunk counts done
    TRACE_DISP_ROWS_DONE = 9,    // dispatch: local rows and the zero-fill complete (warp 4)
    TRACE_ZERO_ISSUED = 10,      // router: output-row zero-fill issued (warp 11)
    TRACE_GATE_LOGITS = 11,      // router: a sub-chunk's logits done
    TRACE_GATE_TOPK = 12,        // router: every sub-chunk's softmax / top-k done
    TRACE_FIRST_REMOTE = 13,     // scheduler: first tile of a packet from another rank ready
    TRACE_DONE_FLAGS = 14,       // fused completion: every expert's done flag seen
    TRACE_TOPK_WARP0 = 15,       // router: warp 0's softmax / top-k of a sub-chunk done
    TRACE_TILE_READY = 16,       // scheduler: the tile's dependencies resolved
    TRACE_TILE_FIRST_KB = 32,    // consumers: first k-block landed
    TRACE_TILE_MMA_DONE = 48,    // consumers: last MMA complete
    TRACE_TILE_EPI_START = 64,   // consumers: epilogue started
    TRACE_TILE_STORES = 80,      // consumers: epilogue stores issued (GEMM0: last h chunk handed over)
    TRACE_TILE_PUBLISHED = 96,   // publisher: tile published
    TRACE_TILE_CLAIMED = 112,    // scheduler: tile claimed
};
static_assert(TRACE_TILE_CLAIMED + TRACE_TILES == TRACE_SLOTS, "per-tile slots fill the buffer");

constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;                  // 16 KiB
constexpr int B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;                  // 32 KiB
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int STAGES = 4;
constexpr int PIPE_BYTES = STAGES * STAGE_BYTES;                      // 192 KiB
constexpr int EPI_ROW_BYTES = 128;                                    // 64 bf16; 16-byte pieces XOR-swizzled by (row & 7)
// The epilogue staging area: two h chunk buffers of 128 rows x 128 B (64 columns of a GEMM0 tile in the TMA's
// SWIZZLE_128B layout).  Consumer warp w owns rows [(w - 4) * 16, +16) of each buffer: it stages its rows of a GEMM0
// chunk there (the publisher warp stores the whole chunk with one TMA store), and its GEMM1 transpose tile is its rows
// of buffer 0.  No warp ever writes another warp's rows, so warps need no ordering among themselves here.
constexpr int EPI_CHUNK_BYTES = BLOCK_M * EPI_ROW_BYTES;              // 16 KiB
constexpr int EPI_BUFS = 2;
constexpr int EPI_BYTES = EPI_BUFS * EPI_CHUNK_BYTES;                 // 32 KiB
constexpr int OFF_EPI = PIPE_BYTES;                                   // 196608 (1 KiB aligned, as SWIZZLE_128B needs)
constexpr int OFF_BARS = OFF_EPI + EPI_BYTES;                         // 229376: the mbarriers (table below)
constexpr int GATE_STAGES = 8;                                        // router GEMM on tensor cores: up to 8 smem stages
constexpr int MAX_EXPERTS = 1024;   // validate_config rejects more; sizes the per-expert arrays below

// Shared-memory plan.  Four phases take turns in the stage area [0, PIPE_BYTES) and the epilogue staging area
// [OFF_EPI, OFF_EPI + EPI_BYTES); every alias below is one of these regions:
//
//   bytes             | router (G)               | dispatch (D)              | expert FFN (F)       | gather combine (C)
//   ------------------+--------------------------+---------------------------+----------------------+-------------------
//   stage [0, 64K)    | Wg chunks (GEMV) or      | x-row staging, 128 KiB    | pipeline stages,     | routing records
//                     | tensor-core stages       | (load issued at the end   | after BAR_DISP_DONE  | c_e/c_s/c_w/c_m,
//                     |                          | of gate_phase)            |                      | 128 KiB
//   [64K, 128K)       | logits [TS][E+1] f32     | (staging, cont.)          | (stages)             | (records, cont.)
//                     | (single-pass tensor-core |                           |                      |
//                     | stages overlay it)       |                           |                      |
//   [128K, 176K)      | sel_e i16 + rank i32,    | read                      | (stages)             |
//                     | G_SEL_MAX each           |                           |                      |
//   [176K, 188K)      | slot_ranks counts (on    | base / total / own,       | (stages)             |
//                     | base), gated score bias  | MAX_EXPERTS each          |                      |
//                     | (on total), training     |                           |                      |
//                     | column sums (on own)     |                           |                      |
//   epilogue [0, 8K)  | zero source of the       | read by the fill's bulk   | chunk buffers        |
//                     | output-row fill (warp 11)| stores until warps 4-11's |                      |
//                     |                          | wait_group.read           |                      |
//   epilogue [8K,32K) |                          | warp 2's remote-row       | chunk buffers, after |
//                     |                          | window (W > 1)            | NAMED_BAR_WINDOW     |
constexpr int G_OFF_WG = 0;                                // bf16 [EG][Hc] gate-weight chunks, or tensor-core stages
constexpr int G_WG_BYTES = 64 * 1024;
constexpr int G_OFF_LOGIT = G_OFF_WG + G_WG_BYTES;         // f32 [TS][E+1]
constexpr int G_LOGIT_BYTES = 64 * 1024;
constexpr int G_SEL_MAX = 8192;                            // max tpc * k (the host rejects more)
constexpr int G_OFF_SEL = G_OFF_LOGIT + G_LOGIT_BYTES;     // int16 sel_e[tpc * k]
constexpr int G_OFF_RANK = G_OFF_SEL + G_SEL_MAX * 2;      // int32 rank[tpc * k]
constexpr int D_OFF_BASE = G_OFF_RANK + G_SEL_MAX * 4;     // int32 base[E]: selections of e by lower chunks
constexpr int D_OFF_TOTAL = D_OFF_BASE + MAX_EXPERTS * 4;  // int32 total[E]: by all chunks
constexpr int D_OFF_OWN = D_OFF_TOTAL + MAX_EXPERTS * 4;   // int32 own[E]: by this chunk
constexpr int D_PREFIX_END = D_OFF_OWN + MAX_EXPERTS * 4;
constexpr int G_OFF_CNT = D_OFF_BASE;                      // int32 [E] slot_ranks' running counts
constexpr int G_OFF_COLSUM = D_OFF_OWN;                    // f32 [E] training: this chunk's sum_t p[t,e]
constexpr int G_OFF_BIAS = D_OFF_TOTAL;                    // f32 [E] gated launch: score_bias (0 without one)
constexpr int D_OFF_XROWS = 0;                             // staged token rows of this chunk
constexpr int D_XROWS_BYTES = 128 * 1024;
constexpr int C_OFF_E = 0;                                 // int32 [tpc * k] expert
constexpr int C_OFF_S = C_OFF_E + G_SEL_MAX * 4;           // int32 [tpc * k] slot
constexpr int C_OFF_W = C_OFF_S + G_SEL_MAX * 4;           // f32 [tpc * k] combine weight
constexpr int C_OFF_M = C_OFF_W + G_SEL_MAX * 4;           // f32 [tpc] mCw
constexpr int C_RECORDS_END = C_OFF_M + G_SEL_MAX * 4;
constexpr int EPI_OFF_ZERO = OFF_EPI;                      // zero source of the output-row fill
constexpr int EPI_ZERO_BYTES = 8 * 1024;
constexpr int D_OFF_WIN = EPI_OFF_ZERO + EPI_ZERO_BYTES;   // warp 2's remote-row window
constexpr int D_WIN_BYTES = OFF_EPI + EPI_BYTES - D_OFF_WIN;
static_assert(D_PREFIX_END <= PIPE_BYTES, "router and dispatch scratch within the stage area");
static_assert(D_OFF_XROWS + D_XROWS_BYTES <= G_OFF_SEL,
              "x-row staging below sel_e / rank: slot_ranks uses them while the first load is in flight");
static_assert(C_RECORDS_END <= PIPE_BYTES, "combine records within the stage area");
static_assert(D_WIN_BYTES > 0 && EPI_ZERO_BYTES + D_WIN_BYTES <= EPI_BYTES,
              "zero source and remote-row window within the epilogue staging area");
static_assert(G_OFF_COLSUM + MAX_EXPERTS * (int)sizeof(float) <= D_PREFIX_END, "a column sum per expert");
static_assert(G_OFF_BIAS >= G_OFF_CNT + MAX_EXPERTS * 4 && G_OFF_BIAS + MAX_EXPERTS * (int)sizeof(float) <= D_PREFIX_END,
              "a score bias per expert, clear of slot_ranks' counts");

// mbarriers (mbar_init / mbar_arrive / bar_wait on bar(smem, id)).  FM_MBARRIERS below declares every group once:
// X(ID, name, first id, count, arrival count); BAR_<ID> is the group's first id, ffn_setup initialises every barrier
// from it, and the host names a timed-out wait's barrier with mbar_name.  "+ tx": the arrival is an arrive.expect_tx,
// and the phase also waits for the TMA's bytes.
//
//   group       | arrive                                  | wait                          | orders
//   ------------+-----------------------------------------+-------------------------------+------------------------------
//   full        | producer (warp 0), + tx                 | consumer warps                | a pipeline stage's A and B
//               |                                         |                               | tiles landed
//   empty       | consumer warps, lane 0                  | producer                      | the MMAs have read the stage
//   sched_full  | scheduler (warp 3)                      | producer, publisher,          | a scheduler-ring slot's
//               |                                         | consumer warps                | TileInfo written
//   sched_empty | producer, publisher, consumer warps     | scheduler                     | every reader is done with
//               |                                         |                               | the slot
//   prod_take   | producer, CLAIM_AHEAD_KB k-blocks before| scheduler, before it claims   | bounds the scheduler's
//               | the end of the slot's tile              | the tile after the next       | look-ahead
//   xrows       | warp 1 (first group), warp 4 (the       | warps 4-11                    | a group of this chunk's x
//               | others), + tx                           |                               | rows staged
//   disp_done   | warp 4, or warp 2 (dense; more than     | producer, before its first    | dispatch is done with the
//               | RANGES_IN_REGS experts on several ranks)| tile                          | stage area
//   pub_full    | consumer warps, after a GEMM1 tile      | publisher                     | the tile's stores / adds
//               |                                         |                               | issued
//   pub_empty   | publisher                               | consumer warps                | the publisher took the slot
//   wg          | warp 0, + tx                            | every router thread           | a gate-weight chunk staged
//   remote      | warp 2, + tx                            | warp 2                        | the remote-row window filled
//   gfull       | warp 0, + tx                            | consumer warps                | a router tensor-core stage
//               |                                         |                               | landed
//   gempty      | consumer warps                          | warp 0                        | the router MMAs have read it
//   stg_full    | consumer warps, after fencing their     | publisher                     | an h chunk staged
//               | rows to the async proxy                 |                               |
//   stg_free    | publisher                               | consumer warps                | the TMA has read the chunk
//               |                                         |                               | buffer
#define FM_MBARRIERS(X)                                            \
    X(FULL,        full,         0, STAGES,      1)                 \
    X(EMPTY,       empty,        4, STAGES,      NUM_EPI_WARPS)     \
    X(SCHED_FULL,  sched_full,   8, NSCHED,      1)                 \
    X(SCHED_EMPTY, sched_empty, 12, NSCHED,      2 + NUM_EPI_WARPS) \
    X(PROD_TAKE,   prod_take,   16, NSCHED,      1)                 \
    X(XROWS,       xrows,       20, 1,           1)                 \
    X(DISP_DONE,   disp_done,   21, 1,           1)                 \
    X(PUB_FULL,    pub_full,    22, 2,           NUM_EPI_WARPS)     \
    X(PUB_EMPTY,   pub_empty,   24, 2,           1)                 \
    X(WG,          wg,          26, 1,           1)                 \
    X(REMOTE,      remote,      27, 1,           1)                 \
    X(GFULL,       gfull,       28, GATE_STAGES, 1)                 \
    X(GEMPTY,      gempty,      36, GATE_STAGES, NUM_EPI_WARPS)     \
    X(STG_FULL,    stg_full,    44, EPI_BUFS,    NUM_EPI_WARPS)     \
    X(STG_FREE,    stg_free,    46, EPI_BUFS,    1)

enum : int {
#define FM_MBAR_ID(ID, name, first, count, arrivals) BAR_##ID = (first),
    FM_MBARRIERS(FM_MBAR_ID)
#undef FM_MBAR_ID
};
#define FM_MBAR_COUNT(ID, name, first, count, arrivals) +(count)
constexpr int NUM_BARS = 0 FM_MBARRIERS(FM_MBAR_COUNT);   // 48
#undef FM_MBAR_COUNT

constexpr bool mbar_groups_contiguous() {
    int next = 0;
#define FM_MBAR_NEXT(ID, name, first, count, arrivals) \
    if ((first) != next) return false;                 \
    next += (count);
    FM_MBARRIERS(FM_MBAR_NEXT)
#undef FM_MBAR_NEXT
    return true;
}
static_assert(mbar_groups_contiguous(), "each mbarrier group starts where the one before it ends, the first at id 0");

// the group and index of barrier `id`, for the host's timeout message
struct MbarName { const char* group; int index; };
constexpr MbarName mbar_name(int id) {
#define FM_MBAR_NAME(ID, name, first, count, arrivals) \
    if (id >= (first) && id < (first) + (count)) return {#name, id - (first)};
    FM_MBARRIERS(FM_MBAR_NAME)
#undef FM_MBAR_NAME
    return {nullptr, id};
}
constexpr bool same_str(const char* a, const char* b) {
    while (*a != 0 && *a == *b) { ++a; ++b; }
    return *a == *b;
}
static_assert(same_str(mbar_name(0).group, "full") && mbar_name(0).index == 0 &&
              same_str(mbar_name(BAR_SCHED_FULL + 2).group, "sched_full") && mbar_name(BAR_SCHED_FULL + 2).index == 2 &&
              same_str(mbar_name(BAR_DISP_DONE).group, "disp_done") && mbar_name(BAR_DISP_DONE).index == 0 &&
              same_str(mbar_name(NUM_BARS - 1).group, "stg_free") && mbar_name(NUM_BARS - 1).index == EPI_BUFS - 1 &&
              mbar_name(NUM_BARS).group == nullptr,
              "mbar_name finds each barrier's group and index");

constexpr int OFF_RING = OFF_BARS + NUM_BARS * 8;                     // the scheduler ring: NSCHED TileInfo slots
constexpr int OFF_LAUNCH = OFF_RING + NSCHED * 64;                    // this launch's Launch record (below)
constexpr int SMEM_USED = OFF_LAUNCH + 64;
constexpr int SMEM_BYTES = SMEM_USED + 1024;                          // + slack for manual 1 KiB alignment
static_assert(OFF_BARS + NUM_BARS * (int)sizeof(uint64_t) == OFF_RING && OFF_BARS % 8 == 0,
              "the mbarriers fill [OFF_BARS, OFF_RING)");
static_assert(OFF_RING % 16 == 0, "ring entries are 16-byte aligned");
static_assert(SMEM_BYTES <= 232448, "227 KiB of dynamic shared memory per CTA");

__device__ __forceinline__ uint64_t* bar(uint8_t* smem, int id) { return reinterpret_cast<uint64_t*>(smem + OFF_BARS) + id; }

// Named barriers (named_sync / named_arrive; id 0 is __syncthreads).  Ids 2-7 are one protocol between warp 2 and warps
// 4-11, from dispatch into the consumers' first epilogue:
//
//   id | threads      | sync / arrive                        | orders
//   ---+--------------+--------------------------------------+----------------------------------------------------------
//   2  | DISP_THREADS | warps 2, 4-11                        | prefix arrays zeroed, then complete
//   3  | DISP_THREADS | 4-11 arrive, 2 syncs                 | this chunk's p.slot is written
//   4  | EPI_THREADS  | warps 4-11                           | x-row staging reuse; local row stores complete before acks
//   5  | DISP_THREADS | 2 arrives, 4-11 sync                 | warp 2 is done reading base / own in the stage area
//   6  | DISP_THREADS | 4-11 arrive, 2 syncs                 | local rows and the zero-fill complete before remote acks
//   7  | DISP_THREADS | 2 arrives, consumers sync before     | remote-row window handed back
//      |              | their first epilogue (W > 1)         |
//   8  | EPI_THREADS  | router consumer warpgroups           | tensor-core stages read before the logits are written
constexpr int EPI_THREADS = 32 * NUM_EPI_WARPS;    // warps 4-11
constexpr int DISP_THREADS = 32 + EPI_THREADS;     // warps 2, 4-11
constexpr int NAMED_BAR_PREFIX = 2;
constexpr int NAMED_BAR_SLOTS = 3;
constexpr int NAMED_BAR_LOCAL = 4;
constexpr int NAMED_BAR_PREFIX_READ = 5;
constexpr int NAMED_BAR_LOCAL_DONE = 6;
constexpr int NAMED_BAR_WINDOW = 7;
constexpr int NAMED_BAR_GATE_MMA = 8;

// The GEMMs of the expert FFN, FmParams::gemm[] ids.  GEMM0 (x.W_up^T) is even, its GEMM1 (h.W_down^T) the next id:
// kind = id & 1.  The shared expert's GEMMs run on the call's tokens, in row blocks of Launch::s_rb.
enum : int { GEMM_UP = 0, GEMM_DOWN = 1, GEMM_S_UP = 2, GEMM_S_DOWN = 3, NUM_GEMMS = 4 };

// One contiguous run of work items: all tiles of one GEMM of one packet.  16 bytes: the scheduler reads two of them for
// every item it claims, skipped items included, and a larger block measured slower on lists of many empty items.
struct __align__(16) TileBlock {
    unsigned short g[NUM_GEMMS];   // blocks of each GEMM before this one in the work list (block_start)
    int gemm;                      // GEMM_* (the sentinel: -1)
    int pkt;   // local packet index = src * nLx + le (the shared expert's: rank * nLx, its tokens are this rank's)
};
static_assert(sizeof(TileBlock) == 16 && 2 * MAX_EXPERTS + NUM_GEMMS <= 0xffff, "16-byte blocks, counts in 16 bits");

// Tensor maps of a launch, FmParams::tm[] ids (encoded by the host from one table in launch()).
enum : int {
    TM_A0,    // GEMM_UP's A: recv_x as [W*nLx*pEC, H] (dense: x as [n_tokens, H]), box {64, 128}
    TM_B0,    // expert_weights as [nLx*2*P, H], box {64, 256} (W_up rows); SwiGLU: [nLx*3*P, H], box {64, 128}
    TM_A1,    // hidden as [W*nLx*pEC, P], box {64, 128}: GEMM_DOWN's A loads and GEMM_UP's h stores
    TM_B1,    // expert_weights as [nLx*2*H, P] (SwiGLU: [nLx*3*H, P]), box {64, 256} (W_down rows)
    TM_GX,    // router on tensor cores: x as [n_tokens, H], box {64, 32}
    TM_GW,    // router on tensor cores: Wg_eff [E, H], box {64, min(128, E rounded up to 64)}
    TM_XS,    // shared expert: x as [n_tokens, H], box {64, 128}: GEMM_S_UP's A
    TM_WS0,   // W_up_s as [Ps, H], box {64, 256}; SwiGLU: the [3, Ps, H] tensor as [3*Ps, H], box {64, 128}
    TM_WS1,   // W_down_s (the same Ps*H block) as [H, Ps], box {64, 256}
    TM_HS,    // h_s as [S, Ps], box {64, 128}: GEMM_S_DOWN's A loads and GEMM_S_UP's h stores
    NUM_TMAPS
};

// Where a GEMM1 epilogue writes its rows, and how the publisher announces them (GemmOp::dest)
enum : int {
    DEST_RETURN = 0,   // the source rank's return buffer ret_y; g1_done, then the row block's return flag
    DEST_FUSED = 1,    // scaled into the tokens' output rows on the source rank; pkt_done, then the done flag
    DEST_Y_S = 2,      // y_s by token (the shared expert's s rows); s1_done
};

// Everything the FFN's warp roles need about one GEMM's operands, filled by the host per launch.  Tile (mblk, ntile) of
// packet pkt = src * nLx + le reads A rows pkt * a_pkt_rows + 128 mblk and B rows b_row0 + le * b_le_rows +
// tile_cols(op) * ntile.  A gated GEMM0 (SwiGLU, glu_rows != 0) reads 128 gate rows there and the 128 up rows glu_rows
// below them, and writes 128 columns of h = silu(g) * u per tile.
struct GemmOp {
    int a, b;               // FmParams::tm ids of the A and B operands (a GEMM0 stores h through its GEMM1's A map)
    int a_pkt_rows;         // A rows per packet: pEC, or 0 where the rows are the call's tokens
    int b_row0, b_le_rows;
    int kblocks;            // K / BLOCK_K
    int n, tn;              // output columns and column tiles, ceil(n / BLOCK_N)
    int from_packet;        // 1: the rows are a dispatched packet's (packet flag and row acks); 0: the call's tokens
    int bias_le;            // bias elements per local expert
    int done_pkt;           // GEMM0: done counters per packet (its row block's counter: done[pkt * done_pkt + mblk])
    int dest;               // GEMM1: DEST_*
    const __nv_bfloat16* bias;   // [n] per local expert, or nullptr
    unsigned int* done;     // GEMM0: its tiles finished per row block (g0_done, s0_done)
    int glu_rows;           // SwiGLU GEMM0: B rows from a tile's gate half to its up half (P, Ps); otherwise 0
};

// Output columns of one column tile: a gated GEMM0's 256-row B tile is two 128-row halves, gate and up.
__device__ __forceinline__ int tile_cols(const GemmOp& op) { return op.glu_rows ? BLOCK_N / 2 : BLOCK_N; }

// Where phase G takes a launch's routing from.  A caller-routed and a gated launch both store mcw = 1 and take the
// scaling combine for every k (k = 1 included); only the router launch copies y unscaled at k = 1.
enum RouteMode : int {
    ROUTE_ROUTER = 0,   // the built-in router: softmax, top-k, renormalise (fm_moe_forward, fm_moe_forward_tokens[_dev])
    ROUTE_CALLER = 1,   // the caller's top-k ids and weights (fm_moe_forward_routed)
    ROUTE_GATED = 2,    // the router's logits, scored and selected by the call's fm_router_t (fm_moe_forward_gated)
};
enum : int { SCORE_SOFTMAX = 0, SCORE_SIGMOID = 1 };   // FmParams::scoring (fm_router_t.scoring)
constexpr int MAX_GROUPS = 32;                        // n_group bound: a token's kept groups are one 32-bit mask

struct FmParams {
    CUtensorMap tm[NUM_TMAPS];   // TM_*; a map the launch does not use is zero
    GemmOp gemm[NUM_GEMMS];      // GEMM_*; the shared expert's are zero without one
    int tc_gate;        // 1 = logits by wgmma (E <= 256); 0 = register-blocked CUDA-core GEMV
    // The call's token count and everything derived from it are resolved on the device (resolve_launch, struct Launch).
    // n_tokens: the count itself, or with n_tokens_dev the context's S -- the rows of the maps over x and the bound of
    // *n_tokens_dev, which the kernel reads when it starts.  pEC and TCM are the context's maximum and are only strides
    // of the per-packet buffers.
    int n_tokens;
    const int* n_tokens_dev;
    int H, P, E, k, W, rank, nLx, pEC, TCM, act;
    int TN1, num_pkts, num_blocks;
    int drop_tokens, ec_mult;   // capacity EC(n) = (drop_tokens ? ceil(n / E) : n) * ec_mult, ec_mult = capacity_factor * k
    int dbg_flags;      // experiments only (results are garbage): bit0 = skip all TMA loads, bit1 = skip MMA issue,
                        // bit2 = skip the A loads, bit3 = skip the B loads
    unsigned long long timeout_ns;
    unsigned long long* launch_ctr;   // [1] launches this context has run (CTA 0 advances it after the grid barrier)
    int* launch_tokens;               // [1] the token count the last launch ran with
    const __nv_bfloat16 *x, *wg;
    __nv_bfloat16* out;
    int* topk_idx;             // [S,k]
    __nv_bfloat16* topk_w;     // [S,k]
    float* mcw;                // [S]
    int* slot;                 // [S,k]
    int* counts;               // [E]
    __nv_bfloat16* gate_out;   // [S,E]
    int* chunk_counts;         // [grid, E]
    unsigned int* claim;       // [1]
    unsigned int* g0_done;     // [num_pkts, TCM]
    unsigned int* g1_done;     // [num_pkts, TCM]
    unsigned long long* grid_bar;
    int* recv_cnt;             // [num_pkts]
    const TileBlock* blocks;   // [num_blocks + 1] (the sentinel's block_start = total_items)
    __nv_bfloat16* hidden;     // [W*nLx*pEC, P]
    __nv_bfloat16* recv_x;     // local symmetric: [W, nLx, pEC, H]
    unsigned long long* recv_flag;  // [W, nLx]  {epoch, rows}: published as soon as the source rank knows the count
    unsigned int* recv_rows;   // local symmetric [2, W*nLx, TCM]: rows of row block b of packet (src, le) that have landed,
                               // indexed by epoch parity (the other parity is zeroed by CTA 0 during this launch)
    __nv_bfloat16* ret_y;      // [E, pEC, H]
    unsigned long long* ret_flag;   // [E, TCM]
    __nv_bfloat16* peer_recv_x[FM_MAX_WORLD];
    unsigned long long* peer_recv_flag[FM_MAX_WORLD];
    unsigned int* peer_recv_rows[FM_MAX_WORLD];
    __nv_bfloat16* peer_ret_y[FM_MAX_WORLD];
    unsigned long long* peer_ret_flag[FM_MAX_WORLD];
    // fused GEMM1 -> combine path (fused != 0): the GEMM1 epilogue scales each row and adds it straight into the
    // source rank's output rows (peer REDG over NVLink); no return buffer, no per-row-block flags, no gather pass
    int fused;
    unsigned int* pkt_done;            // [num_pkts] GEMM1 tiles finished per packet
    uint4* recv_meta;                  // local symmetric [W*nLx*pEC] {token, p~ (f32 bits), mCw (f32 bits), 0}
    unsigned long long* done_flag;     // local symmetric [E] {epoch, 0}: expert e's contributions to my tokens are all in
    __nv_bfloat16* out_acc;            // my accumulation target: caller's out (W == 1) or the symmetric out buffer
    uint4* peer_recv_meta[FM_MAX_WORLD];
    unsigned long long* peer_done_flag[FM_MAX_WORLD];
    __nv_bfloat16* peer_out_acc[FM_MAX_WORLD];
    // training mode (is_training = 1): [2][2E+1] f32 by epoch parity = {gML[E] mean gate probability per expert,
    // gMeC[E] mean routed fraction per expert, loss} (reference moe/gate.cuh:608-635,698-706,763-773); nullptr otherwise
    float* aux;
    int dense;          // E == 1: no router GEMV, no dispatch copy; GEMM0 reads x in place (reference moe/fffn.cuh:31-167)
    // where phase G takes the routing from (RouteMode).  ROUTE_CALLER (fm_moe_forward_routed): the picks and weights
    // come from these [n, k] arrays instead of the router; -1 = no expert.  status_word: the election of the one thread
    // that reports an index outside [-1, E) in a launch (atomicExch of the epoch)
    int route;
    const int* routed_idx;
    const float* routed_w;
    unsigned int* status_word;
    // ROUTE_GATED (fm_moe_forward_gated): the router's logits, then scored_topk with this rule (fm_router_t, checked by
    // the host); score_bias [E] or nullptr, read when the launch starts
    int scoring, n_group, topk_group, group_top, renormalize;
    float route_scale;
    const float* score_bias;
    // shared expert (fm_moe_forward_shared; its GEMMs are gemm[GEMM_S_UP], gemm[GEMM_S_DOWN]): y_s [S, H] staging;
    // s0_done / s1_done [S / 128]: its GEMM0 / GEMM1 tiles finished per row block of tokens
    int shared;
    __nv_bfloat16* y_s;
    unsigned int *s0_done, *s1_done;
    // fm_set_weight_on_input on a caller or gated launch (k = 1): every dispatched row is rne_bf16(x[t] * w~) and the
    // combine takes weight 1 (recv_meta's p~ and the gather path's c_w); 0 on the router route
    int weight_on_input;
    DebugRecord* dbg;
    unsigned long long* trace;  // optional [grid][TRACE_SLOTS] %globaltimer stamps (nullptr = off)
};
static_assert(sizeof(FmParams) <= 4096, "kernel parameters within the 4 KiB every launch path accepts");

// Launch state.  Nothing that changes from launch to launch is a kernel parameter, so a launch captured in a CUDA graph
// computes the right values on every replay: every CTA reads the context's launch counter (and, for a device-side count,
// the count) when it starts and derives the rest.  Launch L = counter + 1 has epoch (uint32) L -- the tag of every flag
// it publishes -- and waits at the grid barrier for the monotonic arrival count L * grid.  CTA 0 stores L after the grid
// barrier, when every CTA of the launch has read the old value; the next launch on the stream sees the new one.
struct Launch {
    unsigned long long launch;       // L
    unsigned long long bar_target;   // L * grid
    unsigned int epoch;              // (uint32) L
    int S;                           // this call's tokens (0 when a device-side count is out of range)
    int EC;                          // its capacity EC(S)
    int tpc;                         // tokens per CTA, ceil(S / grid)
    int tcm_items;                   // row blocks per packet in the work list: TCM of EC at W == 1, the maximum TCM at W > 1
    int total_items;                 // work items of the launch
    int s_rb;                        // the shared expert's row blocks of tokens, ceil(S / 128) (0 without one)
};
static_assert(sizeof(Launch) <= SMEM_USED - OFF_LAUNCH, "the Launch record's shared-memory slot");

// row blocks of each block of GEMM g in this launch: a packet's tcm_items, or the shared expert's s_rb
__device__ __forceinline__ int gemm_row_blocks(const Launch& L, int g) {
    return g < GEMM_S_UP ? L.tcm_items : L.s_rb;
}

// first work item of block b: every earlier block of GEMM g holds its row blocks times its column tiles, so the item
// space follows the call's row-block counts without rebuilding the table (the shared expert's blocks are empty without
// one: s_rb = 0, and every item id is the routed list's)
__device__ __forceinline__ int block_start(const FmParams& p, const Launch& L, const TileBlock& b) {
    int start = 0;
#pragma unroll
    for (int g = 0; g < NUM_GEMMS; ++g) start += b.g[g] * p.gemm[g].tn * gemm_row_blocks(L, g);
    return start;
}

// one thread per CTA, before the prologue's block sync
__device__ __forceinline__ void resolve_launch(const FmParams& p, Launch* L) {
    const unsigned long long launch = *reinterpret_cast<const volatile unsigned long long*>(p.launch_ctr) + 1ull;
    int n = p.n_tokens;
    if (p.n_tokens_dev != nullptr) {
        const int v = *reinterpret_cast<const volatile int*>(p.n_tokens_dev);
        n = (v < 0 || v > p.n_tokens) ? 0 : v;
        // an out-of-range count must not trap (every rank takes part in the collective): the launch runs as n = 0 and
        // the host reports the count at its next check
        if (n != v && blockIdx.x == 0) fm_record(p.dbg, FM_STATUS_BAD_COUNT, (unsigned int)v, (unsigned int)p.n_tokens, 0, 0);
    }
    const int G = (int)gridDim.x;
    const int ec = (p.drop_tokens ? (n + p.E - 1) / p.E : n) * p.ec_mult;
    L->launch = launch;
    L->bar_target = launch * (unsigned long long)G;
    L->epoch = (unsigned int)launch;
    L->S = n;
    L->EC = ec;
    L->tpc = (n + G - 1) / G;
    // one rank knows every packet's capacity, so the work list shrinks to this call's row blocks; a receiver with peers
    // does not know their token counts and keeps the maximum (the empty row blocks are skipped by the scheduler)
    L->tcm_items = p.W == 1 ? (ec + BLOCK_M - 1) / BLOCK_M : p.TCM;
    L->s_rb = p.shared ? (n + BLOCK_M - 1) / BLOCK_M : 0;
    L->total_items = block_start(p, *L, p.blocks[p.num_blocks]);
}

// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void trace_stamp(const FmParams& p, int slot) {
    if (p.trace != nullptr && slot < TRACE_SLOTS)
        p.trace[(size_t)blockIdx.x * TRACE_SLOTS + slot] = globaltimer_ns();
}

// per-tile stamp `base` (TRACE_TILE_*) of this CTA's tile n; only the first TRACE_TILES tiles have slots
__device__ __forceinline__ void trace_tile(const FmParams& p, int base, int n) {
    if (n < TRACE_TILES) trace_stamp(p, base + n);
}

// wait for the phase of parity `parity` of mbarrier `id` to complete; a timeout traps with FM_TRAP_MBAR (id, parity)
__device__ __forceinline__ void bar_wait(const FmParams& p, uint8_t* smem, int id, uint32_t parity) {
    mbar_wait(bar(smem, id), parity, p.dbg, p.timeout_ns, (unsigned int)id);
}

template <int N>
struct Ring {   // a cursor over a ring of N mbarrier-guarded slots: the slot and the parity of its current phase
    int i = 0;
    uint32_t phase = 0;
    __device__ __forceinline__ void next() {
        if (++i == N) { i = 0; phase ^= 1u; }
    }
};

__device__ __forceinline__ void grid_barrier(const FmParams& p, const Launch& L) {
    __syncthreads();
    if (threadIdx.x == 0) {
        atom_acq_rel_gpu_add_u64(p.grid_bar, 1ull);
        SpinGuard g;
        while (ld_acquire_gpu_u64(p.grid_bar) < L.bar_target)
            g.tick(p.dbg, p.timeout_ns, FM_TRAP_GRID_BARRIER, 0, 0, 0);
    }
    __syncthreads();
}

// sum over lanes of acc[i] ends up in lane i (31 shuffles instead of 160)
__device__ __forceinline__ float warp_transpose_reduce(float (&acc)[32], int lane) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const bool upper = (lane & off) != 0;
#pragma unroll
        for (int j = 0; j < off; ++j) {
            const float send = upper ? acc[j] : acc[j + off];
            const float keep = upper ? acc[j + off] : acc[j];
            acc[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
    return acc[0];
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
    f[0] = __uint_as_float(v.x << 16); f[1] = __uint_as_float(v.x & 0xffff0000u);
    f[2] = __uint_as_float(v.y << 16); f[3] = __uint_as_float(v.y & 0xffff0000u);
    f[4] = __uint_as_float(v.z << 16); f[5] = __uint_as_float(v.z & 0xffff0000u);
    f[6] = __uint_as_float(v.w << 16); f[7] = __uint_as_float(v.w & 0xffff0000u);
}

// ============================================================================================================
// Phase G: router.  CTA b owns tokens [b*tpc, min(S, (b+1)*tpc)).
//   logits[t,e] = sum_h x[t,h] * Wg_eff[e,h]       Wg_eff = gate_weights viewed flat as [E,H]  (moe.cuh:107-109)
//   softmax with the reference's online recurrence and fast intrinsics (gate.cuh:575-584), top-k by k rounds of
//   strict-'>' scans in ascending expert order on fp32 p (gate.cuh:654-670), mCw = sum of the picked p.
//   Slots: ascending-token order within the CTA's chunk here; chunk bases after the grid barrier (a legal
//   interleaving of the reference's BlockScan + atomicAdd(eC) order, gate.cuh:678-718).
// ============================================================================================================
// Router logits on the tensor cores (E <= 256): logits[t, e] = sum_h x[t,h] * Wg_eff[e,h] for one sub-chunk of <= 128 tokens
// of this CTA with wgmma: A = the tokens' x rows (TMA, 32-row boxes straight from x), B = Wg_eff in groups of
// GB = min(128, E rounded up to 64) rows (TMA; rows past E read as zero).  Warp 0 loads; the two consumer warpgroups
// (warps 4-11; warpgroup g = token rows [64g, 64g + 64), idle when the sub-chunk has none there) multiply into a GB-column
// register accumulator and write the logits straight into the logits scratch, where the softmax / top-k code finds them
// exactly like after the GEMV.  E > 128 takes one pass over H per group of 128 experts; the stages then stay clear of the
// logits scratch, which the earlier pass has already filled.
// The reference computes the same product with mma.sync tiles padded to 64 experts (gate.cuh:526-535); fp32 accumulation
// order differs between the two (and from the oracle's), which is what the oracle's ambiguity flags are for.
struct GateTcState { int gkb; };
__device__ __forceinline__ void gate_logits_tc(const FmParams& p, uint8_t* smem, int t0, int s0, int n_sub, int rows_cap,
                                               float* logit_s, int ldl, GateTcState& st) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = p.E, E64 = (E + 63) & ~63;
    const int GB = min(128, E64);                                // Wg_eff rows per pass (the tensor map's box height)
    const int npass = (E64 + GB - 1) / GB;                      // 1, or 2 for 129 <= E <= 256
    const int b_bytes = GB * BLOCK_K * 2;
    const int nk = p.H / BLOCK_K;
    const int nb32 = (n_sub + 31) / 32;                          // 32-row boxes of x per k-block
    const uint32_t tx = (uint32_t)(nb32 * 32 * BLOCK_K * 2 + b_bytes);
    // Stages live in the router's weight + logits scratch; compact stride = what a FULL sub-chunk stages (x rows rounded
    // up to a warpgroup's 64), so a 28-token chunk with 64 experts gets 5 stages of 24 KB.  The layout (stride, stage
    // count, offset of the Wg rows) is the same for every sub-chunk of the launch -- the stage / phase arithmetic runs
    // across sub-chunks -- only the number of x boxes loaded follows the sub-chunk's row count.
    const int a_cap = ((rows_cap + 63) / 64) * 64 * BLOCK_K * 2;
    const int stage_bytes = (a_cap + b_bytes + 1023) & ~1023;
    const int region = npass > 1 ? G_WG_BYTES : G_WG_BYTES + G_LOGIT_BYTES;
    const int NS = max(1, min(GATE_STAGES, region / stage_bytes));
    for (int pass = 0; pass < npass; ++pass) {
        const int e0 = pass * GB;
        if (warp == 0 && lane == 0) {          // TMA issuer
            fence_proxy_async_smem();          // earlier generic accesses of the scratch (logits, softmax) -> TMA writes
            for (int kb = 0; kb < nk; ++kb) {
                const int g = st.gkb + kb, s = g % NS;
                const uint32_t ph = (uint32_t)(g / NS) & 1u;
                bar_wait(p, smem, BAR_GEMPTY + s, ph ^ 1u);
                uint8_t* sa = smem + G_OFF_WG + s * stage_bytes;
                uint64_t* full = bar(smem, BAR_GFULL + s);
                mbar_arrive_expect_tx(full, tx);
                for (int j = 0; j < nb32; ++j) tma_load_2d(sa + j * 4096, &p.tm[TM_GX], kb * BLOCK_K, t0 + s0 + j * 32, full);
                tma_load_2d(sa + a_cap, &p.tm[TM_GW], kb * BLOCK_K, e0, full);
            }
        } else if (warp >= EPI_WARP0) {        // consumer warpgroups
            const int wg = (warp - EPI_WARP0) >> 2;
            const bool active = wg * 64 < n_sub;   // warpgroup-uniform
            // one accumulator of 64 or 128 expert columns (the m64n64 fragment is the first half of the m64n128 one)
            float acc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[i] = 0.0f;
            for (int kb = 0; kb < nk; ++kb) {
                const int g = st.gkb + kb, s = g % NS;
                const uint32_t ph = (uint32_t)(g / NS) & 1u;
                bar_wait(p, smem, BAR_GFULL + s, ph);
                if (active) {
                    const uint32_t sa = smem_u32(smem + G_OFF_WG + s * stage_bytes);
                    const uint64_t da = gmma_smem_desc_sw128(sa + wg * 64 * 128);
                    const uint64_t db = gmma_smem_desc_sw128(sa + a_cap);
                    wgmma_fence_regs(acc);   // the accumulator's register writes stay ahead of the fence
                    wgmma_fence();
                    if (GB > 64) {
#pragma unroll
                        for (int kk = 0; kk < BLOCK_K / WGMMA_K; ++kk)
                            wgmma_m64n128k16_bf16(acc, da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2));
                    } else {
#pragma unroll
                        for (int kk = 0; kk < BLOCK_K / WGMMA_K; ++kk)
                            wgmma_m64n64k16_bf16(reinterpret_cast<float(&)[32]>(acc), da + (uint64_t)(kk * 2),
                                                 db + (uint64_t)(kk * 2));
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    wgmma_fence_regs(acc);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(bar(smem, BAR_GEMPTY + s));
            }
            // both warpgroups are done reading the stages (which may overlap the logits scratch)
            named_sync<NAMED_BAR_GATE_MMA, EPI_THREADS>();
            if (active) {
                const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = (lane & 3) * 2;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    if (j * 8 >= GB) break;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = r0 + 8 * h, col = e0 + j * 8 + cq;
                        if (row < n_sub) {
                            if (col < E) logit_s[row * ldl + col] = acc[j * 4 + 2 * h];
                            if (col + 1 < E) logit_s[row * ldl + col + 1] = acc[j * 4 + 2 * h + 1];
                        }
                    }
                }
            }
        }
        st.gkb += nk;
    }
}

// E == 1 (reference: the dense fffn kernel is selected instead of the MoE kernel, moe.cuh:174-177): every token goes to
// expert 0 with probability 1, slot = token index, nothing is dropped (EC >= S).  No GEMV, no softmax.
__device__ __forceinline__ void gate_phase_dense(const FmParams& p, const Launch& L, int t0, int n_tok) {
    const int tid = threadIdx.x;
    for (int i = tid; i < n_tok; i += NUM_THREADS) {
        const int t = t0 + i;
        p.topk_idx[t] = 0;
        p.topk_w[t] = __float2bfloat16_rn(1.0f);
        p.mcw[t] = 1.0f;
        p.gate_out[t] = __float2bfloat16_rn(1.0f);
        p.slot[t] = t;
    }
    if (blockIdx.x == 0 && tid == 0) {
        p.counts[0] = L.S;   // this call's tokens
        p.recv_cnt[0] = L.S;
        if (p.aux != nullptr && L.S > 0) {   // mean probability 1, routed fraction 1, loss 1 * 1 / 1 (no tokens: all zero)
            float* a = p.aux + (size_t)(L.epoch & 1u) * 3;
            a[0] = 1.0f; a[1] = 1.0f; a[2] = 1.0f;
        }
    }
}

// Router logits on the CUDA cores: logits[t, e] = sum_h x[t,h] * Wg_eff[e,h] for one sub-chunk of n_sub tokens of this
// CTA, accumulated into the logits scratch.  Wg_eff is staged by the TMA engine in groups of up to 128 experts by chunks
// of H; the x rows are read straight from global memory.
__device__ __forceinline__ void gate_logits_gemv(const FmParams& p, uint8_t* smem, int t0, int s0, int n_sub,
                                                 float* logit_s, int ldl, uint32_t& wgphase) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = p.E, H = p.H;
    __nv_bfloat16* wg_s = reinterpret_cast<__nv_bfloat16*>(smem + G_OFF_WG);
    uint64_t* wgbar = bar(smem, BAR_WG);   // initialised in the kernel prologue
    const int EG = E < 128 ? E : 128;                      // experts staged per group
    int Hc = (G_WG_BYTES / (EG * 2)) & ~255;               // H columns staged per chunk (multiple of 256)
    if (Hc > H) Hc = H;
    for (int i = tid; i < n_sub * ldl; i += NUM_THREADS) logit_s[i] = 0.0f;
    for (int eg0 = 0; eg0 < E; eg0 += EG) {
        const int eg_len = min(EG, E - eg0);
        for (int hc0 = 0; hc0 < H; hc0 += Hc) {
            const int hc_len = min(Hc, H - hc0);
            __syncthreads();  // previous users of wg_s are done (also orders the logit_s zero fill)
            // stage Wg_eff[eg0 .. eg0+eg_len, hc0 .. hc0+hc_len) -> wg_s[e][Hc] through the TMA engine (1-D bulk copies,
            // one per expert row, or a single one when the rows are contiguous on both sides): no register round trip,
            // and the copy runs under the x loads issued below
            if (warp == 0) {
                if (lane == 0) {
                    fence_proxy_async_smem();   // earlier generic accesses to this scratch -> async-proxy writes
                    mbar_arrive_expect_tx(wgbar, (uint32_t)(eg_len * hc_len * 2));
                }
                __syncwarp();
                if (hc_len == H && Hc == H) {
                    if (lane == 0) bulk_load_1d(wg_s, p.wg + (size_t)eg0 * H, (uint32_t)(eg_len * H * 2), wgbar);
                } else {
                    for (int e = lane; e < eg_len; e += 32)
                        bulk_load_1d(wg_s + (size_t)e * Hc, p.wg + (size_t)(eg0 + e) * H + hc0, (uint32_t)(hc_len * 2), wgbar);
                }
            }
            const bool single = hc_len <= 1024;
            uint4 xv[4][4];
            // the first token block's x rows (HBM) are requested while Wg is in flight, so both latencies overlap
            if (single && warp * 4 < n_sub) {
                const int ntk0 = min(4, n_sub - warp * 4);
                const __nv_bfloat16* xr0 = p.x + (size_t)(t0 + s0 + warp * 4) * H + hc0;
#pragma unroll
                for (int tk = 0; tk < 4; ++tk)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int h = i * 256 + lane * 8;
                        xv[tk][i] = (tk < ntk0 && h < hc_len) ? ld_global_nc_v4(xr0 + (size_t)tk * H + h)
                                                              : make_uint4(0u, 0u, 0u, 0u);
                    }
            }
            bar_wait(p, smem, BAR_WG, wgphase);
            wgphase ^= 1;
            // register-blocked GEMV: a warp takes 4 tokens x 8 experts at a time (32 accumulators per lane, one per
            // (token, expert) pair), lanes split the H columns in 16-byte pieces; all of a step's global loads are
            // issued before the first FMA, and each staged Wg piece is reused by the 4 tokens.
            for (int tb = warp * 4; tb < n_sub; tb += NUM_WARPS * 4) {
                const int ntk = min(4, n_sub - tb);
                const __nv_bfloat16* xr = p.x + (size_t)(t0 + s0 + tb) * H + hc0;
                if (single && tb != warp * 4) {
#pragma unroll
                    for (int tk = 0; tk < 4; ++tk)
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int h = i * 256 + lane * 8;
                            xv[tk][i] = (tk < ntk && h < hc_len) ? ld_global_nc_v4(xr + (size_t)tk * H + h)
                                                                 : make_uint4(0u, 0u, 0u, 0u);
                        }
                }
                for (int g8 = 0; g8 * 8 < eg_len; ++g8) {
                    const int ne = min(8, eg_len - g8 * 8);
                    float acc[32];
#pragma unroll
                    for (int e = 0; e < 32; ++e) acc[e] = 0.0f;
                    for (int pg = 0; pg < hc_len; pg += 1024) {
                        if (!single) {
#pragma unroll
                            for (int tk = 0; tk < 4; ++tk)
#pragma unroll
                                for (int i = 0; i < 4; ++i) {
                                    const int h = pg + i * 256 + lane * 8;
                                    xv[tk][i] = (tk < ntk && h < hc_len) ? ld_global_nc_v4(xr + (size_t)tk * H + h)
                                                                         : make_uint4(0u, 0u, 0u, 0u);
                                }
                        }
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int h = pg + i * 256 + lane * 8;
                            if (h < hc_len) {
                                const __nv_bfloat16* wrow = wg_s + (size_t)(g8 * 8) * Hc + h;
                                float xf[4][8];   // the 4 tokens' 8 columns, unpacked once per piece
#pragma unroll
                                for (int tk = 0; tk < 4; ++tk) unpack8(xv[tk][i], xf[tk]);
#pragma unroll
                                for (int e = 0; e < 8; ++e) {
                                    if (e < ne) {
                                        float wf[8];
                                        unpack8(*reinterpret_cast<const uint4*>(wrow + (size_t)e * Hc), wf);
#pragma unroll
                                        for (int tk = 0; tk < 4; ++tk)
#pragma unroll
                                            for (int q = 0; q < 8; ++q)
                                                acc[tk * 8 + e] = fmaf(xf[tk][q], wf[q], acc[tk * 8 + e]);
                                    }
                                }
                            }
                        }
                    }
                    const float tot = warp_transpose_reduce(acc, lane);   // lane -> (token lane/8, expert lane%8)
                    const int tk = lane >> 3, e = lane & 7;
                    if (tk < ntk && e < ne) logit_s[(tb + tk) * ldl + eg0 + g8 * 8 + e] += tot;
                }
            }
        }
    }
}

// The accumulation rows of this chunk's tokens start at zero (reference clearState zeroes the output,
// moe.cuh:43-48).  Done by the TMA engine from a zeroed piece of the (still unused) epilogue staging area, so no
// thread stalls on a store queue (as plain stores this cost 1.5-3 us on the router's critical path wherever it was
// placed), and issued by gate_phase only after the first sub-chunk's logits: the engine works in order, and at the start
// of the kernel these stores sat in front of the gate-weight load (+5 us).  The LAST warp issues them (softmax_topk
// fills the warps from 0 upwards: with config B's 28 tokens per CTA warps 7-11 have none, and as warp 4's job
// the 3 us of this block were on the router's critical path) and waits for them in dispatch_phase before the
// local rows are acknowledged -- an expert only adds into a token's row after an acknowledgement of this CTA.
__device__ __forceinline__ void zero_fill_out_rows(const FmParams& p, uint8_t* smem, int t0, int n_tok) {
    const int lane = threadIdx.x & 31, H = p.H;
    uint8_t* zbuf = smem + EPI_OFF_ZERO;
    const int row_bytes = H * 2, zbytes = min(row_bytes, EPI_ZERO_BYTES);
    for (int i = lane * 16; i < zbytes; i += 512) *reinterpret_cast<uint4*>(zbuf + i) = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async_smem();
    __syncwarp();
    const int pieces = row_bytes / zbytes;   // H is a multiple of 64, rows above 8 KiB are multiples of 8 KiB or handled below
    for (int i = lane; i < n_tok * pieces; i += 32)
        bulk_store_1d(reinterpret_cast<uint8_t*>(p.out_acc + (size_t)(t0 + i / pieces) * H) + (size_t)(i % pieces) * zbytes, zbuf,
                      (uint32_t)zbytes);
    const int rem = row_bytes - pieces * zbytes;   // (row_bytes not a multiple of 8 KiB: the tail of every row)
    if (rem > 0)
        for (int i = lane; i < n_tok; i += 32)
            bulk_store_1d(reinterpret_cast<uint8_t*>(p.out_acc + (size_t)(t0 + i) * H) + (size_t)pieces * zbytes, zbuf, (uint32_t)rem);
    bulk_commit_group();
    if (lane == 0) trace_stamp(p, TRACE_ZERO_ISSUED);
}

// Lanes per token of softmax_topk: pow2ceil(E) up to 8 experts (one expert per lane), then 4 / 8 / 16 / 32, so that a
// lane owns at most 32 experts.
__device__ __forceinline__ int softmax_topk_lanes(int E) {
    if (E > 8) return E <= 128 ? 4 : E <= 256 ? 8 : E <= 512 ? 16 : 32;
    int lpt = 1;
    while (lpt < E) lpt <<= 1;
    return lpt;
}

// Softmax and top-k of one sub-chunk, for every E in [1, 1024]: a group of LPT = softmax_topk_lanes(E) lanes per token,
// lane `sub` owns experts sub, sub + LPT, ... (C = ceil(E / LPT) <= 32 of them), 32 / LPT tokens per warp, so that a
// sub-chunk of up to 96 tokens at E > 8 is one round of the CTA's 12 warps (the recurrence is a dependent chain of E
// steps per token whatever the lane count; one lane per expert would serialise 111 tokens of the 16k-token sweep point
// into 10 rounds, a thread per token leaves one or two warps doing ~5 E dependent steps each: 17 us at E = 128 with 56
// tokens).  Every lane of a group runs the reference's sequential online-softmax recurrence (gate.cuh:575-584) itself;
// a lane scans its own experts in ascending order with a strict '>', the group reduction prefers the larger value and,
// on equal values, the lower index -- together the reference's ascending scan (gate.cuh:654-670).  A round in which no
// expert compares greater than -inf (a token with NaN logits) picks expert 0, like the reference's scan.  Writes
// gate_out, topk_idx, topk_w, mcw and sel_e, and leaves the probabilities in the logits scratch (the training-mode
// column sums read them).
// The probabilities of one token (row l of the logits scratch, gate_out row go) for a group of LPT lanes: every lane of
// the group runs the reference's recurrence over the whole row, then lane `sub` replaces its experts' logits by p and
// writes them to gate_out (idle groups, !valid, only compute).  softmax_topk and scored_topk share it, so a gated
// launch's softmax scores are the router's bits.  (No FmParams argument: out of line, in scored_topk, every field read
// through the reference would be reloaded after each store.)
__device__ __forceinline__ void softmax_row(float* l, __nv_bfloat16* go, int E, int sub, int LPT, bool valid) {
    float dI = 0.0f, mI = -INFINITY;
    // (unrolled so that the loads, the running maxima and the exponentials of 8 steps are in flight together;
    // the dependent chain is then one max and one fma per step -- same operations in the same order)
#pragma unroll 8
    for (int e = 0; e < E; ++e) {
        const float pM = mI;
        mI = fmaxf(mI, l[e]);
        dI = fmaf(dI, fast_expf(pM - mI), fast_expf(l[e] - mI));
    }
    __syncwarp();   // every lane of the group has read the logits before they are replaced by probabilities
    if (valid)
#pragma unroll 4
        for (int e = sub; e < E; e += LPT) {
            const float pe = __fdividef(fast_expf(l[e] - mI), dI);
            l[e] = pe;
            go[e] = __float2bfloat16_rn(pe);
        }
}

__device__ __forceinline__ void softmax_topk(const FmParams& p, float* logit_s, int ldl, int16_t* sel_e, int t0, int s0,
                                             int n_sub) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int E = p.E, k = p.k;
    const int LPT = softmax_topk_lanes(E), lg = __ffs(LPT) - 1;   // shifts: the compiler cannot see LPT is a power of 2
    const int TPW = 32 >> lg, sub = lane & (LPT - 1);
    for (int tb = warp * TPW; tb < n_sub; tb += NUM_WARPS * TPW) {
        const int ti_raw = tb + (lane >> lg);
        const bool valid = ti_raw < n_sub;
        const int ti = valid ? ti_raw : n_sub - 1;   // (idle groups compute on a copy of the last row, write nothing)
        float* l = logit_s + ti * ldl;
        const int t = t0 + s0 + ti;
        softmax_row(l, p.gate_out + (size_t)t * E, E, sub, LPT, valid);
        unsigned int taken = 0u;
        float sum = 0.0f;
        for (int i = 0; i < k; ++i) {
            float bv = -INFINITY;
            int bi = 0x7fffffff;
            if (valid) {
                int c = 0;
#pragma unroll 4
                for (int e = sub; e < E; e += LPT, ++c) {
                    const float v = l[e];
                    if (v > bv && !((taken >> c) & 1u)) { bv = v; bi = e; }
                }
            }
            for (int off = LPT >> 1; off >= 1; off >>= 1) {
                const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
                if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (bi == 0x7fffffff) { bi = 0; }   // nothing comparable left (NaN logits): the reference's default
            if ((bi & (LPT - 1)) == sub) taken |= 1u << (bi >> lg);
            sum += bv;
            if (sub == 0 && valid) {
                p.topk_idx[(size_t)t * k + i] = bi;
                p.topk_w[(size_t)t * k + i] = __float2bfloat16_rn(bv);
                sel_e[(s0 + ti) * k + i] = (int16_t)bi;
            }
        }
        if (sub == 0 && valid) p.mcw[t] = sum;
        __syncwarp();
    }
}

// Sigmoid score of a gated launch: 1 / (1 + 2^fl(-l * log2e)), the power by ex2.approx.ftz (fast_expf), the sum and
// the reciprocal rounded to nearest.  Relative error against 1 / (1 + e^-l): at most 2^-21 (ex2) + 2^-24 * |l| (the
// rounded argument) + 2 * 2^-24 (sum, reciprocal), to first order; l = -inf or below about -88 gives +0, +inf gives 1.
__device__ __forceinline__ float sigmoid_score(float l) { return __frcp_rn(__fadd_rn(1.0f, fast_expf(-l))); }

// Best candidate of a group of LPT lanes: the larger value, on equal values the lower index (every lane ends with the
// group's winner).  Index 0x7fffffff = nothing compared greater than -inf.
__device__ __forceinline__ void group_argmax(float& bv, int& bi, int LPT) {
    for (int off = LPT >> 1; off >= 1; off >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
}

// Scores and top-k of one sub-chunk of a gated launch (fm_moe_forward_gated), for every E in [2, 1024], on
// softmax_topk's lane groups (lane `sub` owns experts sub, sub + LPT, ...):
//   s_e = the router's softmax probability (softmax_row) or sigmoid_score(l_e), left in the logits scratch and
//         written to gate_out;
//   c_e = fl(s_e + b_e) with b = the staged score bias (zeros without one: s + 0 = s), for selection only;
//   n_group > 1: lane `sub` scores its groups sub, sub + LPT, ... (G_g = the largest c of the group, or fl(largest +
//         second largest)); topk_group argmax rounds give the kept-group mask, and the experts of the other groups
//         start out in `taken`, so the k rounds below never pick them;
//   k rounds of softmax_topk's scan on c (strict '>', lower index on equal values, NaN never greater, a round with
//         nothing greater than -inf takes index 0 -- groups and experts alike);
//   w_j = s_{e_j}; renormalize: W = sum of the w_j in pick order from +0, w_j = W > 0 ? w_j / W : 0 (rounded
//         division); then w_j = fl(w_j * scale).
// Writes gate_out, topk_idx, topk_w = rne_bf16(w), mcw = 1 and sel_e.  Called by every thread of the CTA.  Out of line
// on purpose, like gate_phase_routed, and with few arguments: the kernel keeps the router path's registers, stack and
// spills.  (Inlined, the kernel's spills rose from 156 / 544 B to 184 / 584 B; out of line with the scratch pointers
// as arguments to 164 / 572 B; a whole gated gate_phase out of line grew the kernel's stack from 256 to 432 B.)
__device__ __noinline__ void scored_topk(const FmParams& p, uint8_t* smem, int t0, int s0, int n_sub) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // every field this stage uses, read once: p is a reference here (out of line), and a field read through it in a
    // loop is reloaded after every store
    const int E = p.E, k = p.k;
    const int scoring = p.scoring, NG = p.n_group, topk_group = p.topk_group, group_top = p.group_top;
    const bool renormalize = p.renormalize != 0;
    const float scale = p.route_scale;
    __nv_bfloat16* const gate_out = p.gate_out;
    int* const topk_idx = p.topk_idx;
    __nv_bfloat16* const topk_w = p.topk_w;
    float* const mcw = p.mcw;
    float* logit_s = reinterpret_cast<float*>(smem + G_OFF_LOGIT);
    int16_t* sel_e = reinterpret_cast<int16_t*>(smem + G_OFF_SEL);
    const int ldl = E + 1;
    float* bias_s = reinterpret_cast<float*>(smem + G_OFF_BIAS);
    if (s0 == 0) {   // the launch's first sub-chunk: stage the bias (read once per launch, so a captured graph follows
                     // in-place updates of it)
        const float* score_bias = p.score_bias;
        for (int e = threadIdx.x; e < E; e += NUM_THREADS) bias_s[e] = score_bias != nullptr ? score_bias[e] : 0.0f;
        __syncthreads();
    }
    const int LPT = softmax_topk_lanes(E), lg = __ffs(LPT) - 1;
    const int TPW = 32 >> lg, sub = lane & (LPT - 1);
    const int GS = E / NG;
    // groups per lane: NG <= 32, and LPT >= 4 for E > 8, LPT >= E >= NG below -- at most 8
    constexpr int GPL = MAX_GROUPS / 4;
    for (int tb = warp * TPW; tb < n_sub; tb += NUM_WARPS * TPW) {
        const int ti_raw = tb + (lane >> lg);
        const bool valid = ti_raw < n_sub;
        const int ti = valid ? ti_raw : n_sub - 1;   // (idle groups compute on a copy of the last row, write nothing)
        float* l = logit_s + ti * ldl;
        const int t = t0 + s0 + ti;
        __nv_bfloat16* const go = gate_out + (size_t)t * E;
        if (scoring == SCORE_SOFTMAX) {
            softmax_row(l, go, E, sub, LPT, valid);
        } else if (valid) {
            for (int e = sub; e < E; e += LPT) {
                const float s = sigmoid_score(l[e]);
                l[e] = s;
                go[e] = __float2bfloat16_rn(s);
            }
        }
        __syncwarp();   // every score of the row is in place before lanes read each other's experts
        unsigned int taken = 0u;   // bit c: expert sub + c * LPT is excluded (outside the kept groups) or picked
        if (NG > 1) {
            float gs[GPL];
#pragma unroll
            for (int q = 0; q < GPL; ++q) {
                const int g = sub + q * LPT;
                float m1 = -INFINITY, m2 = -INFINITY;
                if (g < NG)
                    for (int e = g * GS; e < (g + 1) * GS; ++e) {
                        const float v = l[e] + bias_s[e];
                        if (v > m1) { m2 = m1; m1 = v; }
                        else if (v > m2) m2 = v;
                    }
                gs[q] = group_top == 2 ? m1 + m2 : m1;
            }
            unsigned int kept = 0u;
            for (int r = 0; r < topk_group; ++r) {
                float bv = -INFINITY;
                int bg = 0x7fffffff;
#pragma unroll
                for (int q = 0; q < GPL; ++q) {
                    const int g = sub + q * LPT;
                    if (g < NG && gs[q] > bv && !((kept >> g) & 1u)) { bv = gs[q]; bg = g; }
                }
                group_argmax(bv, bg, LPT);
                if (bg == 0x7fffffff) bg = 0;
                kept |= 1u << bg;
            }
            int c = 0;
            for (int e = sub; e < E; e += LPT, ++c)
                if (!((kept >> (e / GS)) & 1u)) taken |= 1u << c;
        }
        float W = 0.0f;
        for (int i = 0; i < k; ++i) {
            float bv = -INFINITY;
            int bi = 0x7fffffff;
            if (valid) {
                int c = 0;
#pragma unroll 4
                for (int e = sub; e < E; e += LPT, ++c) {
                    const float v = l[e] + bias_s[e];
                    if (v > bv && !((taken >> c) & 1u)) { bv = v; bi = e; }
                }
            }
            group_argmax(bv, bi, LPT);
            if (bi == 0x7fffffff) { bi = 0; }   // nothing comparable left (NaN scores): index 0, as softmax_topk
            if ((bi & (LPT - 1)) == sub) taken |= 1u << (bi >> lg);
            if (sub == 0 && valid) {
                W = __fadd_rn(W, l[bi]);
                topk_idx[(size_t)t * k + i] = bi;
                sel_e[(s0 + ti) * k + i] = (int16_t)bi;
            }
        }
        if (sub == 0 && valid) {
            for (int i = 0; i < k; ++i) {
                float w = l[sel_e[(s0 + ti) * k + i]];
                if (renormalize) w = W > 0.0f ? __fdiv_rn(w, W) : 0.0f;
                topk_w[(size_t)t * k + i] = __float2bfloat16_rn(__fmul_rn(w, scale));
            }
            mcw[t] = 1.0f;
        }
        __syncwarp();
    }
}

// Position of every (token, pick) among this chunk's selections of the same expert, ascending (token, pick) order, and
// the chunk's per-expert counts.  One warp walks the entries 32 at a time: lanes holding the same expert find each other
// with match.any, the rank inside the group is a popcount, the running per-expert count lives in shared memory (O(n)
// instead of O(n^2); the 64k-token sweep point has 886 entries per CTA).  A skipped pick of a routed launch (-1) takes no
// rank and is not counted.
__device__ __forceinline__ void slot_ranks(const FmParams& p, uint8_t* smem, int n_tok) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = p.E, k = p.k;
    const int16_t* sel_e = reinterpret_cast<const int16_t*>(smem + G_OFF_SEL);
    int* rank_s = reinterpret_cast<int*>(smem + G_OFF_RANK);
    int* cnt_s = reinterpret_cast<int*>(smem + G_OFF_CNT);
    for (int e = tid; e < E; e += NUM_THREADS) cnt_s[e] = 0;
    __syncthreads();
    const int n_ent = n_tok * k;
    if (warp == 0) {
        for (int i0 = 0; i0 < n_ent; i0 += 32) {
            const int i = i0 + lane;
            const int sel = i < n_ent ? (int)sel_e[i] : -1;
            const bool valid = sel >= 0;
            const int e = valid ? sel : (E + lane);                  // lanes without a pick get unique keys
            const unsigned int same = __match_any_sync(0xffffffffu, e);
            const unsigned int before = same & ((1u << lane) - 1u);
            if (valid) rank_s[i] = cnt_s[e] + __popc(before);
            __syncwarp();
            if (valid && before == 0u) cnt_s[e] += __popc(same);    // one lane per distinct expert of the group
            __syncwarp();
        }
    }
    __syncthreads();
    for (int e = tid; e < E; e += NUM_THREADS) p.chunk_counts[(size_t)blockIdx.x * E + e] = cnt_s[e];
}

// The end of phase G once sel_e holds the chunk's picks (router and caller routing alike).  The Wg / logits scratch is
// free from here on: start staging this chunk's token rows for the dispatch phase now (one bulk load, same barrier and
// layout dispatch_phase expects for its first group), so the load runs under the slot ranks, the grid barrier and the
// prefix pass instead of after them.
__device__ __forceinline__ void gate_tail(const FmParams& p, uint8_t* smem, int t0, int n_tok) {
    if (threadIdx.x == 32 && n_tok > 0) {   // (warp 1: warp 0 is about to compute the slot ranks)
        const int row_bytes = p.H * 2;
        const int rows0 = max(1, min(n_tok, D_XROWS_BYTES / row_bytes));
        uint64_t* xbar = bar(smem, BAR_XROWS);
        fence_proxy_async_smem();
        mbar_arrive_expect_tx(xbar, (uint32_t)(rows0 * row_bytes));
        bulk_load_1d(smem + D_OFF_XROWS, p.x + (size_t)t0 * p.H, (uint32_t)(rows0 * row_bytes), xbar);
    }
    slot_ranks(p, smem, n_tok);
}

// The router launch's phase G, and a gated launch's (p.route == ROUTE_GATED): the same logits, then scored_topk
// instead of softmax_topk.
__device__ __forceinline__ void gate_phase(const FmParams& p, const Launch& L, uint8_t* smem, int t0, int n_tok) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int E = p.E;
    float* logit_s = reinterpret_cast<float*>(smem + G_OFF_LOGIT);
    int16_t* sel_e = reinterpret_cast<int16_t*>(smem + G_OFF_SEL);

    float* aux_s = reinterpret_cast<float*>(smem + G_OFF_COLSUM);   // training: this chunk's sum_t p[t,e]
    if (p.aux != nullptr)
        for (int e = tid; e < E; e += NUM_THREADS) aux_s[e] = 0.0f;   // ordered by the block syncs of the first stage below

    const int ldl = E + 1;                                  // padded logits row (bank spread across a warp's tokens)
    int TS = G_LOGIT_BYTES / (ldl * 4);                     // tokens per sub-chunk
    const bool tc = p.tc_gate != 0;
    if (tc) TS = min(TS, BLOCK_M);                          // two wgmma warpgroups = 128 token rows
    else if (TS > n_tok) TS = n_tok;
    GateTcState tcs;
    tcs.gkb = 0;
    uint32_t wgphase = 0;
    if (tc) __syncthreads();   // the router's stage barriers (initialised in the prologue) are visible to every warp

    for (int s0 = 0; s0 < n_tok; s0 += TS) {
        const int n_sub = min(TS, n_tok - s0);
        if (tc) {
            if (s0 > 0) __syncthreads();   // the logits scratch is reused: everybody is done with the previous sub-chunk
            gate_logits_tc(p, smem, t0, s0, n_sub, min(TS, L.tpc), logit_s, ldl, tcs);
        } else {
            gate_logits_gemv(p, smem, t0, s0, n_sub, logit_s, ldl, wgphase);
        }
        __syncthreads();
        if (tid == 0) trace_stamp(p, TRACE_GATE_LOGITS);
        if (p.fused && s0 == 0 && warp == NUM_WARPS - 1) zero_fill_out_rows(p, smem, t0, n_tok);
        if (p.route == ROUTE_GATED) scored_topk(p, smem, t0, s0, n_sub);
        else softmax_topk(p, logit_s, ldl, sel_e, t0, s0, n_sub);
        if (tid == 0) trace_stamp(p, TRACE_TOPK_WARP0);
        __syncthreads();
        if (p.aux != nullptr) {
            // column sums of the fp32 probabilities of this sub-chunk (the reference block-reduces each gate tile's
            // columns, gate.cuh:611-627): warp w owns experts w, w + NUM_WARPS, ...; lanes stride over the tokens
            for (int e = warp; e < E; e += NUM_WARPS) {
                float acc = 0.0f;
                for (int ti = lane; ti < n_sub; ti += 32) acc += logit_s[ti * ldl + e];
#pragma unroll
                for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
                if (lane == 0) aux_s[e] += acc;
            }
            __syncthreads();
        }
    }
    if (tid == 0) trace_stamp(p, TRACE_GATE_TOPK);
    gate_tail(p, smem, t0, n_tok);
    if (p.aux != nullptr && L.S > 0) {   // gML[e] += (sum over this chunk) / S   (gate.cuh:628-634: atomicAdd(gML + e, colAgg / S))
        float* gml = p.aux + (size_t)(L.epoch & 1u) * (2 * E + 1);
        for (int e = tid; e < E; e += NUM_THREADS) atomicAdd(gml + e, __fdividef(aux_s[e], (float)L.S));
    }
}

// Entry gi of a routed launch's [n, k] arrays names expert e outside [-1, E).  The first thread of the launch to get here
// (atomicExch of the epoch on a device word) writes the status record, so the message comes from one thread.
__device__ __noinline__ void report_bad_expert(const FmParams& p, unsigned int epoch, int gi, int e) {
    if (atomicExch(p.status_word, epoch) != epoch)
        fm_record(p.dbg, FM_STATUS_BAD_EXPERT, (unsigned int)(gi / p.k), (unsigned int)(gi % p.k), (unsigned int)e, 0);
}

// Caller routing (fm_moe_forward_routed): the chunk's n_tok * k picks and weights come from routed_idx / routed_w
// [n, k].  An index outside [-1, E) becomes -1 (no expert) and is reported once per launch -- it must not trap, every
// rank takes part in the collective.  Writes topk_idx, topk_w = rne_bf16(w), mcw = 1 and sel_e; gate_out is not written.
// With mcw = 1 the combine's term rne(w~ * rne(y / 1)) is rne(w~ * y) for every normal bf16 y.  Out of line on purpose:
// inlined into the kernel it raised the kernel's spill loads from 544 to 596 B.
__device__ __noinline__ void gate_phase_routed(const FmParams& p, const Launch& L, uint8_t* smem, int t0, int n_tok) {
    const int tid = threadIdx.x, warp = tid >> 5;
    const int E = p.E, k = p.k;
    int16_t* sel_e = reinterpret_cast<int16_t*>(smem + G_OFF_SEL);
    // no gate-weight load to stay behind here: the output-row zero-fill goes first
    if (p.fused && warp == NUM_WARPS - 1) zero_fill_out_rows(p, smem, t0, n_tok);
    const int first = t0 * k, n_ent = n_tok * k;   // entries [first, first + n_ent) of the [n, k] arrays
    auto route = [&](int i, int e, float w) {      // i: entry of the chunk
        if (e < -1 || e >= E) {
            report_bad_expert(p, L.epoch, first + i, e);
            e = -1;
        }
        p.topk_idx[first + i] = e;
        p.topk_w[first + i] = __float2bfloat16_rn(w);
        sel_e[i] = (int16_t)e;
    };
    // 16-byte loads of the whole aligned quads of entries (the arrays start 16-byte aligned), single loads of the
    // chunk's unaligned head and tail, so no entry outside the chunk is read
    const int head = min(n_ent, (4 - (first & 3)) & 3);
    const int nq = (n_ent - head) >> 2;
    for (int q = tid; q < nq; q += NUM_THREADS) {
        const int i = head + 4 * q;
        const uint4 e4 = ld_global_nc_v4(p.routed_idx + first + i);
        const uint4 w4 = ld_global_nc_v4(p.routed_w + first + i);
        route(i, (int)e4.x, __uint_as_float(w4.x));
        route(i + 1, (int)e4.y, __uint_as_float(w4.y));
        route(i + 2, (int)e4.z, __uint_as_float(w4.z));
        route(i + 3, (int)e4.w, __uint_as_float(w4.w));
    }
    const int tail0 = head + 4 * nq;
    for (int i = tid; i < head + (n_ent - tail0); i += NUM_THREADS) {
        const int j = i < head ? i : tail0 + (i - head);
        route(j, p.routed_idx[first + j], p.routed_w[first + j]);
    }
    for (int i = tid; i < n_tok; i += NUM_THREADS) p.mcw[t0 + i] = 1.0f;
    if (tid == 0) trace_stamp(p, TRACE_GATE_TOPK);
    gate_tail(p, smem, t0, n_tok);   // (its first block sync orders the sel_e writes before the slot ranks)
}

// ============================================================================================================
// Phase D: dispatch (after the grid barrier).  slot = (selections of e by lower chunks) + rank in chunk; kept iff
// slot < EC (gate.cuh:713-717).  Whole token rows go straight into the owner rank's receive buffer (peer-mapped, NVLink)
// -- the reference's P2P branch (os/packet.cuh:114-116,151-166) -- as TMA bulk copies staged through shared memory.
// Signalling (os/packet.cuh:214-237 sends one {rows, tiles, seq} word per (source, expert) once the LAST of its dispatch
// CTAs is done): here the 8-byte {epoch, rows} flag is published as soon as the count is known -- right after the
// prefix pass, before any row moves (also for 0 rows, like the reference's "noop" signal) -- and the data itself is
// acknowledged per 128-row block: every CTA adds the number of rows it has landed in block b of packet (me, e) to the
// owner's arrival counter recv_rows[epoch parity][pkt][b] with a release at system scope.  A GEMM0 tile starts when ITS
// row blocks are complete, not when the slowest CTA of the source rank has finished.
// Runs on warps 2, 4-11 only (see the kernel body).
// ============================================================================================================
// The prefix over chunk_counts [G, E]: base (selections of e by lower chunks), total (by all chunks) and own (by this
// chunk).  Experts go in column groups of V: four with 16-byte loads when E % 4 == 0, else one.  With ncol = E / V groups
// and ncol <= DISP_THREADS, R = DISP_THREADS / ncol threads share a group and stride over the rows by R; with more groups
// thread tid owns groups tid, tid + DISP_THREADS, ...  Sums stay in registers and a thread adds each of its groups into
// total and base once.  These are integer sums: every order gives the same bits.
template <int V>
__device__ __forceinline__ void expert_prefix_cols(const FmParams& p, int tid, int* base_s, int* total_s, int* own_s) {
    const int G = gridDim.x, ncol = p.E / V;
    const int R = max(1, DISP_THREADS / ncol);
    if (tid >= R * ncol) return;
    // group (row r, column group c) is element r * ncol + c of chunk_counts viewed in groups of V
    const int n = G * ncol, mine = (int)blockIdx.x * ncol, step = R * ncol;
    for (int c = tid % ncol; c < ncol; c += DISP_THREADS) {
        int pt[V] = {}, pb[V] = {};
        for (int i0 = tid / ncol * ncol + c; i0 < n; i0 += 8 * step) {
            int v[8][V];
#pragma unroll
            for (int u = 0; u < 8; ++u) {   // all loads of the batch are in flight before the first use
                const int i = i0 + u * step;
                if constexpr (V == 4) {
                    const int4 q = i < n ? ld_global_cg_i4(reinterpret_cast<const int4*>(p.chunk_counts) + i) : make_int4(0, 0, 0, 0);
                    v[u][0] = q.x; v[u][1] = q.y; v[u][2] = q.z; v[u][3] = q.w;
                } else {
                    v[u][0] = i < n ? p.chunk_counts[i] : 0;
                }
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int i = i0 + u * step;
                if (i >= n) break;
                if (i == mine + c) {
                    if constexpr (V == 4) *reinterpret_cast<int4*>(own_s + 4 * c) = make_int4(v[u][0], v[u][1], v[u][2], v[u][3]);
                    else own_s[c] = v[u][0];
                }
#pragma unroll
                for (int q = 0; q < V; ++q) {
                    pt[q] += v[u][q];
                    if (i < mine) pb[q] += v[u][q];
                }
            }
        }
#pragma unroll
        for (int q = 0; q < V; ++q) {
            if (pt[q] != 0) atomicAdd(&total_s[c * V + q], pt[q]);
            if (pb[q] != 0) atomicAdd(&base_s[c * V + q], pb[q]);
        }
    }
}

__device__ __forceinline__ void expert_prefix(const FmParams& p, int tid, int* base_s, int* total_s, int* own_s) {
    for (int e = tid; e < p.E; e += DISP_THREADS) { base_s[e] = 0; total_s[e] = 0; }
    named_sync<NAMED_BAR_PREFIX, DISP_THREADS>();
    if (p.E % 4 == 0) expert_prefix_cols<4>(p, tid, base_s, total_s, own_s);
    else expert_prefix_cols<1>(p, tid, base_s, total_s, own_s);
    named_sync<NAMED_BAR_PREFIX, DISP_THREADS>();
}

// The count of packet (me, e) is known: CTA (e mod G) tells the owner now.  Nothing precedes this word that the reader
// depends on (the rows are acknowledged through recv_rows), so a relaxed system-scope store is enough.
__device__ __forceinline__ void publish_counts(const FmParams& p, const Launch& L, int tid, const int* total_s) {
    const int E = p.E, G = gridDim.x, EC = L.EC;
    for (int e = (int)blockIdx.x + tid * G; e < E; e += DISP_THREADS * G) {
        const int tot = total_s[e];
        p.counts[e] = tot;
        const int rows = tot < EC ? tot : EC;
        const int owner = e / p.nLx, le = e - owner * p.nLx;
        st_relaxed_sys_u64(p.peer_recv_flag[owner] + (size_t)p.rank * p.nLx + le,
                           ((unsigned long long)L.epoch << 32) | (unsigned int)rows);
        if (owner == p.rank) p.recv_cnt[p.rank * p.nLx + le] = rows;   // (also when the work list is empty: S = 0)
        if (p.aux != nullptr && L.S > 0) {   // (S = 0: the buffer stays as cleared, all zero)
            // gMeC[e] = selections of e / S (gate.cuh:698-706 adds each tile's count / S; the chunk totals are summed
            // first here), loss += gML[e] * gMeC[e] / E (gate.cuh:763-773).  Every CTA's gML atomics precede its arrival
            // at the grid barrier, so gML is complete here.
            float* a = p.aux + (size_t)(L.epoch & 1u) * (2 * E + 1);
            const float ce = __fdividef((float)tot, (float)L.S);
            a[E + e] = ce;
            const float me = *reinterpret_cast<volatile float*>(a + e);
            atomicAdd(a + 2 * E, __fdividef(me * ce, (float)E));
        }
    }
}

// This chunk's rows of expert e occupy slots [lo, hi) of packet (me, e): add the rows landed per 128-row block to the
// owner's arrival counters of epoch parity `par`.  The release covers every store of the threads that met at the
// preceding barrier.
__device__ __forceinline__ void ack_rows(const FmParams& p, unsigned int par, int e, int lo, int hi, bool local) {
    if (hi <= lo) return;
    const int owner = e / p.nLx, le = e - owner * p.nLx;
    unsigned int* ctr = p.peer_recv_rows[owner] + ((size_t)par * p.num_pkts + (size_t)(p.rank * p.nLx + le)) * p.TCM;
    for (int b = lo / BLOCK_M; b <= (hi - 1) / BLOCK_M; ++b) {
        const int n = min(hi, (b + 1) * BLOCK_M) - max(lo, b * BLOCK_M);
        if (local) red_release_gpu_add_u32(ctr + b, (unsigned int)n);
        else red_release_sys_add_u32(ctr + b, (unsigned int)n);
    }
}

// Up to RANGES_IN_REGS experts, warp 2 keeps the slot ranges of the remote ones in registers (RMAX per lane) and gives
// the prefix arrays up before its row stream; beyond that it needs them until its acknowledgements.
constexpr int RMAX = 8;
constexpr int RANGES_IN_REGS = 32 * RMAX;

// The router weight on the input (FmParams::weight_on_input, k = 1): staged row r (`nb` bytes at s + r * stride, a whole
// token row or a piece of one) of token t_first + r becomes rne_bf16(fl32(x) * fl32(w~)), w~ = topk_w[t, 0]; the product
// of two bf16 numbers is exact in fp32, so this is torch's bf16 x * w.  Warp `w` of `nw` takes rows w, w + nw, ...  The
// caller fences (async proxy) and synchronises before the bulk stores read the rows.  Out of line on purpose, like
// gate_phase_routed: inlined into the kernel it raised the spill loads from 552 to 560 B.
__device__ __noinline__ void scale_staged_rows(const FmParams& p, uint8_t* s, int t_first, int rows, int stride, int nb,
                                                  int w, int nw) {
    const int lane = threadIdx.x & 31;
    for (int r = w; r < rows; r += nw) {
        const float wt = __bfloat162float(p.topk_w[t_first + r]);
        for (int c = lane * 16; c < nb; c += 32 * 16) {
            uint4* q = reinterpret_cast<uint4*>(s + (size_t)r * stride + c);
            float f[8];
            unpack8(*q, f);
            uint4 o;
            o.x = pack_bf16x2(__fmul_rn(f[0], wt), __fmul_rn(f[1], wt));
            o.y = pack_bf16x2(__fmul_rn(f[2], wt), __fmul_rn(f[3], wt));
            o.z = pack_bf16x2(__fmul_rn(f[4], wt), __fmul_rn(f[5], wt));
            o.w = pack_bf16x2(__fmul_rn(f[6], wt), __fmul_rn(f[7], wt));
            *q = o;
        }
    }
}

// Warps 4-11: every (token, pick) pair's slot and routing record, and the rows for experts on this rank.
__device__ __forceinline__ void dispatch_local_rows(const FmParams& p, const Launch& L, uint8_t* smem, int t0, int n_tok,
                                                    const int* base_s, const int* own_s) {
    const int ltid = threadIdx.x - EPI_WARP0 * 32;
    const int E = p.E, H = p.H, k = p.k, EC = L.EC;
    const int16_t* sel_e = reinterpret_cast<const int16_t*>(smem + G_OFF_SEL);
    const int* rank_s = reinterpret_cast<const int*>(smem + G_OFF_RANK);
    uint64_t* xbar = bar(smem, BAR_XROWS);   // initialised in the kernel prologue
    uint8_t* x_s = smem + D_OFF_XROWS;       // the router's Wg / logits scratch is free now
    const int row_bytes = H * 2;
    const int rows_per_group = max(1, min(n_tok, D_XROWS_BYTES / row_bytes));
    const bool any_remote = p.W > 1;
    const int first_local = p.rank * p.nLx;
    uint32_t xphase = 0;
    for (int g0 = 0; g0 < n_tok; g0 += rows_per_group) {
        const int rows = min(rows_per_group, n_tok - g0);
        if (ltid == 0 && g0 > 0) {   // group 0 was requested at the end of the router (gate_phase)
            mbar_arrive_expect_tx(xbar, (uint32_t)(rows * row_bytes));
            bulk_load_1d(x_s, p.x + (size_t)(t0 + g0) * H, (uint32_t)(rows * row_bytes), xbar);
        }
        bar_wait(p, smem, BAR_XROWS, xphase);
        xphase ^= 1;
        if (p.weight_on_input) {   // (k = 1: a staged row has at most one destination, so it is scaled in place)
            scale_staged_rows(p, x_s, t0 + g0, rows, row_bytes, row_bytes, ltid >> 5, EPI_THREADS / 32);
            fence_proxy_async_smem();   // these generic writes -> the bulk stores' reads and the next group's load
            named_sync<NAMED_BAR_LOCAL, EPI_THREADS>();
        }
        for (int i = ltid; i < rows * k; i += EPI_THREADS) {   // one thread per (token, pick)
            const int tl = i / k, j = i - tl * k;
            const int ti = g0 + tl, t = t0 + ti;
            const int e = sel_e[ti * k + j];
            // a skipped pick (-1, caller routing) gets slot INT32_MAX: every reader of p.slot takes slot >= EC as dropped
            const int s = e < 0 ? INT32_MAX : base_s[e] + rank_s[ti * k + j];
            p.slot[(size_t)t * k + j] = s;
            if (s < EC) {
                const int owner = e / p.nLx, le = e - owner * p.nLx;
                const size_t row = (size_t)(p.rank * p.nLx + le) * p.pEC + s;
                if (p.fused) {   // what the expert's GEMM1 epilogue needs to combine this row
                    uint4 m;
                    m.x = (unsigned int)t;
                    // (the weight already scaled the row: the owner combines it with weight 1, whatever its own setting)
                    m.y = __float_as_uint(p.weight_on_input ? 1.0f : __bfloat162float(p.topk_w[(size_t)t * k + j]));
                    m.z = __float_as_uint(p.mcw[t]);
                    m.w = 0u;
                    st_global_v4(p.peer_recv_meta[owner] + row, m);
                }
                if (owner == p.rank)
                    bulk_store_1d(p.recv_x + row * H, x_s + (size_t)tl * row_bytes, (uint32_t)row_bytes);
            }
        }
        bulk_commit_group();
        if (g0 + rows_per_group < n_tok) {   // the staging buffer is reused: wait until the bulk stores have read it
            bulk_wait_group_read0();
            named_sync<NAMED_BAR_LOCAL, EPI_THREADS>();
        }
    }
    // (the zero-fill stores, an older bulk group of warp 11, read the first 8 KiB of the epilogue staging area, which
    // is warp 2's window: they must have been read before warp 2 starts -- all but the newest group, the row stores)
    bulk_wait_group_read<1>();
    if (any_remote) named_arrive<NAMED_BAR_SLOTS, DISP_THREADS>();   // every slot (p.slot) is written: warp 2 may start
    bulk_wait_group0();        // this thread's local row stores (and warp 11's zero-fill stores) are complete ...
    fence_proxy_async_all();   // ... and ordered (async proxy) before the generic-proxy counter traffic below
    named_sync<NAMED_BAR_LOCAL, EPI_THREADS>();
    if (any_remote) named_arrive<NAMED_BAR_LOCAL_DONE, DISP_THREADS>();   // local rows + zero-fill complete (warp 2's acks wait for this)
    if (ltid == 0) trace_stamp(p, TRACE_DISP_ROWS_DONE);
    if (any_remote) named_sync<NAMED_BAR_PREFIX_READ, DISP_THREADS>();   // warp 2 has taken what it needs from the stage area
    if (ltid < 32) {   // warp 4: acknowledge the local experts, then hand the stage area to the TMA producer
        const unsigned int par = L.epoch & 1u;
        for (int e = first_local + ltid; e < first_local + p.nLx; e += 32)
            ack_rows(p, par, e, base_s[e], min(base_s[e] + own_s[e], EC), true);
        __syncwarp();
        // (more than RANGES_IN_REGS experts on several ranks: warp 2 still needs base / own for its acknowledgements and
        // releases)
        if (ltid == 0 && (!any_remote || E <= RANGES_IN_REGS)) mbar_arrive(bar(smem, BAR_DISP_DONE));
    }
}

// Warp 2, several ranks: the rows for experts on other ranks.
__device__ __forceinline__ void dispatch_remote_rows(const FmParams& p, const Launch& L, uint8_t* smem, int t0, int n_tok,
                                                     const int* base_s, const int* own_s) {
    const int lane = threadIdx.x & 31;
    const int E = p.E, H = p.H, k = p.k, EC = L.EC;
    const int row_bytes = H * 2;
    const int first_local = p.rank * p.nLx;
    const unsigned int par = L.epoch & 1u;
    // the slot ranges of the remote experts go into registers (E <= RANGES_IN_REGS) before the stage area -- where base /
    // own live -- is released by warp 4; beyond that the release waits for this warp
    int rlo[RMAX], rhi[RMAX];
    const bool in_regs = E <= RANGES_IN_REGS;
#pragma unroll
    for (int i = 0; i < RMAX; ++i) {
        const int e = lane + 32 * i;
        const bool remote = in_regs && e < E && (e < first_local || e >= first_local + p.nLx);
        rlo[i] = remote ? base_s[e] : 0;
        rhi[i] = remote ? min(base_s[e] + own_s[e], EC) : 0;
    }
    __syncwarp();
    if (in_regs) named_arrive<NAMED_BAR_PREFIX_READ, DISP_THREADS>();   // done with the stage area
    named_sync<NAMED_BAR_SLOTS, DISP_THREADS>();                        // every slot of this chunk (p.slot) is written
    {
        // Remote rows through the TMA engine (SM-issued peer stores reached only ~400 GB/s over NVLink, bulk stores ~600):
        // a window of the epilogue staging area -- unused until this CTA's first tile is complete; its first 8 KiB hold the
        // zero source of the output zero-fill -- is filled with a run of consecutive token rows of x (one bulk load), every
        // kept (token, pick) pair of those tokens that belongs to another rank is one bulk store of a whole row to that
        // rank's receive buffer, and when the engine has read the window the next run follows.  The link paces the stores.
        uint8_t* win = smem + D_OFF_WIN;
        const int win_bytes = D_WIN_BYTES;
        const int rows_win = max(1, win_bytes / row_bytes);
        uint64_t* rbar = bar(smem, BAR_REMOTE);
        uint32_t rphase = 0;
        const bool fits = row_bytes <= win_bytes;   // (d_model > 12288: rows go piecewise, below)
        for (int tw = 0; tw < n_tok; tw += rows_win) {
            const int rows = min(rows_win, n_tok - tw);
            // does any pair of these tokens go to another rank?  (expert and slot from the routing tables in global memory)
            bool mine = false;
            for (int i = lane; i < rows * k; i += 32) {
                const size_t gi = (size_t)(t0 + tw) * k + i;
                const int owner = p.topk_idx[gi] / p.nLx;
                mine |= owner != p.rank && p.slot[gi] < EC;
            }
            const unsigned int anyone = __ballot_sync(0xffffffffu, mine);
            if (anyone == 0u) continue;
            if (fits) {
                if (lane == 0) {
                    fence_proxy_async_smem();
                    mbar_arrive_expect_tx(rbar, (uint32_t)(rows * row_bytes));
                    bulk_load_1d(win, p.x + (size_t)(t0 + tw) * H, (uint32_t)(rows * row_bytes), rbar);
                }
                bar_wait(p, smem, BAR_REMOTE, rphase);
                rphase ^= 1;
                if (p.weight_on_input) {
                    scale_staged_rows(p, win, t0 + tw, rows, row_bytes, row_bytes, 0, 1);
                    fence_proxy_async_smem();
                    __syncwarp();
                }
                for (int i = lane; i < rows * k; i += 32) {
                    const size_t gi = (size_t)(t0 + tw) * k + i;
                    const int e = p.topk_idx[gi];
                    const int owner = e / p.nLx;
                    const int sl = p.slot[gi];
                    if (owner != p.rank && sl < EC)
                        bulk_store_1d(p.peer_recv_x[owner] + ((size_t)(p.rank * p.nLx + (e - owner * p.nLx)) * p.pEC + sl) * H,
                                      win + (size_t)(i / k) * row_bytes, (uint32_t)row_bytes);
                }
                bulk_commit_group();
                bulk_wait_group_read0();   // the engine has read the window
                __syncwarp();
            } else {
                // very wide rows: one token at a time, in window-sized pieces
                for (int off = 0; off < row_bytes; off += win_bytes) {
                    const int nb = min(win_bytes, row_bytes - off);
                    if (lane == 0) {
                        fence_proxy_async_smem();
                        mbar_arrive_expect_tx(rbar, (uint32_t)nb);
                        bulk_load_1d(win, reinterpret_cast<const uint8_t*>(p.x + (size_t)(t0 + tw) * H) + off, (uint32_t)nb, rbar);
                    }
                    bar_wait(p, smem, BAR_REMOTE, rphase);
                    rphase ^= 1;
                    if (p.weight_on_input) {
                        scale_staged_rows(p, win, t0 + tw, 1, nb, nb, 0, 1);
                        fence_proxy_async_smem();
                        __syncwarp();
                    }
                    for (int i = lane; i < k; i += 32) {
                        const size_t gi = (size_t)(t0 + tw) * k + i;
                        const int e = p.topk_idx[gi];
                        const int owner = e / p.nLx;
                        const int sl = p.slot[gi];
                        if (owner != p.rank && sl < EC)
                            bulk_store_1d(reinterpret_cast<uint8_t*>(p.peer_recv_x[owner] +
                                              ((size_t)(p.rank * p.nLx + (e - owner * p.nLx)) * p.pEC + sl) * H) + off,
                                          win, (uint32_t)nb);
                    }
                    bulk_commit_group();
                    bulk_wait_group_read0();
                    __syncwarp();
                }
            }
        }
        named_arrive<NAMED_BAR_WINDOW, DISP_THREADS>();   // the staging area belongs to the epilogue warps from here
        bulk_wait_group0();        // the rows have arrived on the other ranks ...
        fence_proxy_async_all();   // ... and are ordered before the generic-proxy acknowledgements
    }
    __syncwarp();
    // the remote acknowledgements also tell the peers that this chunk's output rows are zeroed (TMA stores issued by warp 11
    // in the router, completed before it arrives here) and that the routing records are written
    named_sync<NAMED_BAR_LOCAL_DONE, DISP_THREADS>();
    if (in_regs) {
#pragma unroll
        for (int i = 0; i < RMAX; ++i) ack_rows(p, par, lane + 32 * i, rlo[i], rhi[i], false);
    } else {
        for (int e = lane; e < E; e += 32)
            if (e < first_local || e >= first_local + p.nLx) ack_rows(p, par, e, base_s[e], min(base_s[e] + own_s[e], EC), false);
        __syncwarp();
        named_arrive<NAMED_BAR_PREFIX_READ, DISP_THREADS>();
        if (lane == 0) mbar_arrive(bar(smem, BAR_DISP_DONE));
    }
}

__device__ __forceinline__ void dispatch_phase(const FmParams& p, const Launch& L, uint8_t* smem, int t0, int n_tok) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tid = (warp == 2 ? 0 : (warp - 3) * 32) + lane;   // 0..287 within the dispatch subset
    int* base_s = reinterpret_cast<int*>(smem + D_OFF_BASE);
    int* total_s = reinterpret_cast<int*>(smem + D_OFF_TOTAL);
    int* own_s = reinterpret_cast<int*>(smem + D_OFF_OWN);
    expert_prefix(p, tid, base_s, total_s, own_s);
    if (tid == 0) trace_stamp(p, TRACE_DISP_PREFIX);
    publish_counts(p, L, tid, total_s);
    // Row copies.
    //   * Rows for experts on THIS rank (warps 4-11): the chunk's token rows are contiguous in x, so one bulk load stages up
    //     to 128 KiB of them in shared memory (the first group was requested at the end of the router) and every kept
    //     (token, pick) pair is one cp.async.bulk store of a whole row through the TMA engine (no per-lane chains).  They
    //     land in ~4 us and are acknowledged at once (gpu-scope release); the stage area is handed to the TMA producer, the
    //     warps become epilogue warps, and the expert FFN starts on the local packets while
    //   * rows for experts on OTHER ranks (warp 2, from the moment the slots are known) cross NVLink as 16-byte peer stores
    //     read straight from x (L2 hits), sixteen pieces per lane in flight.  The link bounds them (S*k*(1-1/W)*H*2 bytes
    //     at ~770 GB/s) and back-pressures the issuing warp -- which has no other duty until the first tile needs
    //     publishing; it then waits for the stores with a system-scope release and acknowledges them.
    if (warp != 2) dispatch_local_rows(p, L, smem, t0, n_tok, base_s, own_s);
    else if (p.W > 1) dispatch_remote_rows(p, L, smem, t0, n_tok, base_s, own_s);
}

// ============================================================================================================
// Phase F: expert FFN.  Work items (global order, claimed with one atomic counter by the scheduler warp):
//   packets in the order (own rank first, then rank+1, ...); all GEMM0 blocks, then the GEMM1 blocks (host knob FM_G1_LAG
//   interleaves them with a lag instead).  item -> (row block m fastest, column tile n).  Every packet holds tcm_items row
//   blocks per column tile: on one rank the TCM of this call's capacity, with several ranks (where a receiver does not
//   know its peers' token counts) the context's maximum.  Either way the list is a superset: row blocks beyond the
//   packet's row count are skipped once the packet flag is known.  A GEMM1 tile waits until its GEMM0's done counter
//   of its row block (g0_done[pkt][m], or s0_done[m] for the shared expert) reaches that GEMM0's column tiles.  The
//   shared expert's blocks are placed by the host (fm_create) and hold s_rb row blocks of the call's tokens.
// ============================================================================================================
struct TileInfo {     // written by the scheduler warp, read by the producer / consumer / publisher warps
    int gemm;         // GEMM_* (kind = gemm & 1), -1 stop
    int ntile;
    int le;           // local expert
    int a_row;        // TMA row coordinates of the A and B tiles (GemmOp); a GEMM0's h rows are its A rows
    int b_row;
    int pkt;          // local packet index src * nLx + le
    int mblk;         // 128-row block of that packet (the shared expert's: of the call's tokens)
    int rows;         // valid rows of that block
    int src;          // source rank of the packet
    int cnt;          // rows of the whole packet
    int pad[2];
};
static_assert(sizeof(TileInfo) <= 64, "a ring slot is 64 bytes");

struct WorkItem {     // a work item id, decoded
    TileBlock blk;
    int mb;           // row block of the packet
    int nt;           // column tile
    int le, src;      // the packet's local expert and source rank
    int b_row;        // TMA row of the tile's B operand
};

// Item `id` of this launch's work list.  `cursor` is the index of a block at or before the item's; the scheduler keeps it
// across its (increasing) ids.
__device__ __forceinline__ WorkItem decode_item(const FmParams& p, const Launch& L, int id, int& cursor) {
    while (id >= block_start(p, L, p.blocks[cursor + 1])) ++cursor;
    WorkItem w;
    w.blk = p.blocks[cursor];
    const GemmOp& op = p.gemm[w.blk.gemm];
    const int local = id - block_start(p, L, w.blk), rbs = gemm_row_blocks(L, w.blk.gemm);
    w.mb = local % rbs;   // row blocks fastest
    w.nt = local / rbs;
    w.le = w.blk.pkt % p.nLx;
    w.src = w.blk.pkt / p.nLx;
    w.b_row = op.b_row0 + w.le * op.b_le_rows + w.nt * tile_cols(op);
    return w;
}

// warp 3, lane 0: claims work items and resolves their dependencies AHEAD of the TMA producer, so the atomic, the
// packet-flag and the h-row-block-counter round trips overlap the previous tile's loads (the job of the reference's OS
// CTA: subscriber decode + scheduler doorbells, os/subscriber.cuh, os/scheduler.cuh -- here one thread, no queues).
__device__ __forceinline__ void ffn_scheduler(const FmParams& p, const Launch& L, uint8_t* smem) {
    TileInfo* ring = reinterpret_cast<TileInfo*>(smem + OFF_RING);
    Ring<NSCHED> q;      // the slot of tile n
    Ring<NSCHED> prev;   // the slot of tile n - 1: one step behind q from tile 1 on
    int cursor = 0, n = 0;
    bool seen_remote = false;   // trace only: first tile of a packet from another rank
    for (;;) {
        if (n >= 1) {  // bounded look-ahead: wait until the producer is close to finishing tile n-1
            bar_wait(p, smem, BAR_PROD_TAKE + prev.i, prev.phase);
            prev.next();
        }
        TileInfo ti;
        ti.gemm = -1; ti.ntile = 0; ti.le = 0; ti.a_row = 0; ti.b_row = 0; ti.pkt = 0; ti.mblk = 0; ti.rows = 0;
        ti.src = 0; ti.cnt = 0; ti.pad[0] = ti.pad[1] = 0;
        for (;;) {
            const int id = (int)atomicAdd(p.claim, 1u);
            if (id >= L.total_items) break;
            trace_tile(p, TRACE_TILE_CLAIMED, n);
            const WorkItem w = decode_item(p, L, id, cursor);
            const TileBlock& blk = w.blk;
            const GemmOp& op = p.gemm[blk.gemm];
            const int kind = blk.gemm & 1;
            const int mb = w.mb, nt = w.nt, pkt = blk.pkt, le = w.le, src = w.src;
            const bool first_item = mb == 0 && nt == 0;   // the packet's first item of this GEMM
            const bool same_gpu = src == p.rank;   // flag and counters written from this GPU: gpu scope suffices
            const unsigned int epoch = L.epoch;
            // wait for the packet (src, le): flag = {epoch, rows}  (reference subscriber.cuh:52-185)
            // the call's tokens (dense, shared expert): all of the call's rows, in x (the map over x may have more rows --
            // a device-side count reads S rows -- and the rows past the call's count only reach h's padding rows, which
            // GEMM1's epilogue drops: rows below)
            unsigned long long f = ((unsigned long long)epoch << 32) | (unsigned int)L.S;
            bool stale = false;
            if (op.from_packet) {
                SpinGuard g;
                for (;;) {
                    f = same_gpu ? ld_acquire_gpu_u64(p.recv_flag + pkt) : ld_acquire_sys_u64(p.recv_flag + pkt);
                    const int ahead = (int)((unsigned int)(f >> 32) - epoch);
                    if (ahead == 0) break;
                    // The source rank is already in a LATER forward: it only gets there after every real tile of
                    // this packet has been returned to it, so whatever item of the static superset is left here
                    // is an empty row block.
                    if (ahead > 0) { stale = true; break; }
                    g.tick(p.dbg, p.timeout_ns, FM_TRAP_RECV_FLAG, pkt, (unsigned int)(f >> 32), epoch);
                }
            }
            if (stale) continue;
            const int cnt = (int)(f & 0xffffffffull);
            // once per packet and GEMM (its first item): bookkeeping that needs the count
            if (first_item && kind == 0 && op.from_packet) p.recv_cnt[pkt] = cnt;
            if (p.fused && first_item && kind == 1 && cnt == 0)   // nothing to contribute: tell the source now
                st_release_sys_u64(p.peer_done_flag[src] + (size_t)(p.rank * p.nLx + le), (unsigned long long)epoch << 32);
            const int rows = max(0, min(BLOCK_M, cnt - mb * BLOCK_M));
            if (rows == 0) continue;   // an empty row block of the static superset
            SpinGuard g;
            if (kind == 1) {  // GEMM1 needs the whole h row block (reference notifyNext, processor.cuh:490-615)
                const GemmOp& op0 = p.gemm[blk.gemm - 1];
                const unsigned int* ctr = op0.done + (size_t)pkt * op0.done_pkt + mb;
                while (ld_acquire_gpu_u32(ctr) < (unsigned int)op0.tn)
                    g.tick(p.dbg, p.timeout_ns, FM_TRAP_G0_DONE, pkt, mb, (unsigned int)blk.gemm);
            } else if (op.from_packet) {  // GEMM0 needs the rows of this block to have landed (dispatch acks)
                const unsigned int* rctr = p.recv_rows + ((size_t)(epoch & 1u) * p.num_pkts + pkt) * p.TCM + mb;
                for (;;) {
                    const unsigned int got = same_gpu ? ld_acquire_gpu_u32(rctr) : ld_acquire_sys_u32(rctr);
                    if (got >= (unsigned int)rows) break;
                    g.tick(p.dbg, p.timeout_ns, FM_TRAP_RECV_ROWS, pkt, mb, rows);
                }
            }
            ti.gemm = blk.gemm; ti.ntile = nt; ti.le = le; ti.pkt = pkt; ti.mblk = mb; ti.rows = rows;
            ti.src = src; ti.cnt = cnt;
            ti.a_row = pkt * op.a_pkt_rows + mb * BLOCK_M;
            ti.b_row = w.b_row;
            break;
        }
        if (ti.gemm >= 0) trace_tile(p, TRACE_TILE_READY, n);
        if (ti.gemm >= 0 && ti.src != p.rank && !seen_remote) {
            seen_remote = true;
            trace_stamp(p, TRACE_FIRST_REMOTE);
        }
        bar_wait(p, smem, BAR_SCHED_EMPTY + q.i, q.phase ^ 1u);
        ring[q.i] = ti;
        mbar_arrive(bar(smem, BAR_SCHED_FULL + q.i));
        q.next();
        ++n;
        if (ti.gemm < 0) break;
    }
}

// warp 0: TMA producer
__device__ __forceinline__ void ffn_producer(const FmParams& p, uint8_t* smem) {
    const TileInfo* ring = reinterpret_cast<const TileInfo*>(smem + OFF_RING);
    const int lane = threadIdx.x & 31;
    Ring<STAGES> stage;
    Ring<NSCHED> q;
    bool first = true, stamped = false;
    for (;;) {
        int gemm = -1;
        TileInfo ti;
        if (lane == 0) {
            bar_wait(p, smem, BAR_SCHED_FULL + q.i, q.phase);
            ti = ring[q.i];
            mbar_arrive(bar(smem, BAR_SCHED_EMPTY + q.i));
            gemm = ti.gemm;
        }
        gemm = __shfl_sync(0xffffffffu, gemm, 0);
        if (gemm < 0) break;
        const GemmOp& op = p.gemm[gemm];
        int nk = 0;
        if (lane == 0) {
            if (first)   // the stage area doubles as the dispatch staging buffer
                bar_wait(p, smem, BAR_DISP_DONE, 0);
            first = false;
            fence_proxy_async_global();  // rows written by generic-proxy stores (peers / other SMs) -> TMA reads
            nk = op.kblocks;
        }
        nk = __shfl_sync(0xffffffffu, nk, 0);
        const int glu = op.glu_rows;
        const CUtensorMap* ta = &p.tm[op.a];
        const CUtensorMap* tb = &p.tm[op.b];
        const int take_at = min(nk - 1, max(0, nk - CLAIM_AHEAD_KB));
        int a_row = 0, b_row = 0;
        if (lane == 0) {
            a_row = ti.a_row;
            b_row = ti.b_row;
        }
        for (int kb = 0; kb < nk; ++kb) {
            uint8_t* sa = smem + stage.i * STAGE_BYTES;
            const bool ld_a = (p.dbg_flags & 5) == 0, ld_b = (p.dbg_flags & 9) == 0;   // experiments only
            if (lane == 0) {
                if (kb == take_at) mbar_arrive(bar(smem, BAR_PROD_TAKE + q.i));  // lets the scheduler claim the next tile
                bar_wait(p, smem, BAR_EMPTY + stage.i, stage.phase ^ 1u);
                uint64_t* full = bar(smem, BAR_FULL + stage.i);
                const uint32_t tx = (ld_a ? (uint32_t)A_STAGE_BYTES : 0u) + (ld_b ? (uint32_t)B_STAGE_BYTES : 0u);
                if (tx) mbar_arrive_expect_tx(full, tx); else mbar_arrive(full);
                if (ld_a) tma_load_2d(sa, ta, kb * BLOCK_K, a_row, full);
                if (ld_b) tma_load_2d(sa + A_STAGE_BYTES, tb, kb * BLOCK_K, b_row, full);
                // SwiGLU: B's map has 128-row boxes; the up rows fill the stage's second 16 KiB.  16 KiB is a whole
                // number of SWIZZLE_128B periods (1 KiB), so the stage holds exactly what one 256-row box would.
                if (ld_b && glu) tma_load_2d(sa + A_STAGE_BYTES + B_STAGE_BYTES / 2, tb, kb * BLOCK_K, b_row + glu, full);
                if (!stamped) { trace_stamp(p, TRACE_FIRST_TMA); stamped = true; }   // first loads of the first tile issued
            }
            stage.next();
        }
        q.next();
        __syncwarp();
    }
}

__device__ __noinline__ float gelu_erf(float v) {   // GELU, erf form (cutlass::epilogue::thread::GELU); out of line on purpose
    return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));
}

// SwiGLU of one element pair: h = fl(fl(g * sigmoid(g)) * u), sigmoid_score's sigmoid (relative error in DESIGN.md).
__device__ __forceinline__ float silu_mul(float g, float u) { return __fmul_rn(__fmul_rn(g, sigmoid_score(g)), u); }

enum : int {
    EPI_G0_RELU = 0, EPI_G0_GELU = 1, EPI_G1_STORE = 2, EPI_G1_FUSED_ADD = 3, EPI_G1_FUSED_COPY = 4, EPI_G0_SWIGLU = 5
};

// registers (wgmma fragment: rows r0 = lane/4 and r0 + 8 of this warp's 16, column pairs 8j + 2*(lane%4)) of the 64
// accumulator columns [64c, 64c + 64) -> bias / activation / combine scaling in fp32 -> bf16 (RNE) -> 16 rows of 128 B
// at `stg`, 16-byte piece j of row r at piece j ^ (r & 7) (the TMA's 128-byte swizzle when `stg` is 1 KiB aligned).
// `bias` points at the chunk's first column (or is unused).  EPI_G0_SWIGLU: output chunk c in {0, 1} takes the gate
// from accumulator columns [64c, 64c + 64) and the up projection from the same thread's columns 128 further on; the up
// bias is `glu` elements past the gate bias.
template <int MODE, bool HAS_BIAS>
__device__ __forceinline__ void chunk_to_smem(const float (&acc)[128], int c, uint8_t* stg, const __nv_bfloat16* bias,
                                              int lane, const float (&pw)[2], const float (&mcw)[2], int glu = 0) {
    const int r0 = lane >> 2, cq = (lane & 3) * 2;
    // Rows r0 and r0 + 8 share r & 7 = r0, and `stg` is 128-byte aligned, so piece j of either row is one XOR of bits
    // 4-6 away from piece 0 ^ r0 of row r0: one address register instead of sixteen precomputed ones (which the
    // compiler would otherwise keep live, or spill, beside the 128 accumulators).
    const uint32_t row_addr = smem_u32(stg) + r0 * EPI_ROW_BYTES + (r0 << 4) + cq * 2;
#pragma unroll
    for (int j = 0; j < 8; ++j) {   // 8 columns -> one 4-byte smem store per fragment row
        const uint32_t addr = xor_u32(row_addr, j << 4);
        float2 bv = make_float2(0.0f, 0.0f);
        if (HAS_BIAS) bv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + j * 8 + cq));
        float2 bu = make_float2(0.0f, 0.0f);
        if (HAS_BIAS && MODE == EPI_G0_SWIGLU)
            bu = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + glu + j * 8 + cq));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float f[2] = {acc[c * 32 + j * 4 + 2 * h], acc[c * 32 + j * 4 + 2 * h + 1]};
            if (HAS_BIAS) { f[0] += bv.x; f[1] += bv.y; }
            float u[2] = {0.0f, 0.0f};
            if (MODE == EPI_G0_SWIGLU) {
                u[0] = acc[(c + 2) * 32 + j * 4 + 2 * h];
                u[1] = acc[(c + 2) * 32 + j * 4 + 2 * h + 1];
                if (HAS_BIAS) { u[0] += bu.x; u[1] += bu.y; }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                if (MODE == EPI_G0_RELU) f[i] = fmaxf(f[i], 0.0f);                 // ReLU (types.cuh:151-159)
                else if (MODE == EPI_G0_GELU) f[i] = gelu_erf(f[i]);
                else if (MODE == EPI_G0_SWIGLU) f[i] = silu_mul(f[i], u[i]);
                // the reference's combine arithmetic on the bf16-rounded y (processor.cuh:110-169):
                // term = rne( p~ (x) rne( y / mCw ) ); the bf16 accumulation itself is the REDG in drain_accumulator
                else if (MODE == EPI_G1_FUSED_ADD) f[i] = pw[h] * rne_bf16(__fdividef(rne_bf16(f[i]), mcw[h]));
            }
            st_shared_u32(addr + h * 8 * EPI_ROW_BYTES, pack_bf16x2(f[0], f[1]));   // row r0 + 8h
        }
    }
}

// GEMM0 epilogue of one consumer warp: each 64-column chunk of h goes through one of the two staging buffers and is
// stored by the publisher warp (ffn_publisher) with a TMA tensor store.  `chunk` counts the chunks this warp has handed
// over so far; every consumer warp stages the same sequence, so chunk & 1 names the buffer and chunk >> 1 its use.
//
// Hand-off: wait stg_free[b] (the TMA has read the buffer's previous chunk), write this warp's 16 rows, make the
// generic-proxy smem writes visible to the async proxy (fence.proxy.async.shared::cta by every writing lane, then
// __syncwarp), and arrive on stg_full[b].  The warp never waits for a store to complete and never publishes g0_done
// itself: its next tile can be a GEMM1 tile of this CTA over the same row block, whose dependency wait (the scheduler
// spinning on g0_done) must be satisfied without the consumers -- they are then blocked on that tile's first `full`
// barrier, and waiting here would deadlock until the SpinGuard fires.  The publisher issues the stores, waits for them
// (cp.async.bulk.wait_group 0: the async-proxy writes are complete), orders them before its generic-proxy release with
// fence.proxy.async.global, and then red.release.gpu's g0_done; the scheduler's ld.acquire.gpu of g0_done plus the
// producer's fence.proxy.async.global before its TMA loads of h complete the chain on the reading side.
// Rows at or beyond the block's valid rows are staged and stored too: they lie in the packet's pEC padding of h, and
// GEMM1 multiplies them row-independently and drops their results.  `glu`: EPI_G0_SWIGLU's up-bias offset.
template <int MODE, bool HAS_BIAS>
__device__ __forceinline__ void stage_h(const FmParams& p, uint8_t* smem, const float (&acc)[128],
                                        const __nv_bfloat16* bias, int nchunks, int row0, int lane, uint32_t& chunk,
                                        int glu = 0) {
    const float one[2] = {1.0f, 1.0f};
#pragma unroll
    for (int c = 0; c < BLOCK_N / 64; ++c) {
        if (c >= nchunks) break;
        const int b = chunk & 1;
        bar_wait(p, smem, BAR_STG_FREE + b, ((chunk >> 1) & 1) ^ 1);
        chunk_to_smem<MODE, HAS_BIAS>(acc, c, smem + OFF_EPI + b * EPI_CHUNK_BYTES + row0 * EPI_ROW_BYTES,
                                      HAS_BIAS ? bias + c * 64 : nullptr, lane, one, one, glu);
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar(smem, BAR_STG_FULL + b));
        ++chunk;
    }
}

struct DrainArgs {
    uint8_t* stg;                  // this warp's transpose tile: 16 rows of 128 B (16-byte pieces XOR-swizzled by row & 7)
    int nchunks;                   // 64-column chunks of the tile that exist (1 to 4)
    int lane, row0, my_rows, N, n0;
    const __nv_bfloat16* bias;     // [N] or nullptr
    __nv_bfloat16* out_rows;       // row 0 of the destination row block in the return buffer
    __nv_bfloat16* acc_base;       // fused GEMM1: the source rank's output accumulator
    int my_tok;                    // fused GEMM1, lanes 0-15: token of tile row (row0 + lane)
    float my_pw, my_mcw;
};

// GEMM1 epilogue: 64 accumulator columns per step through chunk_to_smem, then the transposed read-back and full-line
// 16-byte global stores (or REDG adds) straight from the warp.
template <int MODE, bool HAS_BIAS>
__device__ __forceinline__ void drain_accumulator(const FmParams& p, const DrainArgs& a, const float (&acc)[128]) {
    const int lane = a.lane, r0 = lane >> 2;
    float pw[2], mcw[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        pw[h] = __shfl_sync(0xffffffffu, a.my_pw, r0 + 8 * h);
        mcw[h] = __shfl_sync(0xffffffffu, a.my_mcw, r0 + 8 * h);
    }
#pragma unroll
    for (int c = 0; c < BLOCK_N / 64; ++c) {
        if (c >= a.nchunks) break;
        chunk_to_smem<MODE, HAS_BIAS>(acc, c, a.stg, HAS_BIAS ? a.bias + a.n0 + c * 64 : nullptr, lane, pw, mcw);
        __syncwarp();
        // transposed read-back: 8 lanes cover one row's 128 bytes, 4 rows per instruction, full-line stores
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int r = it * 4 + (lane >> 3), seg = lane & 7;
            const uint4 o = *reinterpret_cast<const uint4*>(a.stg + r * EPI_ROW_BYTES + ((seg ^ (r & 7)) << 4));
            const int row_in_tile = a.row0 + r;
            if (MODE == EPI_G1_FUSED_ADD || MODE == EPI_G1_FUSED_COPY) {
                // row -> its token's output row on the source rank (k == 1: plain copy, reference processor.cuh:170-203)
                const int tok = __shfl_sync(0xffffffffu, a.my_tok, r);
                if (row_in_tile < a.my_rows) {
                    __nv_bfloat16* dst = a.acc_base + (size_t)tok * a.N + a.n0 + c * 64 + seg * 8;
                    if (MODE == EPI_G1_FUSED_ADD) red_add_bf16x8(dst, o); else st_global_v4(dst, o);
                }
            } else if (row_in_tile < a.my_rows) {   // EPI_G1_STORE: the return buffer on the source rank
                st_global_v4(a.out_rows + (size_t)row_in_tile * a.N + a.n0 + c * 64 + seg * 8, o);
            }
        }
        __syncwarp();
    }
}

// warps 4-11: two consumer warpgroups.  Per tile: wgmma over the k-blocks the producer stages (warpgroup g multiplies A
// rows [64g, 64g + 64) by the whole B tile into 128 fp32 registers per thread), then the epilogue of this warp's 16 rows.
// The consumers do not wait for their stores, nor fence or publish: a GEMM0 tile's h chunks are handed to the publisher
// warp through the staging buffers (stage_h), and after a GEMM1 tile lane 0 of every consumer warp arrives on pub_full[];
// the publisher warp takes over from there (ffn_publisher).
struct Consumer {         // one consumer warp's place in the rings it reads, kept across tiles
    Ring<NSCHED> q;       // scheduler ring
    Ring<STAGES> stage;   // pipeline stages
    Ring<2> pub;          // GEMM1 tiles handed to the publisher (pub_full / pub_empty)
    uint32_t chunk = 0;   // GEMM0 h chunks this warp has staged so far (stage_h)
    int ntiles = 0;
    int lane;
    int wg;               // warpgroup: A rows [64 wg, 64 wg + 64)
    int row0;             // this warp's 16 rows of the tile
    bool stamper;         // the thread that writes the consumers' trace stamps
};

// The k-block loop: one k-block's wgmma group in flight while the previous stage is handed back.  Returns with the last
// k-block's group still in flight, and the stage it reads (-1 when there are no k-blocks).
__device__ __forceinline__ int mainloop(const FmParams& p, uint8_t* smem, float (&acc)[128], int nk, Consumer& c) {
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.0f;
    int prev = -1;
    for (int kb = 0; kb < nk; ++kb) {
        bar_wait(p, smem, BAR_FULL + c.stage.i, c.stage.phase);
        if (kb == 0 && c.stamper) trace_tile(p, TRACE_TILE_FIRST_KB, c.ntiles);
        if (!(p.dbg_flags & 2)) {   // (experiment: no MMA)
            const uint32_t sa = smem_u32(smem + c.stage.i * STAGE_BYTES);
            const uint64_t da = gmma_smem_desc_sw128(sa + c.wg * 64 * 128);
            const uint64_t db = gmma_smem_desc_sw128(sa + A_STAGE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < BLOCK_K / WGMMA_K; ++kk)
                wgmma_m64n256k16_bf16(acc, da + (uint64_t)(kk * 2), db + (uint64_t)(kk * 2));
            wgmma_commit();
        }
        if (prev >= 0) {   // the previous k-block's MMAs have read their stage
            wgmma_wait<1>();
            __syncwarp();
            if (c.lane == 0) mbar_arrive(bar(smem, BAR_EMPTY + prev));
        }
        prev = c.stage.i;
        c.stage.next();
    }
    return prev;
}

// The start of both epilogues, once they have read the tile's fields from its ring slot: the last k-block's MMAs
// complete, and its stage and the ring slot are handed back.
__device__ __forceinline__ void mainloop_done(const FmParams& p, uint8_t* smem, float (&acc)[128], int prev, Consumer& c) {
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    __syncwarp();
    if (c.lane == 0 && prev >= 0) mbar_arrive(bar(smem, BAR_EMPTY + prev));
    if (c.stamper) trace_tile(p, TRACE_TILE_MMA_DONE, c.ntiles);
    if (c.ntiles == 0 && p.W > 1)   // the staging area served as warp 2's window for the remote rows
        named_sync<NAMED_BAR_WINDOW, DISP_THREADS>();
    if (c.lane == 0) mbar_arrive(bar(smem, BAR_SCHED_EMPTY + c.q.i));   // every lane has read the slot (the __syncwarp above)
    c.q.next();
    if (c.stamper) trace_tile(p, TRACE_TILE_EPI_START, c.ntiles);
}

// f(std::true_type) with a bias, f(std::false_type) without: one specialised epilogue instantiation per (epilogue kind,
// bias) pair, with no per-element or per-group branching
template <class F>
__device__ __forceinline__ void with_bias(const __nv_bfloat16* bias, F&& f) {
    if (bias != nullptr) f(std::true_type{});
    else f(std::false_type{});
}

// GEMM0 epilogue: h.  Every warp stages its 16 rows of each 64-column chunk (N is a multiple of 64, not necessarily of
// the tile width) and goes straight on to the next tile; the publisher warp stores and publishes them.
// A SwiGLU tile whose gate half runs past n (P or Ps = 64 mod 128) has read 64 up rows into its gate half's last 64
// accumulator columns and 64 rows of the flat-viewed W_down into its up half's: both lie inside the weight tensor, and
// those columns are never stored (nchunks = 1), as with the rows past n of a 256-row box.
__device__ __forceinline__ void epilogue_h(const FmParams& p, uint8_t* smem, const TileInfo* ti, float (&acc)[128], int prev,
                                           Consumer& c) {
    const GemmOp& op = p.gemm[ti->gemm];
    const int cols = tile_cols(op), n0 = ti->ntile * cols, le = ti->le;
    mainloop_done(p, smem, acc, prev, c);
    const int nchunks = min(cols / 64, (op.n - n0) / 64);
    const __nv_bfloat16* bias = op.bias ? op.bias + (size_t)le * op.bias_le + n0 : nullptr;
    with_bias(bias, [&](auto has_bias) {
        constexpr bool B = decltype(has_bias)::value;
        if (op.glu_rows) stage_h<EPI_G0_SWIGLU, B>(p, smem, acc, bias, nchunks, c.row0, c.lane, c.chunk, op.glu_rows);
        else if (p.act == 0) stage_h<EPI_G0_RELU, B>(p, smem, acc, bias, nchunks, c.row0, c.lane, c.chunk);
        else stage_h<EPI_G0_GELU, B>(p, smem, acc, bias, nchunks, c.row0, c.lane, c.chunk);
    });
    if (c.stamper) trace_tile(p, TRACE_TILE_STORES, c.ntiles);
}

// GEMM1 epilogue: the destination rows are the SOURCE rank's return buffer (peer store), like the reference's GEMM1
// epilogue writing into the peer heap (packet.cuh:338-340, processor.cuh:713-720), or with p.fused the tokens' output
// rows there.  Then the tile is handed to the publisher.
__device__ __forceinline__ void epilogue_out(const FmParams& p, uint8_t* smem, const TileInfo* ti, float (&acc)[128],
                                             int prev, Consumer& c) {
    const int lane = c.lane, row0 = c.row0;
    // While the last k-block's MMAs run: the tile's fields from its ring slot and, for the fused epilogue, lane l < 16's
    // routing record of tile row (row0 + l), so that nothing is fetched after the final wait.
    const int ntile = ti->ntile, le = ti->le, pkt = ti->pkt, mblk = ti->mblk, my_rows = ti->rows, src = ti->src;
    const GemmOp& op = p.gemm[ti->gemm];
    const int dest = op.dest;
    const bool fuse = dest == DEST_FUSED;
    int my_tok = 0;
    float my_pw = 0.0f, my_mcw = 1.0f;
    if (fuse && p.dense) {
        my_tok = mblk * BLOCK_M + row0 + lane;   // row i of the only packet IS token i
    } else if (fuse && lane < 16 && row0 + lane < my_rows) {
        const uint4 m = ld_global_v4(p.recv_meta + (size_t)pkt * p.pEC + (size_t)mblk * BLOCK_M + row0 + lane);
        my_tok = (int)m.x;
        my_pw = __uint_as_float(m.y);
        my_mcw = __uint_as_float(m.z);
    }
    mainloop_done(p, smem, acc, prev, c);

    const int N = op.n, n0 = ntile * BLOCK_N;
    const int e_global = p.rank * p.nLx + le;
    const int nchunks = row0 < my_rows ? min(BLOCK_N / 64, (N - n0) / 64) : 0;
    // this warp's transpose tile is its rows of chunk buffer 0, which the TMA may still be reading for the last
    // GEMM0 tile: wait as stage_h would before buffer 0's next use (chunk `next0`; the wait consumes nothing)
    const uint32_t next0 = (c.chunk + 1) & ~1u;
    bar_wait(p, smem, BAR_STG_FREE, ((next0 >> 1) & 1) ^ 1);
    if (nchunks > 0) {
        DrainArgs da;
        da.stg = smem + OFF_EPI + row0 * EPI_ROW_BYTES; da.nchunks = nchunks; da.lane = lane; da.row0 = row0;
        da.my_rows = my_rows; da.N = N; da.n0 = n0;
        da.bias = op.bias ? op.bias + (size_t)le * op.bias_le : nullptr;
        da.out_rows = dest == DEST_Y_S ? p.y_s + (size_t)mblk * BLOCK_M * N   // by token
                                       : p.peer_ret_y[src] + ((size_t)e_global * p.pEC + (size_t)mblk * BLOCK_M) * N;
        da.acc_base = fuse ? p.peer_out_acc[src] : nullptr;
        da.my_tok = my_tok; da.my_pw = my_pw; da.my_mcw = my_mcw;
        with_bias(da.bias, [&](auto has_bias) {
            constexpr bool B = decltype(has_bias)::value;
            if (!fuse) drain_accumulator<EPI_G1_STORE, B>(p, da, acc);
            // (caller and gated routing scale k = 1 too: one add of rne(w~ * y) onto the zero-filled row is exact)
            else if (p.k > 1 || p.route != ROUTE_ROUTER) drain_accumulator<EPI_G1_FUSED_ADD, B>(p, da, acc);
            else drain_accumulator<EPI_G1_FUSED_COPY, B>(p, da, acc);
        });
    }
    if (c.stamper) trace_tile(p, TRACE_TILE_STORES, c.ntiles);

    // hand the tile to the publisher: this warp's stores / REDs are issued
    __syncwarp();
    if (lane == 0) {
        bar_wait(p, smem, BAR_PUB_EMPTY + c.pub.i, c.pub.phase ^ 1u);
        mbar_arrive(bar(smem, BAR_PUB_FULL + c.pub.i));
    }
    c.pub.next();
}

__device__ __forceinline__ void ffn_consumer(const FmParams& p, uint8_t* smem) {
    const TileInfo* ring = reinterpret_cast<const TileInfo*>(smem + OFF_RING);
    const int tid = threadIdx.x, warp = tid >> 5;
    Consumer c;
    c.lane = tid & 31;
    c.wg = (warp - EPI_WARP0) >> 2;
    c.row0 = c.wg * 64 + (warp & 3) * 16;
    // warp 4, lane 0, from values both epilogues keep in registers (a test of the thread index reloads the spilled index
    // in each of them)
    c.stamper = c.row0 == 0 && c.lane == 0;
    for (;;) {
        bar_wait(p, smem, BAR_SCHED_FULL + c.q.i, c.q.phase);
        // The tile's ring slot stays ours until its epilogue is set up (mainloop_done arrives on sched_empty): the
        // per-tile fields are read from shared memory after the k-block loop instead of being kept live (spilled) across it.
        const TileInfo* ti = ring + c.q.i;
        const int gemm = ti->gemm;
        if (gemm < 0) break;
        float acc[128];
        const int prev = mainloop(p, smem, acc, p.gemm[gemm].kblocks, c);
        if ((gemm & 1) == 0) epilogue_h(p, smem, ti, acc, prev, c);
        else epilogue_out(p, smem, ti, acc, prev, c);
        ++c.ntiles;
    }
}

// warp 2, lane 0: writes h and makes finished tiles visible, for every tile of the ring in order.  The fences and the
// store completion take 1-2 us (more over NVLink); here they overlap the next tile's MMA instead of delaying it.
//
// GEMM0: one TMA tensor store per 64-column chunk the consumer warps have staged (stage_h), each buffer handed back as
// soon as the TMA has read it; then, once the stores are complete, the release-add on the row block's h counter
// (reference notifyNext's tSA counter, processor.cuh:490-615).  `chunk` counts the chunks stored so far, in the
// consumers' staging order.
__device__ __forceinline__ void publish_h(const FmParams& p, uint8_t* smem, const TileInfo& ti, uint32_t& chunk) {
    const GemmOp& op = p.gemm[ti.gemm];
    const int cols = tile_cols(op), n0 = ti.ntile * cols, nchunks = min(cols / 64, (op.n - n0) / 64);
    const int row = ti.a_row;
    const CUtensorMap* map = &p.tm[p.gemm[ti.gemm + 1].a];   // h is its GEMM1's A
    unsigned int* ctr = op.done + (size_t)ti.pkt * op.done_pkt + ti.mblk;
    // both buffers' stores in flight: chunk c is issued as soon as it is staged, and only then does the warp wait for
    // the TMA to have read chunk c - 1, whose buffer the consumers refill with chunk c + 1
    for (int c = 0; c < nchunks; ++c, ++chunk) {
        const int b = chunk & 1;
        bar_wait(p, smem, BAR_STG_FULL + b, (chunk >> 1) & 1);
        tma_store_2d(map, smem + OFF_EPI + b * EPI_CHUNK_BYTES, n0 + c * 64, row);
        bulk_commit_group();
        if (c > 0) {
            bulk_wait_group_read<1>();   // chunk c - 1 has been read: its buffer may be refilled
            mbar_arrive(bar(smem, BAR_STG_FREE + (b ^ 1)));
        }
    }
    bulk_wait_group_read<0>();
    mbar_arrive(bar(smem, BAR_STG_FREE + ((chunk - 1) & 1)));
    bulk_wait_group0();            // the tile's h writes (async proxy) are complete ...
    fence_proxy_async_global();    // ... and ordered before the generic-proxy release below
    red_release_gpu_add_u32(ctr, 1u);
}

// GEMM1: once all consumer warps have issued their stores / REDs, a system-scope fence, then the packet or row-block
// counter and, from the last tile, the flag on the source rank (reference processor.cuh:722-750).
__device__ __forceinline__ void publish_out(const FmParams& p, const Launch& L, uint8_t* smem, const TileInfo& ti,
                                            Ring<2>& pub) {
    bar_wait(p, smem, BAR_PUB_FULL + pub.i, pub.phase);
    mbar_arrive(bar(smem, BAR_PUB_EMPTY + pub.i));
    pub.next();
    const int dest = p.gemm[ti.gemm].dest;
    if (dest == DEST_Y_S) {   // the shared expert's s rows, read on this GPU by the completion phase
        fence_acq_rel_gpu();
        red_release_gpu_add_u32(p.s1_done + ti.mblk, 1u);
        return;
    }
    if (dest == DEST_FUSED) {
        // local packet, output left in place: nobody waits for a flag (see finish_fused) -- no fence, no counter, no
        // flag; kernel completion covers these adds.  With a shared expert the completion phase adds s to the finished
        // rows, so it waits for the local experts too.
        if (ti.src == p.rank && p.out_acc == p.out && !p.shared) return;
        fence_acq_rel_sys();   // this tile's adds are performed before the packet counter moves
        const unsigned int old = atom_acq_rel_gpu_add_u32(p.pkt_done + ti.pkt, 1u);
        const unsigned int want = (unsigned int)(((ti.cnt + BLOCK_M - 1) / BLOCK_M) * p.TN1);
        if (old + 1u == want)   // every GEMM1 tile of packet (src, le) has been added into src's output
            st_release_sys_u64(p.peer_done_flag[ti.src] + (size_t)(p.rank * p.nLx + ti.le), (unsigned long long)L.epoch << 32);
    } else {
        fence_acq_rel_sys();
        const unsigned int old = atom_acq_rel_gpu_add_u32(p.g1_done + (size_t)ti.pkt * p.TCM + ti.mblk, 1u);
        if (old == (unsigned int)p.TN1 - 1u) {  // whole rows of this block are on the source rank
            fence_acq_rel_sys();
            const int e_global = p.rank * p.nLx + ti.le;
            st_release_sys_u64(p.peer_ret_flag[ti.src] + (size_t)e_global * p.TCM + ti.mblk,
                               ((unsigned long long)L.epoch << 32) | (unsigned int)ti.rows);
        }
    }
}

// warp 2: the publisher.  Lane 0 takes every tile of the ring in order and publishes it with publish_h or publish_out.
__device__ __forceinline__ void ffn_publisher(const FmParams& p, const Launch& L, uint8_t* smem) {
    const TileInfo* ring = reinterpret_cast<const TileInfo*>(smem + OFF_RING);
    const int lane = threadIdx.x & 31;
    Ring<NSCHED> q;
    Ring<2> pub;
    int ntiles = 0;
    uint32_t chunk = 0;   // h chunks stored so far (publish_h)
    for (;;) {
        int gemm = -1;
        if (lane == 0) {
            bar_wait(p, smem, BAR_SCHED_FULL + q.i, q.phase);
            const TileInfo ti = ring[q.i];
            mbar_arrive(bar(smem, BAR_SCHED_EMPTY + q.i));
            gemm = ti.gemm;
            if (gemm >= 0) {
                if ((gemm & 1) == 0) publish_h(p, smem, ti, chunk);
                else publish_out(p, L, smem, ti, pub);
                trace_tile(p, TRACE_TILE_PUBLISHED, ntiles);
            }
        }
        gemm = __shfl_sync(0xffffffffu, gemm, 0);
        q.next();
        ++ntiles;
        if (gemm < 0) break;
        __syncwarp();
    }
}

// kernel prologue: barriers of every later phase; runs before the router so it costs nothing on the critical path.
// Warp 3's L2 warm-up needs this launch's work list, so it runs after the block sync that publishes the Launch record.
__device__ __forceinline__ void ffn_setup(const FmParams& p, uint8_t* smem) {
    const int tid = threadIdx.x, warp = tid >> 5;
    if (warp == 1 && (tid & 31) == 0) {
#define FM_MBAR_INIT(ID, name, first, count, arrivals) \
        for (int i = 0; i < (count); ++i) mbar_init(bar(smem, (first) + i), (arrivals));
        FM_MBARRIERS(FM_MBAR_INIT)
#undef FM_MBAR_INIT
        fence_mbar_init();
    }
    if (warp == 0 && (tid & 31) == 0) {
        if (!p.dense || p.n_tokens > 0) tma_prefetch_desc(&p.tm[TM_A0]);   // (dense, no tokens: no map over x was encoded)
        tma_prefetch_desc(&p.tm[TM_B0]);
        tma_prefetch_desc(&p.tm[TM_A1]); tma_prefetch_desc(&p.tm[TM_B1]);
    }
}

__device__ __forceinline__ void ffn_warm_l2(const FmParams& p, const Launch& L) {
    if (threadIdx.x == 3 * 32) {
        // Warm L2 with the 256-row weight tile (SwiGLU: its gate and up halves) this CTA will most likely claim first (item
        // id = CTA index: the first wave is claimed in arrival order), pipeline depth only: HBM is idle during the router
        // and the first tile's loads are then L2 hits.  A wrong guess costs nothing -- the tile is needed by some CTA of
        // the first wave anyway.
        const int id = (int)blockIdx.x;
        if (id < L.total_items) {
            int cursor = 0;
            const WorkItem w = decode_item(p, L, id, cursor);
            const GemmOp& op = p.gemm[w.blk.gemm];
            for (int kb = 0; kb < min(op.kblocks, STAGES); ++kb) {
                tma_prefetch_l2_2d(&p.tm[op.b], kb * BLOCK_K, w.b_row);
                if (op.glu_rows) tma_prefetch_l2_2d(&p.tm[op.b], kb * BLOCK_K, w.b_row + op.glu_rows);
            }
        }
    }
}

// Register split of the expert-FFN phase.  __launch_bounds__(384, 1) gives every warp 168 registers (65536 / 384, rounded
// down to a multiple of 8); the producer warpgroup (warps 0-3: TMA producer, idle warp 1, publisher, scheduler) needs few
// of them, the consumer warpgroups hold 128 fp32 accumulators per thread.  128 * REGS_PROD + 256 * REGS_CONS <= 65536.
// 80 / 208 keeps the consumers' k-block loop free of local-memory traffic; with fewer registers for warps 0-3 the
// scheduler and producer code spill heavily (DESIGN.md section 4).  Warps 0, 1 and 3 alone free 8448 registers, the
// consumers take 10240: one consumer warpgroup completes its increase only when warp 2 has given its registers up, after
// dispatch.  With one rank that is at once; with several it waits for the remote row stream (80 / 200 avoids the wait
// and measured about 3 % slower on one GPU).
constexpr int REGS_ALL = 168, REGS_PROD = 80, REGS_CONS = 208;
static_assert(REGS_ALL == (65536 / NUM_THREADS) / 8 * 8, "the even split __launch_bounds__(NUM_THREADS, 1) gives every warp");
static_assert(128 * REGS_PROD + 256 * REGS_CONS <= 65536, "register file of one SM");

// warp roles of the expert-FFN phase (entered per warp as soon as that warp is free; no block-wide sync on entry).  Every
// warp of a warpgroup executes the same setmaxnreg: warps 0-3 give registers up on entry, warps 4-11 (here after the
// router and dispatch, which they run with the even split) take them.  Phase C runs on all 384 threads with the even
// split again: the consumers hand their registers back before the block sync, warps 0-3 take theirs back after it (an
// increase waits for free registers, so it must not come before every consumer's decrease).
__device__ __forceinline__ void ffn_roles(const FmParams& p, const Launch& L, uint8_t* smem) {
    const int tid = threadIdx.x, warp = tid >> 5;
    if (warp < EPI_WARP0) {
        setmaxnreg_dec<REGS_PROD>();
        if (warp == 0) ffn_producer(p, smem);
        else if (warp == 2) ffn_publisher(p, L, smem);
        else if (warp == 3) { if ((tid & 31) == 0) ffn_scheduler(p, L, smem); __syncwarp(); }
    } else {
        setmaxnreg_inc<REGS_CONS>();
        ffn_consumer(p, smem);
        setmaxnreg_dec<REGS_ALL>();
    }
    __syncthreads();
    if (warp < EPI_WARP0) setmaxnreg_inc<REGS_ALL>();
    if (tid == 0) trace_stamp(p, TRACE_FFN_END);
}

// ============================================================================================================
// Phase C: combine (gather path: k > 2 or FM_FUSED_COMBINE=0; the default for k <= 2 is the fused GEMM1 epilogue +
// finish_fused below).  For token t with picks (e_j, slot_j):
//   k > 1: out[t,c] = bf16-accumulate over kept j of rne( p~_j * rne( y_j[c] / mCw ) )   (processor.cuh:110-169)
//   k = 1: out[t,:] = y_0 (no scaling), zeros if dropped                                  (processor.cuh:170-203)
//          (caller and gated routing scale k = 1 like k > 1, with mCw = 1)
// Deterministic gather (no atomics, no zero-fill pass); for k == 2 it equals the reference's atomicAdd result
// exactly because bf16 addition commutes and 0 + a is exact.
// ============================================================================================================
// The shared expert's term: rne(fl32(r) + fl32(s)) per element, for 8 bf16 routed results r and shared outputs s
__device__ __forceinline__ uint4 add_shared_bf16x8(const uint4& r, const uint4& s) {
    float a[8], b[8];
    unpack8(r, a);
    unpack8(s, b);
    uint4 o;
    o.x = pack_bf16x2(a[0] + b[0], a[1] + b[1]); o.y = pack_bf16x2(a[2] + b[2], a[3] + b[3]);
    o.z = pack_bf16x2(a[4] + b[4], a[5] + b[5]); o.w = pack_bf16x2(a[6] + b[6], a[7] + b[7]);
    return o;
}

// every shared-expert GEMM1 tile of the row blocks holding this CTA's tokens has stored its s rows into y_s
__device__ __noinline__ void wait_shared_rows(const FmParams& p, int t0, int n_tok) {
    if (n_tok == 0) return;
    for (int rb = t0 / BLOCK_M + (int)threadIdx.x; rb <= (t0 + n_tok - 1) / BLOCK_M; rb += NUM_THREADS) {
        SpinGuard g;
        while (ld_acquire_gpu_u32(p.s1_done + rb) < (unsigned int)p.TN1)
            g.tick(p.dbg, p.timeout_ns, FM_TRAP_RET_FLAG, 0x5E, rb, 0);
    }
}

// ys: the shared expert's outputs y_s (added after the k terms) or nullptr
template <int KMAX, int PIECES>
__device__ __forceinline__ void combine_rows(const FmParams& p, int EC, int t0, int n_tok, const int* c_e, const int* c_s,
                                             const float* c_w, const float* c_m, const __nv_bfloat16* ys) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int H = p.H, k = p.k;
    for (int ti = warp; ti < n_tok; ti += NUM_WARPS) {
        const __nv_bfloat16* yrow[KMAX];
        float pw[KMAX];
        bool keep[KMAX];
        const float mcw = c_m[ti];
#pragma unroll
        for (int j = 0; j < KMAX; ++j) {
            keep[j] = false;
            yrow[j] = nullptr;
            pw[j] = 0.0f;
            if (j < k) {
                const int s = c_s[ti * k + j];
                pw[j] = c_w[ti * k + j];
                keep[j] = s < EC;
                yrow[j] = p.ret_y + ((size_t)c_e[ti * k + j] * p.pEC + (keep[j] ? s : 0)) * H;
            }
        }
        __nv_bfloat16* orow = p.out + (size_t)(t0 + ti) * H;
        for (int hg = 0; hg < H; hg += PIECES * 256) {
            uint4 yv[KMAX][PIECES];   // every load of this column group is issued before the arithmetic
#pragma unroll
            for (int j = 0; j < KMAX; ++j)
#pragma unroll
                for (int i = 0; i < PIECES; ++i) {
                    const int h = hg + i * 256 + lane * 8;
                    if (j < k && keep[j] && h < H) yv[j][i] = ld_global_v4(yrow[j] + h);
                }
#pragma unroll
            for (int i = 0; i < PIECES; ++i) {
                const int h = hg + i * 256 + lane * 8;
                if (h >= H) continue;
                float acc[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) acc[q] = 0.0f;
#pragma unroll
                for (int j = 0; j < KMAX; ++j) {
                    if (j < k && keep[j]) {
                        float y[8];
                        unpack8(yv[j][i], y);
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const float qv = rne_bf16(__fdividef(y[q], mcw));
                            const float term = rne_bf16(pw[j] * qv);
                            acc[q] = rne_bf16(acc[q] + term);
                        }
                    }
                }
                uint4 o;
                o.x = pack_bf16x2(acc[0], acc[1]); o.y = pack_bf16x2(acc[2], acc[3]);
                o.z = pack_bf16x2(acc[4], acc[5]); o.w = pack_bf16x2(acc[6], acc[7]);
                if (ys != nullptr) o = add_shared_bf16x8(o, ld_global_v4(ys + (size_t)(t0 + ti) * H + h));
                st_global_v4(orow + h, o);
            }
        }
    }
}

// fused path: the output rows were accumulated by the GEMM1 epilogues; wait until every expert (local or remote) has
// reported all of its contributions, then (W > 1) move my rows from the symmetric accumulator to the caller's tensor.
// With a shared expert, out[t] = rne(r[t] + s[t]) once r[t] is complete (the routed terms were added onto +0, which keeps
// k <= 2 order-independent; a third add in arrival order would not be): in place at W = 1, in the copy at W > 1.
__device__ __forceinline__ void finish_fused(const FmParams& p, const Launch& L, int t0, int n_tok) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // Contributions of experts on THIS GPU need no flag when the rows are left where they were accumulated (out == the
    // accumulation target): they are complete when the kernel is, and nobody reads them before.  Only the experts on other
    // ranks -- whose adds arrive over NVLink at their own pace -- must have reported; with a separate caller tensor (the
    // copy below), or a shared expert's term to add to the finished rows, the local ones must have, too (a CTA without
    // tokens has no rows to read).
    const bool need_local = p.out_acc != p.out || (p.shared && n_tok > 0);
    for (int e = tid; e < p.E; e += NUM_THREADS) {
        if (!need_local && e / p.nLx == p.rank) continue;
        SpinGuard g;
        while ((ld_acquire_sys_u64(p.done_flag + e) >> 32) != L.epoch)
            g.tick(p.dbg, p.timeout_ns, FM_TRAP_RET_FLAG, e, 0xD0E, 0);
    }
    if (p.shared) wait_shared_rows(p, t0, n_tok);
    __syncthreads();
    if (tid == 0) trace_stamp(p, TRACE_DONE_FLAGS);   // every expert's contributions to this rank's tokens are in
    if (p.out_acc != p.out || p.shared) {
        const __nv_bfloat16* ys = p.shared ? p.y_s : nullptr;
        for (int ti = warp; ti < n_tok; ti += NUM_WARPS) {
            const size_t row = (size_t)(t0 + ti) * p.H;
            const __nv_bfloat16* src = p.out_acc + row;
            __nv_bfloat16* dst = p.out + row;
            for (int hg = 0; hg < p.H; hg += 1024) {
                uint4 v[4], s[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int h = hg + i * 256 + lane * 8;
                    if (h < p.H) v[i] = ld_global_v4(src + h);
                    if (h < p.H && ys != nullptr) s[i] = ld_global_v4(ys + row + h);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int h = hg + i * 256 + lane * 8;
                    if (h < p.H) st_global_v4(dst + h, ys != nullptr ? add_shared_bf16x8(v[i], s[i]) : v[i]);
                }
            }
        }
    }
}

__device__ __forceinline__ void combine_phase(const FmParams& p, const Launch& L, uint8_t* smem, int t0, int n_tok) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = p.H, k = p.k, EC = L.EC;
    // the pipeline stage area is free again: stage this chunk's routing records, and let one thread per (token, pick)
    // poll its return flag so the waits overlap instead of chaining per token
    int* c_e = reinterpret_cast<int*>(smem + C_OFF_E);
    int* c_s = reinterpret_cast<int*>(smem + C_OFF_S);
    float* c_w = reinterpret_cast<float*>(smem + C_OFF_W);
    float* c_m = reinterpret_cast<float*>(smem + C_OFF_M);
    const int n = n_tok * k;
    for (int i = tid; i < n; i += NUM_THREADS) {
        const size_t gi = (size_t)t0 * k + i;
        const int e = p.topk_idx[gi];
        const int s = p.slot[gi];
        c_e[i] = e;
        c_s[i] = s;
        c_w[i] = p.weight_on_input ? 1.0f : __bfloat162float(p.topk_w[gi]);   // (the weight scaled the dispatched row)
        if (s < EC) {
            const unsigned long long* fl = p.ret_flag + (size_t)e * p.TCM + (s / BLOCK_M);
            SpinGuard g;
            while ((ld_acquire_sys_u64(fl) >> 32) != L.epoch)
                g.tick(p.dbg, p.timeout_ns, FM_TRAP_RET_FLAG, e, s, t0 + i / k);
        }
    }
    for (int i = tid; i < n_tok; i += NUM_THREADS) c_m[i] = p.mcw[t0 + i];
    if (p.shared) wait_shared_rows(p, t0, n_tok);
    __syncthreads();
    const __nv_bfloat16* ys = p.shared ? p.y_s : nullptr;   // the shared expert's term, added after the k terms
    if (k == 1 && p.route == ROUTE_ROUTER) {
        for (int ti = warp; ti < n_tok; ti += NUM_WARPS) {
            const bool keep = c_s[ti] < EC;
            const __nv_bfloat16* yrow = p.ret_y + ((size_t)c_e[ti] * p.pEC + (keep ? c_s[ti] : 0)) * H;
            __nv_bfloat16* orow = p.out + (size_t)(t0 + ti) * H;
            for (int h = lane * 8; h < H; h += 256) {
                uint4 v = make_uint4(0u, 0u, 0u, 0u);
                if (keep) v = ld_global_v4(yrow + h);
                if (ys != nullptr) v = add_shared_bf16x8(v, ld_global_v4(ys + (size_t)(t0 + ti) * H + h));
                st_global_v4(orow + h, v);
            }
        }
    } else if (k <= 2) {   // (k = 1 with caller or gated routing: the scaled term rne(w~ * y))
        combine_rows<2, 4>(p, EC, t0, n_tok, c_e, c_s, c_w, c_m, ys);
    } else {
        combine_rows<8, 1>(p, EC, t0, n_tok, c_e, c_s, c_w, c_m, ys);
    }
}

// ============================================================================================================
__global__ void __launch_bounds__(NUM_THREADS, 1) fm_moe_forward_kernel(const __grid_constant__ FmParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5;
    Launch* launch_s = reinterpret_cast<Launch*>(smem + OFF_LAUNCH);

    if (tid == 0) trace_stamp(p, TRACE_START);
    if (tid == 2 * 32) resolve_launch(p, launch_s);   // (warp 2 has no part in the prologue)
    ffn_setup(p, smem);   // mbarriers for the later phases (visible to everyone after the next block sync)
    __syncthreads();
    const Launch& L = *launch_s;
    const int t0 = blockIdx.x * L.tpc;
    const int n_tok = max(0, min(L.tpc, L.S - t0));
    ffn_warm_l2(p, L);
    // per-launch reset of the work counters (reference clearState, moe.cuh:21-70); consumed only after the grid barrier
    if (blockIdx.x == 0) {
        for (int i = tid; i < p.num_pkts * p.TCM; i += NUM_THREADS) {
            p.g0_done[i] = 0u;
            p.g1_done[i] = 0u;
        }
        for (int i = tid; i < p.num_pkts; i += NUM_THREADS) p.pkt_done[i] = 0u;
        if (p.shared)   // the shared expert's row-block counters (every row block this launch can have)
            for (int i = tid; i < L.s_rb; i += NUM_THREADS) p.s0_done[i] = p.s1_done[i] = 0u;
        // the arrival counters of the NEXT epoch's parity: nobody reads them any more (launch epoch-1 is over) and no
        // peer can write them yet (a rank starts forward epoch+1 only after this launch has returned all its rows)
        unsigned int* next_rows = p.recv_rows + (size_t)((L.epoch + 1u) & 1u) * p.num_pkts * p.TCM;
        for (int i = tid; i < p.num_pkts * p.TCM; i += NUM_THREADS) next_rows[i] = 0u;
        if (p.aux != nullptr) {   // the loss buffers of the next launch (reference clearState, moe.cuh:49-54)
            float* next_aux = p.aux + (size_t)((L.epoch + 1u) & 1u) * (2 * p.E + 1);
            for (int i = tid; i < 2 * p.E + 1; i += NUM_THREADS) next_aux[i] = 0.0f;
        }
        if (tid == 0) *p.claim = 0u;
    }
    if (p.dense) gate_phase_dense(p, L, t0, n_tok);
    else if (p.route == ROUTE_CALLER) gate_phase_routed(p, L, smem, t0, n_tok);
    else gate_phase(p, L, smem, t0, n_tok);   // (the router, and a gated launch's logits)
    if (tid == 0) trace_stamp(p, TRACE_GATE_DONE);
    grid_barrier(p, L);
    if (tid == 0) trace_stamp(p, TRACE_BARRIER);
    // every CTA has read the launch counter (resolve_launch, before its arrival at the barrier): advance it for the next
    // launch on the stream, and record this launch's token count beside it (fm_last_launch)
    if (blockIdx.x == 0 && tid == 0) {
        *p.launch_ctr = L.launch;
        *p.launch_tokens = L.S;
    }

    // From here the warps specialise.  Warps 0 and 3 (TMA producer, tile scheduler) enter their FFN roles at once -- the
    // scheduler claims its first tile and spins on the packet flag while warps 2, 4-11 dispatch this CTA's rows; warps
    // 4-11 then become the consumer warpgroups.
    const bool disp_warp = (warp == 2) || (warp >= EPI_WARP0);
    if (disp_warp) {
        if (!p.dense) dispatch_phase(p, L, smem, t0, n_tok);
        else if (warp == 2 && (tid & 31) == 0)   // nothing to copy: GEMM0's TMA reads x in place; release the producer
            mbar_arrive(bar(smem, BAR_DISP_DONE));
        if (warp == 2 && (tid & 31) == 0) trace_stamp(p, TRACE_DISPATCH_END);
    }
    if (tid == EPI_WARP0 * 32) trace_stamp(p, TRACE_FFN_START);
    ffn_roles(p, L, smem);

    __syncthreads();
    if (p.fused) finish_fused(p, L, t0, n_tok);
    else combine_phase(p, L, smem, t0, n_tok);
    __syncthreads();
    if (tid == 0) trace_stamp(p, TRACE_KERNEL_END);
}

}  // namespace fm
