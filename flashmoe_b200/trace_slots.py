"""Columns of the kernel's trace buffer (`MoEContext.read("trace")`, [grid, SLOTS] %globaltimer stamps in ns, 0 where
nothing was stamped): the names of `enum TraceSlot` in csrc/fm_kernel.cuh without their TRACE_ prefix.  Per-tile stamp
`TILE_*` of a CTA's tile i (i < TILES) is column TILE_* + i."""

SLOTS = 128
TILES = 16

# phase stamps
START = 0             # kernel entry
GATE_DONE = 1         # router done, before the grid barrier
BARRIER = 2           # past the grid barrier
DISPATCH_END = 3      # warp 2 done with dispatch
FFN_START = 4         # warp 4 enters the expert FFN
FFN_END = 5           # every FFN role done
KERNEL_END = 6
FIRST_TMA = 7         # producer: first loads of the first tile issued
DISP_PREFIX = 8       # dispatch: prefix over the chunk counts done
DISP_ROWS_DONE = 9    # dispatch: local rows and the zero-fill complete
ZERO_ISSUED = 10      # router: output-row zero-fill issued
GATE_LOGITS = 11      # router: a sub-chunk's logits done
GATE_TOPK = 12        # router: every sub-chunk's softmax / top-k done
FIRST_REMOTE = 13     # scheduler: first tile of a packet from another rank ready
DONE_FLAGS = 14       # fused completion: every expert's done flag seen
TOPK_WARP0 = 15       # router: warp 0's softmax / top-k of a sub-chunk done

# per-tile bases
TILE_READY = 16       # scheduler: dependencies resolved
TILE_FIRST_KB = 32    # consumers: first k-block landed
TILE_MMA_DONE = 48    # consumers: last MMA complete
TILE_EPI_START = 64   # consumers: epilogue started
TILE_STORES = 80      # consumers: epilogue stores issued
TILE_PUBLISHED = 96   # publisher: tile published
TILE_CLAIMED = 112    # scheduler: tile claimed
