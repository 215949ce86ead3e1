"""Exact inputs and the tiling regime of the shared expert (fm_moe_forward_shared); tests/exact.py checks it.

A shared expert is a dense FFN of intermediate size Ps on every token: h_s = RNE(act(x W_up_s^T + b_up_s)) [n, Ps] and
s = y_s = RNE(h_s W_down_s^T + b_down_s) [n, H], with a routed expert's arithmetic; the launch's output is
out = rne_bf16(fl32(r) + fl32(s)) (exact.add_shared), r the routed result the same call writes without one.  Its weights
are drawn on the routed experts' grids, so h_s and y_s are exact under the conditions of exact.py: h_s bit for bit for
ReLU and inside the GELU interval, y_s bit for bit from the device's own h_s (exact.shared_stage).

`regime` states where the kernel's shared-expert items fall (column tiles TN0s of Ps and TN1 of H, their partial last
tiles, row blocks s_rb, tokens per CTA, and the work-list block the GEMM1 items follow); tests/test_shared_exact_cases.py
pins its constants to the sources.  No pytest in here.
"""
from __future__ import annotations

import dataclasses

import numpy as np
import torch

from tests import exact as ex

# ----------------------------------------------------------------------------- the kernel's tiling (fm_kernel.cuh)
BLOCK_M = 128   # token rows per tile: a row block of the shared expert
BLOCK_N = 256   # output columns per tile


@dataclasses.dataclass(frozen=True)
class Regime:
    TN0s: int            # GEMM0 column tiles, ceil(Ps / BLOCK_N)
    ps_tail: int         # columns of the last, partial Ps tile (0: none)
    TN1: int             # GEMM1 column tiles, ceil(H / BLOCK_N)
    h_tail: int          # columns of the last, partial H tile (0: none)
    s_rb: int            # row blocks of tokens, ceil(n / BLOCK_M)
    tpc: int             # tokens per CTA, ceil(n / grid)
    rb_per_cta: int      # most row blocks one CTA's tokens touch (wait_shared_rows' loop)
    split_blk: int       # routed work-list blocks ahead of the shared GEMM1 items

    def line(self) -> str:
        return (f"TN0s {self.TN0s}{f' (tail {self.ps_tail})' if self.ps_tail else ''}, TN1 {self.TN1}"
                f"{f' (tail {self.h_tail})' if self.h_tail else ''}, s_rb {self.s_rb}, tpc {self.tpc}, "
                f"row blocks per CTA {self.rb_per_cta}, split_blk {self.split_blk}")


def split_blk(E: int, lag: int = -1) -> int:
    """Leading local GEMM0 blocks of a one-rank work list (fm_create): all E GEMM0 blocks, or with FM_G1_LAG = lag in
    [1, E) the GEMM0 blocks up to the first GEMM1 block, which comes after GEMM0 of unit lag."""
    kinds = []
    if 1 <= lag < E:
        for i in range(E):
            kinds.append(0)
            if i >= lag:
                kinds.append(1)
    else:
        kinds = [0] * E + [1] * E
    return kinds.index(1)


def regime(H: int, Ps: int, n: int, grid: int, E: int, lag: int = -1) -> Regime:
    tpc = -(-n // grid)
    rbs = 0
    for c in range(grid):
        t0, nt = c * tpc, max(0, min(tpc, n - c * tpc))
        if nt:
            rbs = max(rbs, (t0 + nt - 1) // BLOCK_M - t0 // BLOCK_M + 1)
    return Regime(-(-Ps // BLOCK_N), Ps % BLOCK_N, -(-H // BLOCK_N), H % BLOCK_N, -(-n // BLOCK_M), tpc, rbs,
                  split_blk(E, lag))


# ----------------------------------------------------------------------------- inputs
def shared_inputs(H: int, Ps: int, seed: int, *, act: int = 0, up_range: int = 8, down_range: int = 4,
                  bias: bool = False, gelu_friendly: bool = False, down_density: float = 1.0) -> ex.Experts:
    """A seeded exact shared expert of activation `act` (an exact.Experts record with E = 1) on exact.exact_inputs'
    grids: W_up_s integers in [-up_range, up_range] * 2^-3 (with `gelu_friendly`, sparse ones in [1, up_range] at
    density 4 / H, as exact_inputs draws W_up), W_down_s integers in [-down_range, down_range] * 2^-5, kept at density
    `down_density` (a sparse W_down_s keeps a long GEMM1 sum exact); b_up_s on 2^-3 (>= 0 with `gelu_friendly`),
    b_down_s on 2^-8.  Drawn as int8, so that model-sized experts (exact_gated.layer_inputs' ranges: up_range =
    down_range = 2) stay cheap."""
    g = np.random.default_rng(seed)
    if gelu_friendly:
        up = g.integers(1, up_range + 1, size=(Ps, H), dtype=np.int8) * (g.random((Ps, H), dtype=np.float32) < 4.0 / H)
    else:
        up = g.integers(-up_range, up_range + 1, size=(Ps, H), dtype=np.int8)
    down = g.integers(-down_range, down_range + 1, size=(H, Ps), dtype=np.int8)
    if down_density < 1.0:
        down *= (g.random((H, Ps), dtype=np.float32) < down_density).astype(np.int8)
    w = torch.stack([torch.from_numpy(up.astype(np.int8)).float() * 2.0 ** ex.WUP_GRID,
                     (torch.from_numpy(down).float() * 2.0 ** ex.WDOWN_GRID).reshape(Ps, H)]).bfloat16()
    bu = bd = None
    if bias:
        lo = 0 if gelu_friendly else -16
        bu = torch.from_numpy(g.integers(lo, 17, size=Ps).astype(np.float32) * 2.0 ** ex.WUP_GRID).bfloat16()[None]
        bd = torch.from_numpy(g.integers(-256, 257, size=H).astype(np.float32)
                              * 2.0 ** (ex.WUP_GRID + ex.WDOWN_GRID)).bfloat16()[None]
    return ex.Experts(w[None], bu, bd, act)
