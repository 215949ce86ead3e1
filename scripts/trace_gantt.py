"""Per-tile timeline of the fused kernel from its own %globaltimer stamps (fm_set_trace): where the time of the expert-FFN
phase goes.  Usage: python scripts/trace_gantt.py [--cfg B] [--world-note ...]   (environment knobs FM_* apply).
Prints medians over all CTAs of: claim -> dependencies resolved -> first k-block landed -> MMA complete -> epilogue
start -> epilogue stores issued -> published, per GEMM kind, plus the idle gaps between tiles."""
import argparse
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

from flashmoe_b200 import trace_slots as ts
from flashmoe_b200.config import BASELINE_CONFIGS, MoEConfig
from flashmoe_b200.runtime import MoEContext

CFGS = dict(BASELINE_CONFIGS)
CFGS["small"] = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)


def analyse(tr, cfg, label=""):
    tr = tr.astype(np.int64)
    t00 = tr[:, ts.START].min()
    us = lambda a: (a - t00) / 1e3  # noqa: E731
    names = {ts.START: "start", ts.GATE_LOGITS: "gate_gemv", ts.ZERO_ISSUED: "zero_issued", ts.TOPK_WARP0: "topk_warp0",
             ts.GATE_TOPK: "gate_topk", ts.GATE_DONE: "gate_done", ts.BARRIER: "barrier", ts.DISP_PREFIX: "disp_prefix",
             ts.DISP_ROWS_DONE: "disp_rows_done", ts.DISPATCH_END: "dispatch_end", ts.FIRST_TMA: "first_tma_issued",
             ts.FFN_START: "ffn_start", ts.FFN_END: "ffn_end", ts.KERNEL_END: "kernel_end"}
    print(f"--- {label} phases (us after the first CTA's start; min / median / max over CTAs)")
    for i, nm in names.items():
        v = us(tr[:, i][tr[:, i] > 0])
        if len(v):
            print(f"  {nm:14s} {v.min():8.1f} {np.median(v):8.1f} {v.max():8.1f}")
    rows = []
    for c in range(tr.shape[0]):   # every CTA runs its own scheduler, producer and consumer warpgroups
        n = int((tr[c, ts.TILE_FIRST_KB:ts.TILE_FIRST_KB + ts.TILES] > 0).sum())
        for i in range(n):
            rows.append(dict(c=c, i=i, claim=tr[c, ts.TILE_CLAIMED + i], ready=tr[c, ts.TILE_READY + i],
                             first=tr[c, ts.TILE_FIRST_KB + i], mma=tr[c, ts.TILE_MMA_DONE + i],
                             epi=tr[c, ts.TILE_EPI_START + i], stores=tr[c, ts.TILE_STORES + i],
                             pub=tr[c, ts.TILE_PUBLISHED + i],
                             prev_mma=tr[c, ts.TILE_MMA_DONE + i - 1] if i else tr[c, ts.FFN_START]))
    if not rows:
        print("  no tile stamps")
        return
    span = np.array([r["mma"] - r["first"] for r in rows]) / 1e3
    nk = {0: cfg.H // 64, 1: cfg.P // 64}
    kinds = np.array([1 if s > 0.6 * span.max() and span.max() > 1.8 * span.min() else 0 for s in span])
    print(f"--- {label} tiles recorded (first {ts.TILES} per CTA): {len(rows)}; GEMM0-like {int((kinds == 0).sum())}, GEMM1-like {int((kinds == 1).sum())}")
    for kd in (0, 1):
        sel = [r for r, k in zip(rows, kinds) if k == kd]
        if not sel:
            continue
        f = lambda a, b: np.array([r[a] - r[b] for r in sel]) / 1e3  # noqa: E731
        main = f("mma", "first")
        print(f"  GEMM{kd} (nk={nk[kd]}): n={len(sel)}")
        for nm, v in (("claim->ready", f("ready", "claim")), ("ready->first k-block landed", f("first", "ready")),
                      ("first landed->MMA complete", main),
                      ("  per k-block (us)", main / nk[kd]),
                      ("MMA complete->epilogue start", f("epi", "mma")),
                      ("epilogue start->stores issued", f("stores", "epi")),
                      ("stores issued->published", f("pub", "stores")),
                      ("MMA idle before this tile (first landed - prev MMA complete)", f("first", "prev_mma")),
                      ):
            v = v[np.isfinite(v)]
            print(f"    {nm:62s} med {np.median(v):7.2f}  p10 {np.percentile(v, 10):7.2f}  p90 {np.percentile(v, 90):7.2f}")
    t0rows = [r for r in rows if r["i"] == 0]
    if t0rows:
        g = lambda key: np.median([(r[key] - t00) / 1e3 for r in t0rows])  # noqa: E731
        print(f"  per CTA, first tile: claimed {g('claim'):.1f}, rows ready {g('ready'):.1f}, first k-block landed {g('first'):.1f} us (medians)")
    # tensor-busy time per CTA over the FFN phase (only the first ts.TILES tiles of a CTA are stamped)
    busy = {}
    for r in rows:
        busy[r["c"]] = busy.get(r["c"], 0) + (r["mma"] - r["first"])
    b = np.array(list(busy.values())) / 1e3
    t_first = np.array([min(r["first"] for r in rows if r["c"] == c) for c in busy]) - t00
    t_last = np.array([max(r["mma"] for r in rows if r["c"] == c) for c in busy]) - t00
    print(f"  per CTA: mainloop-busy med {np.median(b):.1f} us; first k-block landed at med {np.median(t_first) / 1e3:.1f} "
          f"(min {t_first.min() / 1e3:.1f}, max {t_first.max() / 1e3:.1f}) us; last MMA complete med {np.median(t_last) / 1e3:.1f} max {t_last.max() / 1e3:.1f} us; "
          f"kernel end {us(tr[:, ts.KERNEL_END].max()):.1f} us")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="B")
    ap.add_argument("--label", default="")
    ap.add_argument("--save", default="")
    args = ap.parse_args()
    cfg = CFGS[args.cfg]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(cfg.mini_batch, cfg.sequence_len, cfg.H, generator=g).bfloat16().cuda()
    wg = torch.randn(cfg.H, cfg.E, generator=g).bfloat16().cuda()
    we = torch.randn(cfg.E, 2, cfg.P, cfg.H, generator=g).bfloat16().cuda()
    ctx = MoEContext(cfg, timeout_ms=5000)
    out = torch.empty_like(x)
    for _ in range(5):
        ctx.forward(x, wg, we, out=out)
    ctx.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        ctx.forward(x, wg, we, out=out)
    e1.record()
    ctx.synchronize()
    print(f"=== {args.label or args.cfg}: {e0.elapsed_time(e1) / 20 * 1e3:.1f} us / forward (FM_DBG_FLAGS={os.environ.get('FM_DBG_FLAGS', '0')})")
    ctx.set_trace(True)
    ctx.forward(x, wg, we, out=out)
    ctx.synchronize()
    tr = ctx.read("trace")
    if args.save:
        np.save(args.save, tr)
    analyse(tr, cfg, args.label or args.cfg)
    ctx.close()


if __name__ == "__main__":
    main()
