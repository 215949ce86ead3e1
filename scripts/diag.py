"""GPU bring-up diagnostic: runs one fused forward on one H100 and compares every intermediate buffer with the CPU
oracle: routing tables, dispatched rows (recv_x), the expert FFN's h (hidden) and y (ret_y), and the output.
Usage: python scripts/diag.py [--cfg small|A|B] [--noscale] [--all-experts]
The per-phase and per-tile times come from the kernel's own stamps: scripts/trace_gantt.py (single GPU) and
scripts/trace_multi.py (torchrun)."""
import argparse, os, sys, time
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

from flashmoe_b200.config import MoEConfig, BASELINE_CONFIGS
from flashmoe_b200.runtime import MoEContext
from oracle import moe_oracle as mo

CFGS = dict(BASELINE_CONFIGS)
CFGS["small"] = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)
CFGS["tiny"] = MoEConfig(num_experts=4, expert_top_k=2, sequence_len=128, hidden_size=64, intermediate_size=256)
MAX_RELF = 1e-2   # bf16 outputs of fp32-accumulated GEMMs


def make_inputs(cfg, seed=0, scale=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(cfg.mini_batch, cfg.sequence_len, cfg.H, generator=g)
    wg = torch.randn(cfg.H, cfg.E, generator=g)
    we = torch.randn(cfg.E, 2, cfg.P, cfg.H, generator=g)
    if scale:
        wg = wg * cfg.H ** -0.5
        we = we * cfg.H ** -0.5
    return x.bfloat16(), wg.bfloat16(), we.bfloat16()


def oracle(cfg, x, wg, we):
    up, down = mo.split_expert_weights(mo.to_bits(we))
    return mo.forward(mo.to_bits(x.view(cfg.S, cfg.H)), mo.gate_weights_effective(mo.to_bits(wg), cfg.E, cfg.H), up, down,
                      k=cfg.k, EC=cfg.EC, act=cfg.hidden_act), up, down


def cmp_bf16(name, got_bits, ref_bits):
    g = mo.bits_to_f32(got_bits).astype(np.float64); r = mo.bits_to_f32(ref_bits).astype(np.float64)
    diff = np.abs(g - r)
    relf = np.linalg.norm(g - r) / max(np.linalg.norm(r), 1e-30)
    exact = float((got_bits == ref_bits).mean())
    nan = int(np.isnan(g).sum())
    print(f"  {name}: relF={relf:.3e} max|d|={diff.max():.4g} max|ref|={np.abs(r).max():.4g} bit-exact={exact:.6f} "
          f"nan={nan}")
    return relf <= MAX_RELF and nan == 0


def run(args):
    # the gather-combine path keeps the experts' outputs in the return buffer (ret_y); the fused path has none
    os.environ["FM_FUSED_COMBINE"] = "0"
    cfg = CFGS[args.cfg]
    x, wg, we = make_inputs(cfg, scale=not args.noscale)
    t0 = time.time(); ref, up, down = oracle(cfg, x, wg, we); print(f"oracle {time.time()-t0:.2f}s; cfg {args.cfg}: S={cfg.S} H={cfg.H} P={cfg.P} E={cfg.E} k={cfg.k} EC={cfg.EC}")
    ctx = MoEContext(cfg, timeout_ms=3000)
    print("dims", ctx.dims)
    S, H, E, k, EC = cfg.S, cfg.H, cfg.E, cfg.k, cfg.EC
    failures = []
    out = ctx.forward(x.cuda(), wg.cuda(), we.cuda()); ctx.synchronize()

    print("routing")
    topk = ctx.read("topk_idx"); slot = ctx.read("slot"); counts = ctx.read("counts"); mcw = ctx.read("mcw")
    amb = ref.ambiguous
    mism = (topk != ref.topk_idx).any(1)
    print(f"  topk mismatching tokens {int(mism.sum())} (ambiguous {int(amb.sum())}, mismatching&non-ambiguous {int((mism & ~amb).sum())})")
    if (mism & ~amb).any(): failures.append("topk_idx")
    print(f"  slot equal {bool((slot == ref.slot).all())} counts equal {bool((counts == ref.counts).all())} counts {counts.tolist()}")
    print(f"  mcw max rel diff {float(np.max(np.abs(mcw - ref.mcw) / np.maximum(ref.mcw, 1e-30))):.3e}")
    tw = ctx.read("topk_w"); refw = np.take_along_axis(ref.gate_out, ref.topk_idx, axis=1)
    print(f"  topk_w bit-exact frac {float((tw == refw).mean()):.6f}")
    go = ctx.read("gate_out"); print(f"  gate_out bit-exact frac {float((go == ref.gate_out).mean()):.6f}")

    print("dispatch")
    rx = ctx.read("recv_x")  # [E(pkts), pEC, H]
    xb = mo.to_bits(x.view(S, H)); bad = 0; tot = 0
    for t in range(S):
        for j in range(k):
            if ref.kept[t, j] and not mism[t]:
                tot += 1
                if not (rx[ref.topk_idx[t, j], ref.slot[t, j]] == xb[t]).all(): bad += 1
    print(f"  dispatch rows checked {tot}, wrong {bad}")
    if bad: failures.append("recv_x")

    print("expert FFN (on the received rows)")
    hid = ctx.read("hidden"); ry = ctx.read("ret_y"); rc = ctx.read("recv_cnt")
    print("  recv_cnt", rc.tolist())
    for e in range(E):
        n = int(min(counts[e], EC))
        if n == 0: continue
        h_ref, y_ref = mo.expert_ffn(rx[e, :n], up[e], down[e], act=cfg.hidden_act)
        if not cmp_bf16(f"expert {e} rows {n} hidden", hid[e, :n], h_ref): failures.append(f"hidden[{e}]")
        if not cmp_bf16(f"expert {e} rows {n} y     ", ry[e, :n], y_ref): failures.append(f"ret_y[{e}]")
        if e >= 1 and not args.all_experts: break

    print("combine")
    if not cmp_bf16("out", mo.to_bits(out.cpu().view(S, H)), ref.out): failures.append("out")
    ctx.close()
    print("FAILED: " + ", ".join(failures) if failures else "all buffers match the oracle")
    return 1 if failures else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="small")
    ap.add_argument("--noscale", action="store_true"); ap.add_argument("--all-experts", dest="all_experts", action="store_true")
    sys.exit(run(ap.parse_args()))
