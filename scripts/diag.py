"""GPU bring-up diagnostic: runs the fused kernel phase by phase on one H100 and compares every intermediate
buffer with the CPU oracle.  Usage: python scripts/diag.py [--cfg small|A|B] [--stage all|gate|ffn|combine|full|time]
Each stage runs in its own process when invoked with --stage all (a device trap poisons the CUDA context)."""
import argparse, json, os, subprocess, sys, time
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import numpy as np
import torch

from flashmoe_b200.config import MoEConfig, BASELINE_CONFIGS
from flashmoe_b200.runtime import MoEContext
from oracle import moe_oracle as mo

CFGS = dict(BASELINE_CONFIGS)
CFGS["small"] = MoEConfig(num_experts=8, expert_top_k=2, sequence_len=512, hidden_size=256, intermediate_size=512)
CFGS["tiny"] = MoEConfig(num_experts=4, expert_top_k=2, sequence_len=128, hidden_size=64, intermediate_size=256)


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
    print(f"  {name}: relF={relf:.3e} max|d|={diff.max():.4g} max|ref|={np.abs(r).max():.4g} bit-exact={exact:.6f} "
          f"nan={int(np.isnan(g).sum())}")
    return relf


def stage(args):
    cfg = CFGS[args.cfg]
    x, wg, we = make_inputs(cfg, scale=not args.noscale)
    t0 = time.time(); ref, up, down = oracle(cfg, x, wg, we); print(f"oracle {time.time()-t0:.2f}s; cfg {args.cfg}: S={cfg.S} H={cfg.H} P={cfg.P} E={cfg.E} k={cfg.k} EC={cfg.EC}")
    ctx = MoEContext(cfg, timeout_ms=3000)
    print("dims", ctx.dims)
    xd, wgd, wed = x.cuda(), wg.cuda(), we.cuda()
    S, H, P, E, k, EC, pEC = cfg.S, cfg.H, cfg.P, cfg.E, cfg.k, cfg.EC, cfg.pEC
    st = args.stage
    if st in ("gate", "ffn", "combine"):
        out = ctx.forward(xd, wgd, wed, phase_mask=1); ctx.synchronize()
        topk = ctx.read("topk_idx"); slot = ctx.read("slot"); counts = ctx.read("counts"); mcw = ctx.read("mcw")
        amb = ref.ambiguous
        mism = (topk != ref.topk_idx).any(1)
        print(f"  topk mismatching tokens {int(mism.sum())} (ambiguous {int(amb.sum())}, mismatching&non-ambiguous {int((mism & ~amb).sum())})")
        print(f"  slot equal {bool((slot == ref.slot).all())} counts equal {bool((counts == ref.counts).all())} counts {counts.tolist()}")
        print(f"  mcw max rel diff {float(np.max(np.abs(mcw - ref.mcw) / np.maximum(ref.mcw, 1e-30))):.3e}")
        tw = ctx.read("topk_w"); refw = np.take_along_axis(ref.gate_out, ref.topk_idx, axis=1)
        print(f"  topk_w bit-exact frac {float((tw == refw).mean()):.6f}")
        go = ctx.read("gate_out"); print(f"  gate_out bit-exact frac {float((go == ref.gate_out).mean()):.6f}")
        rx = ctx.read("recv_x")  # [E(pkts), pEC, H]
        xb = mo.to_bits(x.view(S, H)); bad = 0; tot = 0
        for t in range(S):
            for j in range(k):
                if ref.kept[t, j] and not mism[t]:
                    tot += 1
                    if not (rx[ref.topk_idx[t, j], ref.slot[t, j]] == xb[t]).all(): bad += 1
        print(f"  dispatch rows checked {tot}, wrong {bad}")
    if st in ("ffn", "combine"):
        ctx.forward(xd, wgd, wed, phase_mask=2); ctx.synchronize()
        rx = ctx.read("recv_x"); hid = ctx.read("hidden"); rc = ctx.read("recv_cnt")
        ry = ctx.read("ret_y")  # needs FM_FUSED_COMBINE=0 (the fused path has no return buffer)
        print("  recv_cnt", rc.tolist())
        for e in range(E):
            n = int(min(counts[e], EC))
            if n == 0: continue
            h_ref, y_ref = mo.expert_ffn(rx[e, :n], up[e], down[e], act=cfg.hidden_act)
            cmp_bf16(f"expert {e} rows {n} hidden", hid[e, :n], h_ref)
            cmp_bf16(f"expert {e} rows {n} y     ", ry[e, :n], y_ref)
            if e >= 1 and not args.all_experts: break
    if st == "combine":
        out = torch.empty_like(xd)
        ctx.forward(xd, wgd, wed, out=out, phase_mask=4); ctx.synchronize()
        cmp_bf16("out (staged)", mo.to_bits(out.cpu().view(S, H)), ref.out)
    if st == "full":
        out = ctx.forward(xd, wgd, wed); ctx.synchronize()
        topk = ctx.read("topk_idx"); mism = (topk != ref.topk_idx).any(1)
        print(f"  topk mismatching tokens {int(mism.sum())} non-ambiguous {int((mism & ~ref.ambiguous).sum())}")
        cmp_bf16("out (fused)", mo.to_bits(out.cpu().view(S, H)), ref.out)
        out2 = ctx.forward(xd, wgd, wed); ctx.synchronize()
        print("  second launch identical:", bool((out2 == out).all()))
    if st == "time":
        out = ctx.forward(xd, wgd, wed); ctx.synchronize()
        for _ in range(5): ctx.forward(xd, wgd, wed, out=out)
        ev0 = torch.cuda.Event(enable_timing=True); ev1 = torch.cuda.Event(enable_timing=True)
        n = 20
        ev0.record()
        for _ in range(n): ctx.forward(xd, wgd, wed, out=out)
        ev1.record(); ctx.synchronize()
        ms = ev0.elapsed_time(ev1) / n
        flops = 4.0 * min(S * k, E * EC) * H * P + 2.0 * S * H * E
        print(f"  {ms*1e3:.1f} us/forward  {S/ms*1e3/1e6:.2f} Mtok/s  ~{flops/ms/1e9:.1f} TFLOP/s (upper bound on rows)")
        for mask, nm in ((1, "gate+dispatch"), (2, "ffn"), (4, "combine")):
            ev0.record()
            for _ in range(n): ctx.forward(xd, wgd, wed, out=out, phase_mask=mask)
            ev1.record(); ctx.synchronize()
            print(f"  phase {nm}: {ev0.elapsed_time(ev1)/n*1e3:.1f} us")
    if st == "trace":
        print("  the per-tile timeline lives in scripts/trace_gantt.py (single GPU) and scripts/trace_multi.py (torchrun)")
    ctx.close()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", default="small"); ap.add_argument("--stage", default="all")
    ap.add_argument("--noscale", action="store_true"); ap.add_argument("--all-experts", dest="all_experts", action="store_true")
    args = ap.parse_args()
    if args.stage == "all":
        for st in ("gate", "ffn", "combine", "full", "time"):
            print(f"===== stage {st} ({args.cfg}) =====", flush=True)
            cmd = [sys.executable, __file__, "--cfg", args.cfg, "--stage", st] + (["--noscale"] if args.noscale else [])
            r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
            print(r.stdout[-6000:]); 
            if r.returncode != 0: print("STAGE FAILED rc", r.returncode, "\n", r.stderr[-3000:])
    else:
        stage(args)
