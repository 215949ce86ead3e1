"""What the per-feature benchmark scripts share: the card description, the command-line pieces, CUDA-event windows, the
alternating rounds of arms, and the workloads more than one script runs.

Every script runs two or three arms (ways of doing the same forward) alternately: each arm is warmed up, then timed
once per round in a window of `steps` calls, so that drift of the clocks or of the other work on the host spreads over
all arms alike.
"""
from __future__ import annotations

import statistics
import sys

import torch

import bench
from flashmoe_b200.config import MoEConfig
from flashmoe_b200.router import RouterSpec

RULE = RouterSpec("sigmoid", 8, 4, 2, True, 2.5)   # DeepSeek-V3's router rule
# DeepSeek-V3's layer shape on one GPU: 15 GB of expert weights, generated on the device by inputs()
DSV3 = MoEConfig(num_experts=256, expert_top_k=8, sequence_len=4096, hidden_size=7168, intermediate_size=2048)


def card(dev):
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None, "sm_max_mhz": None}
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(dev.index)
        info["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:
        pass
    return info


def add_run_args(ap, tokens, steps, warmup, rounds):
    """--tokens (required when `tokens` is None), --steps, --warmup and --rounds with the script's defaults."""
    ap.add_argument("--tokens", default=tokens, required=tokens is None, metavar="N1,N2,..")
    ap.add_argument("--steps", type=int, default=steps)
    ap.add_argument("--warmup", type=int, default=warmup)
    ap.add_argument("--rounds", type=int, default=rounds)


def parse_tokens(ap, text, S):
    try:
        tokens = [int(t) for t in text.split(",") if t.strip()]
    except ValueError:
        ap.error(f"--tokens takes a comma-separated list of integers, got {text!r}")
    if not tokens or any(n < 0 or n > S for n in tokens):
        ap.error(f"--tokens: every count must be in [0, S = {S}]")
    return tokens


def parse_names(ap, flag, text, known):
    """The comma-separated workload names of `flag`, each a key of `known`."""
    names = [c for c in text.split(",") if c]
    bad = [c for c in names if c not in known]
    if not names or bad:
        ap.error(f"{flag}: unknown {bad}; choose from {sorted(known)}")
    return names


def check_counts(ap, args, warmup=False):
    """--steps and --rounds >= 1, and with `warmup` also --warmup >= 0."""
    if args.steps < 1 or args.rounds < 1 or (warmup and args.warmup < 0):
        ap.error("--steps and --rounds must be >= 1" + (", --warmup >= 0" if warmup else ""))


def no_cuda(script):
    """Exit status 3 for a machine without a CUDA device: there is nothing to time."""
    print(f"{script}: no CUDA device; the MoE forward path has no CPU fallback", file=sys.stderr)
    return 3


def device_ms(fn, steps, settle):
    """Device time per call of `steps` calls of fn between two CUDA events; settle() runs after the second is recorded
    and must wait for it (a device synchronise, or a barrier that includes one)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    settle()
    return e0.elapsed_time(e1) / steps


def alternate(arms, warmup, rounds, settle, window):
    """Warm up every arm `warmup` times, settle() once, then `rounds` rounds that each time every arm once with
    window(fn), in the order of `arms`.  Returns {arm: [one result per round]}."""
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    settle()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(window(fn))
    return times


def medians(times):
    """{arm: median of its windows, arm + "_runs": the windows} for the JSON line."""
    out = {}
    for k, v in times.items():
        out[k] = statistics.median(v)
        out[k + "_runs"] = v
    return out


def inputs(name, cfg, dev):
    """Seeded x [S, H], gate weights and expert weights on the device: bench.py's for its configs, else generated on the
    device (DSV3)."""
    if name in bench.BASELINE_CONFIGS:
        x, wg, we = bench.make_inputs(cfg, cfg.E, 0)
        return x.to(dev).view(cfg.S, cfg.H), wg.to(dev), we.to(dev)
    g = torch.Generator(device=dev).manual_seed(0x5EED)
    x = torch.randn(cfg.S, cfg.H, generator=g, device=dev).bfloat16()
    wg = (torch.randn(cfg.H, cfg.E, generator=g, device=dev) * cfg.H ** -0.5).bfloat16()
    we = torch.empty(cfg.E, 2, cfg.P, cfg.H, dtype=torch.bfloat16, device=dev)
    for e in range(cfg.E):   # (one expert at a time: no fp32 copy of the 15 GB)
        we[e] = (torch.randn(2, cfg.P, cfg.H, generator=g, device=dev) * cfg.H ** -0.5).bfloat16()
    return x, wg, we
