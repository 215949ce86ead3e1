"""Per-GPU worker (reference flashmoe/worker.py): initialise, build synthetic tensors from the config JSON, run the
forward with the reference's measurement protocol (32 warm-up + 32 timed launches, csrc/include/flashmoe/moe/moe.cuh:146-184)
and print the reference's result line."""
from __future__ import annotations

import json
import os
import sys

import torch

if __package__ in (None, ""):
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from flashmoe_b200 import _C, config as _config
else:
    from . import _C, config as _config

# schema enum (csrc/flashmoe_config.schema.json): 0 fp32, 1 tf32, 2 bf16, 3 fp16; the reference's worker maps
# {0: float16, 1: float32} and cannot reach bf16 (worker.py:47-48) -- fixed here.
DTYPES = {0: torch.float32, 1: torch.float32, 2: torch.bfloat16, 3: torch.float16}


def make_inputs(cfg: "_config.MoEConfig", nlx: int, rank: int, device, scaled: bool = False):
    """x per rank, gate weights identical on all ranks (seeded), local expert weights per rank."""
    dtype = DTYPES[cfg.torch_dtype]
    g = torch.Generator(device="cpu").manual_seed(0x5EED + rank)
    gw = torch.Generator(device="cpu").manual_seed(0x5EED)
    x = torch.randn(cfg.mini_batch, cfg.sequence_len, cfg.H, generator=g)
    wg = torch.randn(cfg.H, cfg.E, generator=gw)
    we = torch.randn(nlx, cfg.expert_mats, cfg.P, cfg.H, generator=g)   # SwiGLU: [nLx, 3, P, H]
    if scaled:
        wg, we = wg * cfg.H ** -0.5, we * cfg.H ** -0.5
    return x.to(dtype).to(device), wg.to(dtype).to(device), we.to(dtype).to(device)


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        print("ERROR: Config path not provided", file=sys.stderr)
        return 1
    raw = json.load(open(argv[0]))
    cfg = _config.from_dict(raw)
    compiled = _config.from_dict(_C._lib.compiled_config().raw(), validate=False)
    if cfg.raw() != compiled.raw():
        print("ERROR: config file does not match the compiled configuration; rebuild with "
              "`python -m flashmoe_b200._build`", file=sys.stderr)
        return 2
    _C.initialize()
    ctx = _C.context()
    rank, world = ctx.rank, ctx.world
    print(f"Process {rank}/{world} using GPU {ctx.device.index}", flush=True)
    nlx = _C.get_num_local_experts()
    print(f"Process {rank}: Creating {nlx} local experts (total {cfg.E})", flush=True)
    x, wg, we = make_inputs(cfg, nlx, rank, ctx.device)
    print(f"Process {rank}: Calling moe_forward...", flush=True)
    out = torch.empty_like(x)
    warm, trials = 32, 32
    for _ in range(warm):
        ctx.forward(x, wg, we, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(trials):
        ctx.forward(x, wg, we, out=out)
    e1.record()
    ctx.synchronize()
    ms = e0.elapsed_time(e1) / trials
    print(f"Process {rank}: FlashMoE forward pass took {ms:.2f} ms", flush=True)
    print(f"Process {rank}: Completed! Output: {out.shape}", flush=True)
    _C.finalize()
    return 0


if __name__ == "__main__":
    sys.exit(main())
