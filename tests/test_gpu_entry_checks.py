"""The argument checks of the forward entry points on one H100: each rejection through every entry point it applies to,
with the return code and message, no launch issued and the next good call on the context exact; and the tensor maps
over the symmetric slab re-keyed when a world-1 context adopts an external one (fm_symm_use_external)."""
import ctypes
import re

import pytest
import torch

from flashmoe_b200 import _lib
from flashmoe_b200.config import MoEConfig
from tests.util import make_inputs

pytestmark = pytest.mark.gpu

# E = 32: the router runs on the tensor cores, so the maps over x and the gate weights are encoded too
CFG = MoEConfig(num_experts=32, expert_top_k=2, sequence_len=256, hidden_size=128, intermediate_size=128)
S = CFG.S


def _ctx(cfg):
    from flashmoe_b200.runtime import MoEContext

    return MoEContext(cfg, timeout_ms=5000)


class Args:
    """Good arguments for every entry point of one context (device pointers as ints), and the calls themselves."""

    def __init__(self, ctx, cfg, seed):
        dev = ctx.device
        x, wg, we, bu, bd = make_inputs(cfg, seed=seed, bias=True)
        g = torch.Generator().manual_seed(seed)
        self.ctx = ctx
        self.keep = dict(
            x=x.reshape(cfg.S, cfg.H).to(dev), gw=wg.to(dev), we=we.to(dev), bu=bu.to(dev), bd=bd.to(dev),
            out=torch.empty(cfg.S, cfg.H, dtype=torch.bfloat16, device=dev),
            idx=torch.randint(0, cfg.E, (cfg.S, cfg.k), generator=g, dtype=torch.int32).to(dev),
            w=torch.rand(cfg.S, cfg.k, generator=g).to(dev),
            sb=(torch.randn(cfg.E, generator=g) * 0.05).to(dev),
            count=torch.full((4,), cfg.S, dtype=torch.int32, device=dev),
            x_host=x.reshape(cfg.S, cfg.H).pin_memory(),
            out_host=torch.empty(cfg.S, cfg.H, dtype=torch.bfloat16).pin_memory())
        groups = 4 if cfg.E % 4 == 0 else 1   # a rule valid on every context here
        self.router = _lib.FmRouter(scoring=1, n_group=groups, topk_group=min(2, groups), group_top=2, renormalize=1,
                                    scale=2.5)
        self.ptr = {k: t.data_ptr() for k, t in self.keep.items()}
        self.ptr.update(n=cfg.S, n_dev=None, router=ctypes.byref(self.router),
                        stream=torch.cuda.current_stream(dev).cuda_stream)

    def good(self, entry):
        return {**self.ptr, "n_dev": self.ptr["count"]} if entry == "tokens_dev" else dict(self.ptr)

    def call(self, entry, a):
        L, c, s = self.ctx._L, self.ctx._ctx, a["stream"]
        if entry == "forward":
            return L.fm_moe_forward(c, a["x"], a["gw"], a["we"], a["bu"], a["bd"], a["out"], s)
        if entry == "tokens":
            return L.fm_moe_forward_tokens(c, a["x"], a["n"], a["gw"], a["we"], a["bu"], a["bd"], a["out"], s)
        if entry == "tokens_dev":
            return L.fm_moe_forward_tokens_dev(c, a["x"], a["n_dev"], a["gw"], a["we"], a["bu"], a["bd"], a["out"], s)
        if entry == "routed":
            return L.fm_moe_forward_routed(c, a["x"], a["n"], a["n_dev"], a["idx"], a["w"], a["we"], a["bu"], a["bd"],
                                           a["out"], s)
        if entry == "gated":
            return L.fm_moe_forward_gated(c, a["x"], a["n"], a["n_dev"], a["gw"], a["router"], a["sb"], a["we"],
                                          a["bu"], a["bd"], a["out"], s)
        assert entry == "host"
        ticket = ctypes.c_uint64()
        rc = L.fm_host_submit(c, a["x_host"], a["gw"], a["we"], a["bu"], a["bd"], a["out_host"], s,
                              ctypes.byref(ticket))
        return rc if rc else L.fm_host_wait(c, ticket.value)

    def good_output(self, entry):
        """The bits of the output of a good call."""
        assert self.call(entry, self.good(entry)) == 0, self.ctx._L.fm_last_error()
        self.ctx.synchronize()
        return self.keep["out_host" if entry == "host" else "out"].view(torch.int16).clone()


DEVICE = ("forward", "tokens", "tokens_dev", "routed", "gated")
HOST_COUNT = ("tokens", "routed", "gated")
CASES = {
    # name: (entry points, the bad arguments (from the good pointers), pattern of fm_last_error)
    "n_minus_one": (HOST_COUNT, lambda p: {"n": -1}, rf"^n_tokens = -1 not in \[0, S = {S}\]"),
    "n_S_plus_one": (HOST_COUNT, lambda p: {"n": S + 1}, rf"^n_tokens = {S + 1} not in \[0, S = {S}\]"),
    "device_count_n_not_S": (("routed", "gated"), lambda p: {"n": 5, "n_dev": p["count"]},
                             rf"^with n_tokens_dev, n_tokens must be S = {S}"),
    "null_count_pointer": (("tokens_dev",), lambda p: {"n_dev": None}, r"^n_tokens_dev must point"),
    "misaligned_count_pointer": (("tokens_dev", "routed", "gated"), lambda p: {"n_dev": p["count"] + 2},
                                 r"^n_tokens_dev must be 4-byte aligned"),
    "null_x": (DEVICE, lambda p: {"x": None}, r"^x must be a non-null device pointer"),
    "null_out": (DEVICE, lambda p: {"out": None}, r"^out must be a non-null device pointer"),
    "null_expert_w": (DEVICE + ("host",), lambda p: {"we": None}, r"^expert_w must be a non-null device pointer"),
    "null_gate_w": (("forward", "tokens", "tokens_dev", "gated", "host"), lambda p: {"gw": None},
                    r"^gate_w must be a non-null device pointer"),
    "null_topk": (("routed",), lambda p: {"idx": None}, r"^topk_idx must be a non-null device pointer"),
    "null_router": (("gated",), lambda p: {"router": None}, r"^router must point to an fm_router_t"),
    "misaligned_x": (DEVICE, lambda p: {"x": p["x"] + 2}, r"^x must be 16-byte aligned"),
    "misaligned_out": (DEVICE, lambda p: {"out": p["out"] + 2}, r"^out must be 16-byte aligned"),
    "misaligned_expert_w": (DEVICE + ("host",), lambda p: {"we": p["we"] + 2}, r"^expert_w must be 16-byte aligned"),
    "misaligned_topk_idx": (("routed",), lambda p: {"idx": p["idx"] + 4}, r"^topk_idx must be 16-byte aligned"),
    "misaligned_topk_w": (("routed",), lambda p: {"w": p["w"] + 4}, r"^topk_w must be 16-byte aligned"),
    "misaligned_score_bias": (("gated",), lambda p: {"sb": p["sb"] + 4}, r"^score_bias must be 16-byte aligned"),
}
PAIRS = [(case, entry) for case, (entries, _, _) in CASES.items() for entry in entries]


@pytest.fixture(scope="module")
def env():
    ctx = _ctx(CFG)
    args = Args(ctx, CFG, seed=71)
    want = {entry: args.good_output(entry) for entry in DEVICE + ("host",)}
    yield args, want
    ctx.close()


@pytest.mark.parametrize("case,entry", PAIRS, ids=[f"{c}-{e}" for c, e in PAIRS])
def test_rejected_through_every_entry_point(env, case, entry):
    args, want = env
    _, bad, pattern = CASES[case]
    launches = args.ctx.launch_count
    assert args.call(entry, {**args.good(entry), **bad(args.ptr)}) == -1
    msg = args.ctx._L.fm_last_error().decode()
    assert re.search(pattern, msg), msg
    assert args.ctx.launch_count == launches
    assert torch.equal(args.good_output(entry), want[entry])


@pytest.mark.parametrize("entry", ["routed", "gated"])
@pytest.mark.parametrize("kw,pattern", [(dict(num_experts=1, expert_top_k=1), "E = 1"),
                                        (dict(is_training=1), "is_training")], ids=["E1", "training"])
def test_rejected_contexts(kw, pattern, entry):
    cfg = CFG.replace(**kw)
    ctx = _ctx(cfg)
    args = Args(ctx, cfg, seed=72)
    want = args.good_output("tokens")
    launches = ctx.launch_count
    assert args.call(entry, args.good(entry)) == -1
    msg = ctx._L.fm_last_error().decode()
    assert pattern in msg, msg
    assert ctx.launch_count == launches
    assert torch.equal(args.good_output("tokens"), want)
    ctx.close()


def test_external_slab_rekeys_the_maps_over_it():
    """A forward, a forward on other inputs, then the context moves to a zeroed external slab: the first forward again
    is bit-identical.  (A map left over the old slab would read the other inputs' dispatched rows.)"""
    ctx = _ctx(CFG)
    dev = ctx.device
    x, wg, we, _, _ = make_inputs(CFG, seed=73)
    x2, _, _, _, _ = make_inputs(CFG, seed=74)
    xd, x2d, wgd, wed = x.to(dev), x2.to(dev), wg.to(dev), we.to(dev)
    want = ctx.forward(xd, wgd, wed).clone()
    ctx.forward(x2d, wgd, wed)
    ctx.synchronize()
    nbytes = ctypes.c_size_t()
    _lib.check(ctx._L.fm_symm_size(ctx._ctx, ctypes.byref(nbytes)))
    slab = torch.zeros(nbytes.value + 1024, dtype=torch.uint8, device=dev)
    base = (slab.data_ptr() + 1023) // 1024 * 1024
    _lib.check(ctx._L.fm_symm_use_external(ctx._ctx, base, nbytes.value))
    got = ctx.forward(xd, wgd, wed)
    ctx.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    assert slab.any(), "the forward did not use the external slab"
    ctx.close()
