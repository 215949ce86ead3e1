"""Host-side runtime above the C-ABI: one `MoEContext` per process / GPU.

Mirrors what the reference does in `flashmoe::initialize()` + `moe_forward` (csrc/include/flashmoe/bootstrap.cuh:278-547,
csrc/python_bindings.cu:17-151) with torch used only for device memory, streams and the out-of-band exchange of
CUDA IPC handles (`torch.distributed`, any backend) -- plumbing, not the product.  All math runs in the native
library; nothing here falls back to torch ops.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import _lib, trace_slots
from .config import MoEConfig
from .router import RouterSpec

_BUFFER_SPECS = {
    "topk_idx": (_lib.BUF_TOPK_IDX, np.int32),
    "topk_w": (_lib.BUF_TOPK_W, np.uint16),
    "mcw": (_lib.BUF_MCW, np.float32),
    "slot": (_lib.BUF_SLOT, np.int32),
    "counts": (_lib.BUF_COUNTS, np.int32),
    "recv_x": (_lib.BUF_RECV_X, np.uint16),
    "hidden": (_lib.BUF_HIDDEN, np.uint16),
    "ret_y": (_lib.BUF_RET_Y, np.uint16),
    "gate_out": (_lib.BUF_GATE_OUT, np.uint16),
    "recv_cnt": (_lib.BUF_RECV_CNT, np.int32),
    "trace": (_lib.BUF_TRACE, np.uint64),
    "aux_loss": (_lib.BUF_AUX_LOSS, np.float32),
    "shared_y": (_lib.BUF_SHARED_Y, np.uint16),
    "shared_hidden": (_lib.BUF_SHARED_HIDDEN, np.uint16),
}


def env_rank_world() -> Tuple[int, int, int]:
    """(rank, world, local_rank) from torchrun's env, falling back to the launchers the reference's worker reads
    (OMPI / PMI / SLURM, reference flashmoe/worker.py:24-29)."""
    def first(*names: str, default: str) -> int:
        for n in names:
            if n in os.environ:
                return int(os.environ[n])
        return int(default)

    rank = first("RANK", "OMPI_COMM_WORLD_RANK", "PMI_RANK", "SLURM_PROCID", default="0")
    world = first("WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "PMI_SIZE", "SLURM_NTASKS", default="1")
    local = first("LOCAL_RANK", "OMPI_COMM_WORLD_LOCAL_RANK", "SLURM_LOCALID", default=str(rank))
    return rank, world, local


def exchange_blobs(mine: bytes, world: int, group=None) -> bytes:
    """All-gather one fixed-size byte string per rank over torch.distributed (any backend) and return them
    concatenated in rank order -- the out-of-band channel for the CUDA IPC handles of the symmetric slabs."""
    import torch.distributed as dist

    if not dist.is_initialized():
        raise RuntimeError("world > 1 needs an initialised torch.distributed process group")
    gathered = [None] * world
    dist.all_gather_object(gathered, mine, group=group)
    if any(len(g) != len(mine) for g in gathered):
        raise RuntimeError("peers exported handles of different sizes")
    return b"".join(gathered)


def _check_tensor(name: str, t: torch.Tensor, device: torch.device, dtype: torch.dtype = torch.bfloat16,
                  shape: Optional[Dict[str, int]] = None, aligned: bool = True) -> None:
    """A tensor argument of a C call: a contiguous CUDA tensor on `device` of `dtype`, shaped `shape` when given (named
    dimensions: {"n": 5, "k": 2} is [n=5, k=2]), starting on a 16-byte boundary when `aligned`.  Reads metadata only (no
    .item()): a check must not synchronise, and may run under stream capture."""
    if not isinstance(t, torch.Tensor) or t.device != device:
        raise RuntimeError(f"{name} must be a CUDA tensor on {device}, got {getattr(t, 'device', type(t).__name__)}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must be {dtype}, got {t.dtype}")
    if shape is not None and t.shape != tuple(shape.values()):
        dims = ", ".join(f"{k}={v}" for k, v in shape.items())
        raise RuntimeError(f"{name} must be [{dims}], got {list(t.shape)}")
    if aligned and t.data_ptr() % 16:
        raise RuntimeError(f"{name} must start on a 16-byte boundary (TMA tensor maps, bulk row copies and the vector "
                           f"accesses need it); got storage offset {t.storage_offset()}")


class SharedExpert(NamedTuple):
    """A shared expert (fm_moe_forward_shared): a dense FFN every token passes through, its output added to the routed
    combine.  `w` bf16 [2, Ps, H] is one routed expert's layout ([0] = W_up [Ps, H], [1] flat-viewed as W_down [H, Ps]);
    `bias_up` bf16 [Ps] and `bias_down` bf16 [H] are optional.  Ps is a multiple of 64.  In a SwiGLU context
    (hidden_act = 2) `w` is [3, Ps, H] (W_gate, W_up, W_down flat-viewed) and `bias_up` [2, Ps] (gate, then up).  Several shared experts of size P
    are one of size n_shared * P: concatenate their W_up rows and their W_down columns."""
    w: torch.Tensor
    bias_up: Optional[torch.Tensor] = None
    bias_down: Optional[torch.Tensor] = None


def shared_expert_struct(se: SharedExpert, device: torch.device, H: int, reserved: Optional[int],
                         swiglu: bool = False) -> _lib.FmSharedExpert:
    """Check a `SharedExpert` against a context on `device` with hidden size H and reserved intermediate size `reserved`
    (None: not reserved), SwiGLU experts when `swiglu`, and return its fm_shared_expert_t.  The caller keeps the tensors
    alive."""
    if not isinstance(se, SharedExpert):
        raise TypeError(f"shared_expert must be a SharedExpert, got {type(se).__name__}")
    if reserved is None:
        raise RuntimeError("this context has no shared-expert staging: create it with shared_inter=")
    mats = "[3, Ps, H]" if swiglu else "[2, Ps, H]"
    if not isinstance(se.w, torch.Tensor) or se.w.dim() != 3:
        raise RuntimeError(f"shared_expert.w must be a 3-D tensor {mats}, got {getattr(se.w, 'shape', se.w)}")
    ps = int(se.w.shape[1])
    _check_tensor("shared_expert.w", se.w, device,
                  shape={"gate/up/down": 3, "Ps": ps, "H": H} if swiglu else {"up/down": 2, "Ps": ps, "H": H})
    if ps <= 0 or ps % 64:
        raise RuntimeError(f"shared_expert.w: Ps = {ps} must be a positive multiple of 64")
    if ps > reserved:
        raise RuntimeError(f"shared_expert.w: Ps = {ps} is above the context's shared_inter = {reserved}")
    up_dims = {"gate/up": 2, "Ps": ps} if swiglu else {"Ps": ps}
    for name, b, dims in (("bias_up", se.bias_up, up_dims), ("bias_down", se.bias_down, {"H": H})):
        if b is not None:
            _check_tensor(f"shared_expert.{name}", b, device, shape=dims)
    return _lib.FmSharedExpert(se.w.data_ptr(), se.bias_up.data_ptr() if se.bias_up is not None else None,
                               se.bias_down.data_ptr() if se.bias_down is not None else None, ps)


def _check_weight_on_input(enable, cfg: MoEConfig) -> None:
    """The conditions of fm_set_weight_on_input, checked before any native call."""
    if enable not in (True, False):
        raise ValueError(f"weight_on_input must be a bool, got {enable!r}")
    if enable and cfg.k != 1:
        raise ValueError(f"weight_on_input needs k = 1 (each pick would need its own copy of the row); got k = {cfg.k}")
    if enable and cfg.E == 1:
        raise ValueError("weight_on_input needs E > 1 (an E = 1 context has no routing)")


class MoEContext:
    """Owns the native context (workspaces, symmetric slab, peer mappings) for one rank."""

    def __init__(self, cfg: Optional[MoEConfig] = None, rank: int = 0, world: int = 1,
                 device: Optional[int] = None, group=None, timeout_ms: Optional[int] = None,
                 symmetric: Optional[str] = None, shared_inter: Optional[int] = None, weight_on_input: bool = False):
        """`symmetric` selects how the peers' slabs are mapped when world > 1: "ipc" (default; cudaMalloc + CUDA IPC
        handles over torch.distributed) or "torch" (the slab is allocated with torch.distributed._symmetric_memory --
        the allocator PyTorch backs with CUDA VMM / NVSHMEM -- and the peer pointers come from its rendezvous; this is
        the hook for externally managed symmetric heaps, reference bootstrap.cuh:359-360,442-443).  Environment
        override: FM_SYMM=ipc|torch.

        `shared_inter`: reserve the staging of a shared expert of intermediate size up to this (a multiple of 64;
        fm_shared_reserve), so that the forward calls accept `shared_expert=`.

        `weight_on_input`: scale each routed token's input row by its router weight instead of the expert's output
        (fm_set_weight_on_input; Llama 4): on `forward_routed` and `forward_gated` a kept pick dispatches
        rne_bf16(x[t] * rne_bf16(w)) and the combine takes weight 1, so out equals a plain context's
        `forward_routed(x', topk_idx, ones)` on the scaled rows x' bit for bit; a shared expert still sees the unscaled x.
        The router route (`forward`, `forward_tokens`) is unchanged.  Needs k = 1 and E > 1 (ValueError otherwise)."""
        if weight_on_input:
            _check_weight_on_input(weight_on_input, cfg if cfg is not None else _lib.compiled_config())
        self._L = _lib.load()
        self._ctx = ctypes.c_void_p()
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", device)
        self.rank, self.world = rank, world
        ccfg = _lib.FmConfig.from_config(cfg) if cfg is not None else None
        _lib.check(self._L.fm_create(ctypes.byref(ccfg) if ccfg is not None else None, rank, world, device,
                                     ctypes.byref(self._ctx)))
        d = _lib.FmDims()
        _lib.check(self._L.fm_get_dims(self._ctx, ctypes.byref(d)))
        self.dims: Dict[str, int] = {k: int(getattr(d, k)) for k, _ in d._fields_}
        self.cfg = cfg if cfg is not None else _lib.compiled_config()
        if timeout_ms is not None:
            _lib.check(self._L.fm_set_timeout_ms(self._ctx, int(timeout_ms)))
        self.shared_inter: Optional[int] = None
        if shared_inter is not None:
            _lib.check(self._L.fm_shared_reserve(self._ctx, int(shared_inter)))
            self.shared_inter = int(shared_inter)
        self.weight_on_input = False
        if weight_on_input:
            self.set_weight_on_input(True)
        # tokens of the last forward (valid rows of the routing tables `read` returns); None after a call with a
        # device-side count (launch_record() has it)
        self.last_tokens: Optional[int] = 0
        self.symmetric = (symmetric or os.environ.get("FM_SYMM") or "ipc").lower()
        self._symm_tensor = None   # keeps an externally allocated slab alive
        if world > 1:
            if self.symmetric == "ipc":
                self._attach_peers(group)
            elif self.symmetric == "torch":
                self._attach_torch_symmetric_memory(group)
            else:
                raise ValueError(f"symmetric must be 'ipc' or 'torch', got {self.symmetric!r}")

    # ------------------------------------------------------------------ peers
    def _attach_peers(self, group) -> None:
        """Exchange CUDA IPC handles of the symmetric slab over torch.distributed and map every peer
        (replaces nvshmem_malloc + nvshmem_ptr, reference bootstrap.cuh:359-360,442-443)."""
        import torch.distributed as dist

        handle = (ctypes.c_ubyte * _lib.FM_IPC_HANDLE_BYTES)()
        _lib.check(self._L.fm_symm_export(self._ctx, handle))
        blob = exchange_blobs(bytes(handle), self.world, group)
        assert len(blob) == self.world * _lib.FM_IPC_HANDLE_BYTES
        _lib.check(self._L.fm_symm_attach_ipc(self._ctx, blob))
        torch.cuda.synchronize(self.device)
        dist.barrier(group=group)  # every rank's slab is mapped (and zeroed) before anyone dispatches into it

    def _attach_torch_symmetric_memory(self, group) -> None:
        """Externally allocated symmetric slab: torch.distributed._symmetric_memory.empty + rendezvous give every rank a
        same-sized allocation and the peers' mapped base pointers; the library adopts them through
        fm_symm_use_external + fm_symm_attach_ptrs (no cudaMalloc / CUDA IPC of its own)."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem

        nbytes = ctypes.c_size_t()
        _lib.check(self._L.fm_symm_size(self._ctx, ctypes.byref(nbytes)))
        n = (nbytes.value + 1023) // 1024 * 1024
        t = symm_mem.empty(n, dtype=torch.uint8, device=self.device)
        t.zero_()
        if t.data_ptr() % 1024:
            raise RuntimeError("symmetric memory allocation is not 1 KiB aligned")
        hdl = symm_mem.rendezvous(t, group if group is not None else dist.group.WORLD)
        ptrs = [int(p) for p in hdl.buffer_ptrs]
        if len(ptrs) != self.world or ptrs[self.rank] != t.data_ptr():
            raise RuntimeError("unexpected symmetric-memory rendezvous result")
        _lib.check(self._L.fm_symm_use_external(self._ctx, t.data_ptr(), n))
        arr = (ctypes.c_void_p * self.world)(*ptrs)
        _lib.check(self._L.fm_symm_attach_ptrs(self._ctx, arr))
        self._symm_tensor, self._symm_handle = t, hdl
        torch.cuda.synchronize(self.device)
        dist.barrier(group=group)

    # ------------------------------------------------------------------ hot path
    @property
    def num_local_experts(self) -> int:
        return self.dims["num_local_experts"]

    def _validate_weights(self, gate_weights: Optional[torch.Tensor], expert_weights: torch.Tensor) -> None:
        """`gate_weights` None: a routed call, which has none."""
        d = self.dims
        if gate_weights is not None:
            _check_tensor("Gate weights", gate_weights, self.device, shape={"H": d["H"], "E": d["E"]})
        _check_tensor("Expert weights", expert_weights, self.device)
        nlx = d["num_local_experts"]
        s = expert_weights.shape
        if len(s) != 4 or s[0] != nlx:
            raise RuntimeError(f"Expert count mismatch. Expected {nlx} local experts, got {s[0]}")
        m = self.cfg.expert_mats
        if s[1] != m:
            raise RuntimeError("Expert weights must have up and down projections [nLx, 2, P, H]" if m == 2 else
                               "SwiGLU expert weights must have gate, up and down projections [nLx, 3, P, H]; got "
                               f"{s[1]} matrices per expert")
        if s[2] != d["P"] or s[3] != d["H"]:
            raise RuntimeError(f"Expert weights must be [*, {m}, P={d['P']}, H={d['H']}]. Got [*, {m}, {s[2]}, {s[3]}]")

    def _validate(self, input: torch.Tensor, gate_weights: Optional[torch.Tensor], expert_weights: torch.Tensor,
                  exact_s: bool = True) -> int:
        """Same conditions as the reference's TORCH_CHECKs (python_bindings.cu:22-65) plus dtype and alignment checks.
        `exact_s`: the input is [batch, seq, H] with batch*seq == S (forward); otherwise any [..., H] holding at most S
        tokens (forward_tokens).  Returns the number of tokens."""
        d = self.dims
        _check_tensor("Input", input, self.device)
        s = input.shape
        if exact_s:
            if len(s) != 3:
                raise RuntimeError("Input must be 3D [batch, seq, H]")
            if s[0] * s[1] != d["S"]:
                raise RuntimeError(f"Input batch*seq must equal compiled S={d['S']}. Got batch={s[0]}, seq={s[1]} "
                                   f"(product={s[0] * s[1]})")
        elif len(s) < 1:
            raise RuntimeError("Input must be [..., H]")
        if s[-1] != d["H"]:
            raise RuntimeError(f"Input hidden_size must equal compiled H={d['H']}. Got {s[-1]}")
        n = input.numel() // d["H"]
        if n > d["S"]:
            raise RuntimeError(f"Input holds {n} tokens, more than the context's S={d['S']}")
        self._validate_weights(gate_weights, expert_weights)
        return n

    def _output(self, input: torch.Tensor, out: Optional[torch.Tensor]) -> torch.Tensor:
        if out is None:
            return torch.empty_like(input)
        _check_tensor("out", out, self.device)
        if out.shape != input.shape:
            raise RuntimeError("out must have the input's shape")
        return out

    def _bias_ptrs(self, bias_up, bias_down):
        d = self.dims
        nlx = d["num_local_experts"]
        up = {"nLx": nlx, "gate/up": 2, "P": d["P"]} if self.cfg.expert_mats == 3 else {"nLx": nlx, "P": d["P"]}
        for name, b, dims in (("bias_up", bias_up, up), ("bias_down", bias_down, {"nLx": nlx, "H": d["H"]})):
            if b is not None:
                _check_tensor(name, b, self.device, shape=dims)
        return (bias_up.data_ptr() if bias_up is not None else None,
                bias_down.data_ptr() if bias_down is not None else None)

    def forward(self, input: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor,
                bias_up: Optional[torch.Tensor] = None, bias_down: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Enqueue one fused forward on torch's current stream; returns the [B,T,H] output tensor (async)."""
        self._validate(input, gate_weights, expert_weights)
        bu, bd = self._bias_ptrs(bias_up, bias_down)
        out = self._output(input, out)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self._L.fm_moe_forward(self._ctx, input.data_ptr(), gate_weights.data_ptr(),
                                          expert_weights.data_ptr(), bu, bd, out.data_ptr(), stream))
        self.last_tokens = self.dims["S"]
        return out

    def forward_tokens(self, x: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor,
                       bias_up: Optional[torch.Tensor] = None, bias_down: Optional[torch.Tensor] = None,
                       out: Optional[torch.Tensor] = None, n_tokens: Optional[torch.Tensor] = None,
                       shared_expert: Optional[SharedExpert] = None) -> torch.Tensor:
        """Enqueue one fused forward over the n = x.numel() // H tokens of `x` (contiguous bf16 [..., H], 0 <= n <= S)
        on torch's current stream; returns `out` (default: a tensor like `x`), async.  The result is exactly what a
        context created for S = n computes: routing, capacity `cfg.EC_of(n)`, drops, outputs and, in training mode, the
        auxiliary loss over the n tokens.  Nothing past row n of `out` is written.  With world > 1 every rank passes its
        own n (n = 0 included) and all ranks call the same number of times.  The routing tables `read` returns then
        hold `last_tokens` valid rows.

        `n_tokens`: a one-element int32 CUDA tensor on this context's device holding n, read by the kernel when it starts
        (fm_moe_forward_tokens_dev): no host synchronisation, and one captured CUDA graph serves every n.  `x` must then
        hold exactly S tokens; its rows n and above may hold anything and affect no result, and rows n and above of
        `out` are not written.  `last_tokens` is then None -- `launch_record()` returns the count the launch ran with.
        A count outside [0, S] runs the launch on 0 tokens and makes the next `check` / `synchronize` raise.

        `shared_expert`: a `SharedExpert` whose output s[t] every token adds to its routed result r[t] (the row this call
        writes without one): out[t] = rne_bf16(r[t] + s[t]); everything else is unchanged.  Needs a context created with
        `shared_inter` >= its Ps; `read("shared_y")` returns the s rows and `read("shared_hidden")` their h_s [S, Ps].
        The same keyword works on `forward_routed` and `forward_gated`."""
        n = self._validate(x, gate_weights, expert_weights, exact_s=False)
        bu, bd = self._bias_ptrs(bias_up, bias_down)
        out = self._output(x, out)
        L, c, stream = self._L, self._ctx, torch.cuda.current_stream(self.device).cuda_stream
        gw, we = gate_weights.data_ptr(), expert_weights.data_ptr()
        if shared_expert is not None:
            se = self._shared(shared_expert)
            self._launch(lambda nd, xp, op: L.fm_moe_forward_shared(c, xp, n, nd, gw, None, None, None, None, we, bu, bd,
                                                                    se, op, stream), n, n_tokens, x, out)
            return out
        # the two C calls differ in their third argument only: the count, or the pointer to it
        fn = L.fm_moe_forward_tokens if n_tokens is None else L.fm_moe_forward_tokens_dev
        self._launch(lambda nd, xp, op: fn(c, xp, n if nd is None else nd, gw, we, bu, bd, op, stream),
                     n, n_tokens, x, out)
        return out

    def forward_routed(self, x: torch.Tensor, topk_idx: torch.Tensor, topk_weight: torch.Tensor,
                       expert_weights: torch.Tensor, bias_up: Optional[torch.Tensor] = None,
                       bias_down: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
                       n_tokens: Optional[torch.Tensor] = None,
                       shared_expert: Optional[SharedExpert] = None) -> torch.Tensor:
        """`forward_tokens` on the caller's routing instead of the built-in router (fm_moe_forward_routed): `topk_idx`
        int32 [n, k] names each token's experts (global ids; -1 = no expert) and `topk_weight` float32 [n, k] their
        weights, both contiguous CUDA tensors on this context's device (no conversions are made here; see
        `FlashMoELayer.forward` for one that converts).  out[t] is the bf16 accumulation, in pick order, of
        rne(rne_bf16(w_j) * y_j) over the kept picks -- for k = 1 too (the router path copies y unscaled there).
        Capacity and slots are the router path's.  An index outside [-1, E) is treated as -1 and makes the next
        `check` / `synchronize` raise once.  Not available on E = 1 or is_training = 1 contexts.

        `n_tokens` (one-element int32 CUDA tensor): as in `forward_tokens`; x, out and the routing tensors then hold S
        rows, of which the kernel reads the first n when it starts."""
        n = self._validate(x, None, expert_weights, exact_s=False)
        routing = {"n": n, "k": self.dims["k"]}
        _check_tensor("topk_idx", topk_idx, self.device, torch.int32, shape=routing, aligned=n > 0)
        _check_tensor("topk_weight", topk_weight, self.device, torch.float32, shape=routing, aligned=n > 0)
        bu, bd = self._bias_ptrs(bias_up, bias_down)
        out = self._output(x, out)
        L, c, stream = self._L, self._ctx, torch.cuda.current_stream(self.device).cuda_stream
        we = expert_weights.data_ptr()
        if shared_expert is not None:
            se = self._shared(shared_expert)
            self._launch(lambda nd, xp, op, ip, wp: L.fm_moe_forward_shared(c, xp, n, nd, None, None, None, ip, wp, we, bu,
                                                                            bd, se, op, stream),
                         n, n_tokens, x, out, topk_idx, topk_weight)
            return out
        self._launch(lambda nd, xp, op, ip, wp: L.fm_moe_forward_routed(c, xp, n, nd, ip, wp, we, bu, bd, op, stream),
                     n, n_tokens, x, out, topk_idx, topk_weight)
        return out

    def forward_gated(self, x: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor,
                      router: RouterSpec, score_bias: Optional[torch.Tensor] = None,
                      bias_up: Optional[torch.Tensor] = None, bias_down: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None, n_tokens: Optional[torch.Tensor] = None,
                      shared_expert: Optional[SharedExpert] = None) -> torch.Tensor:
        """`forward_tokens` with the routing rule `router` (a `RouterSpec`) applied in the kernel to the router's logits
        (fm_moe_forward_gated): softmax or sigmoid scores, an optional `score_bias` added for selection only, a group
        limit, top-k, renormalisation and a route scale.  From the routing on, the launch runs exactly as
        `forward_routed` on its own topk_idx and weights: the weights are `rne_bf16(w)`, k = 1 is scaled, mcw = 1,
        gate_out holds the unbiased scores.  `score_bias`: contiguous float32 [E] CUDA tensor on this device (global
        expert ids), read when each launch starts (a captured graph follows in-place updates).  `n_tokens` as in
        `forward_tokens`.  Not available on E = 1 or is_training = 1 contexts."""
        if not isinstance(router, RouterSpec):
            raise TypeError(f"router must be a RouterSpec, got {type(router).__name__}")
        d = self.dims
        router.check(d["E"], d["k"])
        n = self._validate(x, gate_weights, expert_weights, exact_s=False)
        if score_bias is not None:
            _check_tensor("score_bias", score_bias, self.device, torch.float32, shape={"E": d["E"]})
        bu, bd = self._bias_ptrs(bias_up, bias_down)
        out = self._output(x, out)
        L, c, stream = self._L, self._ctx, torch.cuda.current_stream(self.device).cuda_stream
        gw, rt, we = gate_weights.data_ptr(), ctypes.byref(router.to_c()), expert_weights.data_ptr()
        sb = score_bias.data_ptr() if score_bias is not None else None
        if shared_expert is not None:
            se = self._shared(shared_expert)
            self._launch(lambda nd, xp, op: L.fm_moe_forward_shared(c, xp, n, nd, gw, rt, sb, None, None, we, bu, bd, se,
                                                                    op, stream), n, n_tokens, x, out)
            return out
        self._launch(lambda nd, xp, op: L.fm_moe_forward_gated(c, xp, n, nd, gw, rt, sb, we, bu, bd, op, stream),
                     n, n_tokens, x, out)
        return out

    def _shared(self, se: SharedExpert):
        return ctypes.byref(shared_expert_struct(se, self.device, self.dims["H"], self.shared_inter,
                                                 swiglu=self.cfg.expert_mats == 3))

    def _launch(self, call, n: int, n_tokens: Optional[torch.Tensor], *rows: torch.Tensor) -> None:
        """The token-count convention of the forward calls: run `call(n_tokens_dev, *row pointers)`, where `rows` are
        the tensors with one row per token (x, out, the routing arrays), then set `last_tokens`.  A host count (n_tokens
        None) passes no count pointer, and no row pointers at n = 0 (nothing reads them).  A device count is a
        one-element int32 CUDA tensor the kernel reads when it starts; the rows are then S, and `last_tokens` is None
        (`launch_record()` has the count)."""
        if n_tokens is None:
            _lib.check(call(None, *[t.data_ptr() for t in rows]) if n else call(None, *[None] * len(rows)))
            self.last_tokens = n
            return
        _check_tensor("n_tokens", n_tokens, self.device, torch.int32, aligned=False)   # the C side asks for 4 bytes
        if n_tokens.numel() != 1:
            raise RuntimeError(f"n_tokens must be a one-element torch.int32 tensor, got {n_tokens.numel()} elements")
        if n != self.dims["S"]:
            raise RuntimeError(f"with a device-side n_tokens, x must hold exactly S={self.dims['S']} tokens (got {n})")
        _lib.check(call(n_tokens.data_ptr(), *[t.data_ptr() for t in rows]))
        self.last_tokens = None

    def launch_record(self) -> Tuple[int, int]:
        """(launches, n_tokens): how many launches this context has run on the device -- graph replays included, unlike
        `launch_count` -- and the token count the last one ran with (0 after an out-of-range device count).
        Synchronises the device."""
        launches, n = ctypes.c_uint64(), ctypes.c_int32()
        _lib.check(self._L.fm_last_launch(self._ctx, ctypes.byref(launches), ctypes.byref(n)))
        return int(launches.value), int(n.value)

    def _host_args(self, input_host, gate_weights, expert_weights, out_host, bias_up, bias_down):
        d = self.dims
        for name, t in (("input_host", input_host), ("out_host", out_host)):
            if t is None:
                continue
            if t.is_cuda or t.dtype != torch.bfloat16 or not t.is_contiguous():
                raise RuntimeError(f"{name} must be a contiguous CPU torch.bfloat16 tensor")
            if t.numel() != d["S"] * d["H"]:
                raise RuntimeError(f"{name} must hold S*H = {d['S'] * d['H']} elements")
        self._validate_weights(gate_weights, expert_weights)
        bu, bd = self._bias_ptrs(bias_up, bias_down)
        if out_host is None:
            out_host = torch.empty_like(input_host, pin_memory=True)
        return out_host, bu, bd

    def forward_host(self, input_host: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor,
                     out_host: Optional[torch.Tensor] = None, bias_up: Optional[torch.Tensor] = None,
                     bias_down: Optional[torch.Tensor] = None) -> torch.Tensor:
        """End-to-end call with HOST activations (pinned for full PCIe rate): H2D copy, fused forward, D2H copy, wait.
        Weights stay device-resident (they are parameters, not per-step inputs).  Blocking; for throughput use
        submit_host / wait_host, which keep up to three steps in flight so the copies overlap the kernels."""
        out_host, bu, bd = self._host_args(input_host, gate_weights, expert_weights, out_host, bias_up, bias_down)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self._L.fm_moe_forward_host(self._ctx, input_host.data_ptr(), gate_weights.data_ptr(),
                                               expert_weights.data_ptr(), bu, bd, out_host.data_ptr(), stream))
        return out_host

    def submit_host(self, input_host: torch.Tensor, gate_weights: torch.Tensor, expert_weights: torch.Tensor,
                    out_host: torch.Tensor, bias_up: Optional[torch.Tensor] = None,
                    bias_down: Optional[torch.Tensor] = None) -> int:
        """Asynchronous host-buffer step: enqueue H2D copy -> layer -> D2H copy and return a ticket at once
        (at most `_lib.FM_HOST_SLOTS` tickets outstanding).  `out_host` is complete after `wait_host(ticket)`."""
        out_host, bu, bd = self._host_args(input_host, gate_weights, expert_weights, out_host, bias_up, bias_down)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        ticket = ctypes.c_uint64()
        _lib.check(self._L.fm_host_submit(self._ctx, input_host.data_ptr(), gate_weights.data_ptr(),
                                          expert_weights.data_ptr(), bu, bd, out_host.data_ptr(), stream,
                                          ctypes.byref(ticket)))
        return int(ticket.value)

    def wait_host(self, ticket: int) -> None:
        _lib.check(self._L.fm_host_wait(self._ctx, int(ticket)))

    def output_buffer(self) -> torch.Tensor:
        """A [mini_batch, seq, H] bf16 tensor to pass as `out=`.  With world > 1 it aliases the region of this rank's
        symmetric slab that the experts accumulate into, so `forward(..., out=ctx.output_buffer())` leaves the result in
        place instead of copying it to a caller tensor at the end of the kernel (it is overwritten by the next forward
        and dies with the context).  With world == 1 the kernel accumulates into any `out`; a fresh tensor is returned."""
        shape = (self.cfg.mini_batch, self.cfg.sequence_len, self.dims["H"])
        ptr, nbytes = ctypes.c_void_p(), ctypes.c_size_t()
        _lib.check(self._L.fm_output_buffer(self._ctx, ctypes.byref(ptr), ctypes.byref(nbytes)))
        if not ptr.value:
            return torch.empty(shape, dtype=torch.bfloat16, device=self.device)

        class _Raw:  # CUDA array interface view of the slab region (int16 elements, reinterpreted below)
            __cuda_array_interface__ = {"shape": (nbytes.value // 2,), "typestr": "<i2", "data": (ptr.value, False),
                                        "version": 3}

        return torch.as_tensor(_Raw(), device=self.device).view(torch.bfloat16).view(shape)

    def sync_ranks(self, group=None) -> None:
        """Optional host-side rendezvous before a forward (world > 1).  The kernel's waits are bounded (default 120 s,
        `timeout_ms`) and end in a trap when a peer never shows up; ranks whose skew may exceed that -- first-iteration
        compilation, checkpoint I/O, a debugger -- can line up here first."""
        if self.world > 1:
            import torch.distributed as dist

            torch.cuda.synchronize(self.device)
            dist.barrier(group=group)

    def set_trace(self, enable: bool) -> None:
        _lib.check(self._L.fm_set_trace(self._ctx, 1 if enable else 0))

    def set_weight_on_input(self, enable: bool) -> None:
        """Turn the router weight on the input (the constructor's `weight_on_input`) on or off for the next launches; a
        captured graph keeps the setting it was captured with."""
        _check_weight_on_input(enable, self.cfg)
        _lib.check(self._L.fm_set_weight_on_input(self._ctx, 1 if enable else 0))
        self.weight_on_input = bool(enable)

    def check(self) -> None:
        """Raise if the last kernel reported a protocol timeout (call after a synchronise)."""
        _lib.check(self._L.fm_check(self._ctx))

    def synchronize(self) -> None:
        try:
            torch.cuda.synchronize(self.device)
        finally:
            self.check()

    def read(self, name: str) -> np.ndarray:
        """Copy an internal buffer (routing tables, staging areas) to host -- tests and debugging only."""
        which, dt = _BUFFER_SPECS[name]
        nbytes = ctypes.c_size_t()
        _lib.check(self._L.fm_buffer_bytes(self._ctx, which, ctypes.byref(nbytes)))
        arr = np.empty(nbytes.value // np.dtype(dt).itemsize, dtype=dt)
        _lib.check(self._L.fm_read_buffer(self._ctx, which, arr.ctypes.data_as(ctypes.c_void_p), nbytes.value))
        d = self.dims
        k, E, S, H, P = d["k"], d["E"], d["S"], d["H"], d["P"]
        npk = d["world"] * d["num_local_experts"]
        shapes = {"topk_idx": (S, k), "topk_w": (S, k), "mcw": (S,), "slot": (S, k), "counts": (E,),
                  "recv_x": (npk, d["pEC"], H), "hidden": (npk, d["pEC"], P), "ret_y": (E, d["pEC"], H),
                  "gate_out": (S, E), "recv_cnt": (npk,), "trace": (d["grid"], trace_slots.SLOTS), "aux_loss": (2 * E + 1,),
                  "shared_y": (S, H), "shared_hidden": (S, arr.size // S)}   # (Ps of the last shared launch)
        return arr.reshape(shapes[name])

    @property
    def launch_count(self) -> int:
        """Launches issued through this API (graph replays are not counted; see `launch_record`)."""
        return int(self._L.fm_launch_count(self._ctx))

    def close(self) -> None:
        if self._ctx:
            self._L.fm_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
