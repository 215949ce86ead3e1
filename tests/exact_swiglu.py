"""The exact-input reference (tests/exact.py) for SwiGLU experts (hidden_act = 2): h's interval and the inputs.

An expert's weights are [3, P, H]: W_gate, W_up and the P*H block flat-viewed as W_down [H, P].  The kernel computes
g = fl(x W_gate^T + b_g), u = fl(x W_up^T + b_u) (both exact here: the inputs keep every partial sum exact in fp32) and
h = rne_bf16(fl(fl(g * sigma(g)) * u)) with sigma(g) = rcp_rn(fl(1 + ex2.approx.ftz(fl(-g * fl32(log2 e))))).

Error bound of h against the real g * sigmoid(g) * u, relative, first order (eps_swiglu):
  fl32(log2 e) is log2 e (1 + d0), |d0| < 2^-26, and the product rounds once (2^-24): the exponent a = -g log2 e is off
  by at most |a| (2^-24 + 2^-26), which moves 2^a by ln 2 * |a| * 1.25 * 2^-24 = 1.25 * |g| * 2^-24 relative;
  ex2.approx.ftz: 2^-21 (exact.EPS_EX2); 1 + e rounds once (2^-24) and does not amplify e's relative error (e >= 0);
  the reciprocal rounds once (2^-24); g * sigma and the product with u round once each (2 * 2^-24).
  Total 2^-21 + 2^-24 * (1.25 |g| + 4); one more 2^-24 covers the second-order terms: eps = 2^-21 + 2^-24 (1.25|g| + 5).
The final fp32 -> bf16 RNE is monotone, so h lies in [rne(v (1 - eps)), rne(v (1 + eps))] for the real v.  That holds
while sigma is a normal fp32 number: the power argument a = fl(-g log2e) <= 125 (g >= -86.6).  For large positive g
the power flushes to +0 and sigma is exactly 1, inside the bound.  Below that the relative bound is false:
  - a in (126, 128), g in about [-88.7, -87.4]: 1 + 2^a > 2^126 and the correctly rounded reciprocal is subnormal,
    kept as such (no -ftz), with an absolute 2^-150 error;
  - a >= 128, g below about -88.72: ex2.approx returns +inf, sigma is +0 and h is exactly +-0, although the real
    g sigmoid(g) u still rounds to a nonzero bf16 down to g = -99 or so (-7.4e-38 at g = -90, u = 1).
There (a > 125) the interval follows the kernel's steps from the two ends of ex2's result (silu_mul_f32_ends).
swiglu_weights keeps g in [-4, 4]; tests/exact_tails.py reaches g in [-136, 136].

GEMM1 is exact given the device's own h (exact.gemm1_reference): the generator keeps |h| in [2^-4, 2^6] and W_down
sparse, so y's sums stay on one fp32 grid.  No pytest in here.
"""
from __future__ import annotations

import numpy as np
import torch

from flashmoe_b200.config import MoEConfig
from tests import exact as ex

G_MIN = -64.0   # the generator keeps every gate pre-activation at or above this


def eps_swiglu(g: np.ndarray) -> np.ndarray:
    """Relative error bound of the kernel's h = silu(g) * u (module docstring)."""
    return 2.0 ** -21 + 2.0 ** -24 * (1.25 * np.abs(g) + 5.0)


def silu_mul_rounded(g: np.ndarray, u: np.ndarray) -> ex.Rounded:
    """The interval of the kernel's bf16 h = silu_mul(g, u) for exact fp32 pre-activations g, u (float64 arrays):
    relative eps_swiglu where sigma(g) is a normal number (power argument a = fl(-g log2e) <= ex.NORMAL_A), and
    beyond it the kernel's steps from ex2's ends (silu_mul_f32_ends): the subnormal sigma band and the +-0 past the
    overflow cliff (a >= 128).  `exact` is the real g sigmoid(g) u."""
    g, u = np.broadcast_arrays(np.asarray(g, np.float64), np.asarray(u, np.float64))
    with np.errstate(over="ignore"):
        v = g / (1.0 + np.exp(-g)) * u
    e = eps_swiglu(g)
    a, b = ex.f64_to_bf16(v * (1 - e)), ex.f64_to_bf16(v * (1 + e))
    tail = power_arg(g) > ex.NORMAL_A
    if tail.any():
        lo, hi = silu_mul_f32_ends(g[tail], u[tail])
        a[tail], b[tail] = ex.f32_to_bf16(lo), ex.f32_to_bf16(hi)
    swap = ex.order_key(a) > ex.order_key(b)
    return ex.Rounded(np.where(swap, b, a), np.where(swap, a, b), v)


def power_arg(g: np.ndarray) -> np.ndarray:
    """a = fl(-g * fl32(log2 e)), the argument of the kernel's ex2 (exact: a product of two fp32 numbers)."""
    return (-np.asarray(g, np.float64) * float(ex.LOG2E_F32)).astype(np.float32).astype(np.float64)


def silu_mul_f32_ends(g: np.ndarray, u: np.ndarray):
    """Bounds (float32, unordered) of the kernel's fp32 h = fl(fl(g * sigma) * u), sigma = sigmoid_score(g) between
    exact.sigmoid_f32_ends' ends: both products are monotone in sigma, so its two ends give h's.  At a >= 128 sigma
    is +0 and h = +-0; for a in (126, 128) sigma is subnormal, still kept by __frcp_rn."""
    s_lo, s_hi = ex.sigmoid_f32_ends(power_arg(g))
    g32, u32 = np.asarray(g, np.float32), np.asarray(u, np.float32)
    return (((g32 * s_lo).astype(np.float32) * u32).astype(np.float32),
            ((g32 * s_hi).astype(np.float32) * u32).astype(np.float32))


# ----------------------------------------------------------------------------- inputs
def _bf(a: np.ndarray) -> torch.Tensor:
    t = torch.from_numpy(np.ascontiguousarray(a)).bfloat16()
    assert np.array_equal(t.double().numpy(), a), "generator produced a value that is not a bf16 number"
    return t


def swiglu_weights(E: int, P: int, H: int, rng: np.random.Generator, bias: bool, gate_nz: int = 3, up_nz: int = 2,
                   down_nz: int = 8):
    """(we [E, 3, P, H], bu [E, 2, P] or None, bd [E, H] or None) as float64 arrays for x in {-1, 0, 1}: W_gate rows
    with gate_nz entries in {-1, -1/2, 1/2, 1}, b_g in {-1, ..., 1} on 1/2 (so g in [-4, 4] on a grid of 1/2:
    silu(g) is 0 or at least 0.07 in magnitude); W_up rows with up_nz integers in [-4, 4], b_u integers in [-2, 2]
    (u an integer, |u| <= 4 up_nz + 2); W_down on 2^-5 with about down_nz nonzeros per output column."""
    def sparse_rows(nz, vals):
        w = np.zeros((E, P, H))
        for e in range(E):
            for p in range(P):
                cols = rng.choice(H, size=nz, replace=False)
                w[e, p, cols] = rng.choice(vals, size=nz)
        return w

    gate = sparse_rows(gate_nz, np.array([-1.0, -0.5, 0.5, 1.0]))
    up = sparse_rows(up_nz, np.array([v for v in range(-4, 5) if v]).astype(np.float64))
    down = (rng.integers(-4, 5, size=(E, H, P)) * (rng.random((E, H, P)) < down_nz / P)) * 2.0 ** ex.WDOWN_GRID
    we = np.stack([gate, up, down.reshape(E, -1).reshape(E, P, H)], axis=1)
    bu = bd = None
    if bias:
        bu = np.stack([rng.integers(-2, 3, size=(E, P)) * 0.5, rng.integers(-2, 3, size=(E, P)).astype(np.float64)], 1)
        bd = rng.integers(-64, 65, size=(E, H)) * 2.0 ** -8
    return we, bu, bd


def swiglu_inputs(cfg: MoEConfig, seed: int, bias: bool = False, **router_kw) -> ex.ExactInputs:
    """Seeded exact inputs for a hidden_act = 2 context `cfg`: the router's x and gate weights from exact.exact_inputs
    (x in {-1, 0, 1}; `router_kw` goes there), the experts from swiglu_weights."""
    assert cfg.hidden_act == 2
    inp = ex.exact_inputs(cfg, seed, x_range=1, **router_kw)
    inp.experts = swiglu_experts(cfg.E, cfg.P, cfg.H, np.random.default_rng(seed + 1), bias)
    return inp


def swiglu_experts(E: int, P: int, H: int, rng: np.random.Generator, bias: bool) -> ex.Experts:
    we, bu, bd = swiglu_weights(E, P, H, rng, bias)
    return ex.Experts(_bf(we), None if bu is None else _bf(bu), None if bd is None else _bf(bd), 2)


def shared_swiglu(H: int, Ps: int, seed: int, bias: bool = False) -> ex.Experts:
    """A seeded SwiGLU shared expert (E = 1)."""
    return swiglu_experts(1, Ps, H, np.random.default_rng(seed), bias)
