"""Exact restatements, float64 references, checkers and input generators for the SwiGLU kernels (``xtb_swiglu``,
``xtb_swiglu_bwd``, ``csrc/permute.cu``) and the fp8 quantisation kernels (``xtb_fp8_per_tile_quant``,
``xtb_fp8_block_scales``, ``xtb_fp8_block_cast``, ``csrc/fp8.cu``).  Test infrastructure only; nothing under
``xtuner_b200/`` imports it.  Plain torch on whatever device the operands are on.

SwiGLU forward, ``a = bf16(s u)`` with ``s = bf16(silu(g))``.  The product of two bf16 values is exact in fp32, so ``a``
is fixed once ``s`` is: the only inexact step is the kernel's fp32 silu (``common.cuh``, ``sigmoid_fast``):

  E = __expf(-x), D = fl(1 + E), sigma = __frcp_rn(D), v = fl(x sigma)

From x = -88.72 (ln of the fp32 maximum) down, E and D are inf and sigma is exactly 0, so v = -0: the value the
reference's own fp32 silu (x / (1 + exp(-x)) under torch) gives there too, although x e^x is a normal float down to
x = -92.  The references below model that band as the kernel and the reference compute it (sigma = 0, no error); the
exhaustive sweep pins it bit for bit.  An e^x branch below -88 would give the float64 value, at a measured cost in the
grouped GEMM's SwiGLU epilogue, which shares sigmoid_fast.

Error model: every fp32 rounding is fl(y) = y (1 + d) + n with |d| <= u = 2^-24 and |n| <= 2^-150 (the subnormal
range; the build does not flush).  ``__expf`` is within n_e = 2 + floor(1.173 |x|) ulp (CUDA's documented bound), and
one ulp of a float y is at most max(2^-23 |y|, 2^-149), so |E - e| <= n_e 2^-23 e + 2^-126 (where e^-x is below 2^-126
a flushed or subnormal E is off by at most 2^-126, which only ever meets the add to 1):

  e = e^-x:  |D - (1 + e)| <= n_e 2^-23 e + 2^-126 + u (1 + E), so D is off by
             rel_D = (n_e 2^-23 e + 2^-126) / (1 + e) + u relative; 1 / D is then off by rel_D / (1 - rel_D), and the
             correctly rounded reciprocal (subnormal from x = -87.3 down) adds u relative and 2^-150 absolute:
             |sigma - s(x)| <= 1.01 (rel_D + u) s(x) + 2^-150.
  silu:      |v - x s(x)| <= |x| err_sigma + u |x| (s(x) + err_sigma) + 2^-150, taken 1.01 times (:func:`silu_ref`).

Where the float64 silu lies farther than that bound from the midpoint between its two bf16 neighbours, ``s`` is the
correctly rounded value and ``a`` must match bit for bit; inside the window ``s`` may be either neighbour
(:func:`s_candidates`), and the checks count those cases.

SwiGLU backward, with the rounding points of ``swiglu_bwd_vec``:

  ds     = bf16(d u)                      exact restatement (one rounding of an exact fp32 product)
  grad_u = bf16(d s)                      exact, given s as above
  grad_g = bf16((ds sigma) (1 + x (1 - sigma)))
           p = fl(ds sigma); t = fl(1 - sigma); q = 1 + x t, one fma or a product and an add.  With F = 1 + x (1 - s(x)):
           |q - F| <= |x| err_sigma (1 + 3u) + 3u (1 + |x| (1 - s(x)) + |x| err_sigma)   -- absolute: F crosses zero
           at x = -1.2785, where a relative bound would be 0;
           |p - ds s(x)| <= |ds| (err_sigma + u (s(x) + err_sigma)) + 2^-150;
           |fl(p q) - ds s(x) F| <= (e_p (|F| + e_q) + |ds| s(x) e_q)(1 + u) + u |ds s(x) F| + 2^-150, taken 1.01 times
           (:func:`grad_g_ref`), and checked with ``check_near_tie``.

fp8: scale = fp32(max(amax, 1e-12) / 448) in float64, q = e4m3(fp32(x) / scale) with a saturating round to nearest
even (:func:`e4m3_bits`, a float64 model of the cast checked against torch's).  amax follows torch: a NaN anywhere in a
1x128 tile or 128x128 block makes the scale NaN, an inf makes it inf; then x / scale is NaN for every element
(NaN scale) or for the inf element (inf / inf), 0 for the finite ones, and NaN stays NaN through the cast.
"""
from __future__ import annotations

import math
from typing import Tuple

import torch

from tests.norm_combine_reference import U32, assert_bits_equal, check_bound, check_near_tie  # noqa: F401

F32_TINY = 2.0 ** -150  # largest absolute error of one fp32 rounding into the subnormal range
SIG_OVERFLOW = -math.log(3.4028234663852886e38)  # below this 1 + e^-x is inf in fp32 and sigmoid_fast is 0
BF16_MAX = (2 - 2.0 ** -7) * 2.0 ** 127
BF16_OVERFLOW = 2.0 ** 128 - 2.0 ** 119  # |x| at or above this rounds to inf
E4M3_MAX = 448.0
FP8_EPS = 1e-12
SW_ROWS = 8  # kSwRows of the backward's row split
SW_I8_MAX = 23170  # the largest I / 8 with kSwRows * I8^2 < 2^32

# the u values the exhaustive sweep pairs with every bf16 g
SWEEP_U = (1.0, -1.0, 3.0, 2.0 ** -100, BF16_MAX, 0.0, float("nan"))


# ---- bf16 helpers ----------------------------------------------------------------------------------------------------


def all_bf16() -> torch.Tensor:
    """The 65,536 bf16 bit patterns in order, ±0, subnormals, ±inf and NaNs included."""
    return torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)


def bf16_round(x: torch.Tensor) -> torch.Tensor:
    """float64 -> bf16 with one round to nearest even (a direct ``.to(bfloat16)`` may round through fp32 first)."""
    _, e = torch.frexp(x)
    q = torch.pow(2.0, (e - 8).clamp_min(-133).to(x.dtype))
    r = torch.where(torch.isfinite(x), torch.round(x / q) * q, x)
    return r.to(torch.bfloat16)  # r is a bf16 value (or 2^128, which overflows to inf as it should)


def bf16_neighbour(r: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """The bf16 neighbour of bf16 ``r`` on the side of float64 ``x`` (``r`` itself where x == r)."""
    bits = r.view(torch.int16).to(torch.int32) & 0xFFFF
    mag, neg = bits & 0x7FFF, bits >= 0x8000
    rd = r.double()
    away = x.abs() > rd.abs()
    zero = mag == 0
    new_mag = torch.where(zero, torch.ones_like(mag), torch.where(away, mag + 1, mag - 1))
    new_neg = torch.where(zero, x < 0, neg)
    out = (new_mag | (new_neg.to(torch.int32) << 15)).to(torch.int16).view(torch.bfloat16)
    return torch.where(x == rd, r, out)


def assert_bits_equal_nan(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """``assert_bits_equal`` with NaN compared as NaN-ness (payload and sign of a NaN are not pinned)."""
    gn, wn = torch.isnan(got), torch.isnan(want)
    if bool((gn != wn).any()):
        i = tuple(int(v) for v in (gn != wn).nonzero()[0])
        raise AssertionError(f"{what}: NaN positions differ ({int((gn != wn).sum())} elements); first at {i}: "
                             f"got {got[i].item()!r}, want {want[i].item()!r}")
    z = torch.zeros((), dtype=got.dtype, device=got.device)
    assert_bits_equal(torch.where(gn, z, got), torch.where(wn, z, want), what)


# ---- SwiGLU: float64 references --------------------------------------------------------------------------------------


def _expf_ulps(x: torch.Tensor) -> torch.Tensor:
    return 2 + torch.floor(1.173 * x.abs())


def sigmoid_ref(g: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(sigmoid, bound)`` in float64: the logistic function of bf16 ``g`` (0 where 1 + e^-g overflows fp32, as the
    kernel and the reference compute it) and how far ``sigmoid_fast`` may be from it (module docstring).  The bound is
    0 where g is not finite or in the overflow band."""
    x = g.double()
    ov = x < SIG_OVERFLOW
    sig = torch.where(ov, torch.zeros_like(x), torch.special.expit(x))
    e = torch.exp(-x)
    rel_d = (_expf_ulps(x) * 2.0 ** -23 * e + 2.0 ** -126) / (1 + e) + U32
    err = 1.01 * (rel_d + U32) * sig + F32_TINY
    return sig, torch.where(torch.isfinite(x) & ~ov, err, torch.zeros_like(err))


def silu_ref(g: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(silu, bound)`` in float64: g sigmoid(g) and the bound on the kernel's fp32 silu before the bf16 round."""
    x = g.double()
    sig, es = sigmoid_ref(g)
    b = 1.01 * (x.abs() * es + U32 * x.abs() * (sig + es) + F32_TINY)
    return x * sig, torch.where(torch.isfinite(x), b, torch.zeros_like(b))


def s_candidates(g: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``(s, s_alt, tie)``: the correctly rounded bf16 silu of ``g``, its bf16 neighbour on the other side of the
    float64 value, and where the float64 value lies within the kernel's bound of the midpoint between the two (there
    the kernel's ``s`` may be either)."""
    ref, bound = silu_ref(g)
    s = bf16_round(ref)
    alt = bf16_neighbour(s, ref)
    mid = (s.double() + alt.double()) / 2
    tie = torch.isfinite(ref) & (alt.view(torch.int16) != s.view(torch.int16)) & ((ref - mid).abs() <= bound)
    return s, alt, tie


def grad_g_ref(g: torch.Tensor, ds: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(grad_g, bound)`` in float64 from bf16 ``g`` and the restated bf16 ``ds`` (module docstring)."""
    x, dsd = g.double(), ds.double()
    sig, es = sigmoid_ref(g)
    F = 1 + x * (1 - sig)
    eq = x.abs() * es * (1 + 3 * U32) + 3 * U32 * (1 + x.abs() * (1 - sig) + x.abs() * es)
    P = dsd * sig
    ep = dsd.abs() * (es + U32 * (sig + es)) + F32_TINY
    ref = P * F
    b = 1.01 * ((ep * (F.abs() + eq) + P.abs() * eq) * (1 + U32) + U32 * ref.abs() + F32_TINY)
    return ref, torch.where(torch.isfinite(b), b, torch.zeros_like(b))


# ---- SwiGLU: exact restatements given s ------------------------------------------------------------------------------


def _mul_bf16(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """bf16(a b) of two bf16 tensors through fp32, as the kernels round."""
    return (a.float() * b.float()).to(torch.bfloat16)


def swiglu_a(s: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    return _mul_bf16(s, u)


# ---- SwiGLU: checks --------------------------------------------------------------------------------------------------


def _pick(got: torch.Tensor, want: torch.Tensor, alt: torch.Tensor, tie: torch.Tensor) -> torch.Tensor:
    """``want``, replaced by ``alt`` at the near ties where ``got`` took it."""
    took_alt = tie & (got.view(torch.int16) == alt.view(torch.int16))
    return torch.where(took_alt, alt, want)


def check_swiglu_fwd(h: torch.Tensor, a: torch.Tensor, what: str = "swiglu") -> int:
    """``a`` of ``xtb_swiglu`` on ``h [M, 2I]``: bit-exact where ``s`` is fixed, one of the two candidates at the near
    ties of ``s``.  Returns the number of near ties."""
    I = h.shape[1] // 2
    g, u = h[:, :I], h[:, I:]
    s, alt, tie = s_candidates(g)
    want = _pick(a, swiglu_a(s, u), swiglu_a(alt, u), tie)
    assert_bits_equal_nan(a, want, what)
    return int(tie.sum())


def check_bf16_near_tie(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = ""
                        ) -> Tuple[float, int]:
    """``check_near_tie`` extended to the non-finite values: NaN where the float64 value is NaN, inf only where the
    float64 value rounds to that inf or lies within the bound of the overflow threshold."""
    gn, rn = torch.isnan(got), torch.isnan(ref)
    if bool((gn != rn).any()):
        i = tuple(int(v) for v in (gn != rn).nonzero()[0])
        raise AssertionError(f"{what}: NaN positions differ ({int((gn != rn).sum())} elements); first at {i}: "
                             f"got {got[i].item()!r}, fp64 {ref[i].item()!r}")
    gi = torch.isinf(got)
    ok_inf = (ref.abs() + bound >= BF16_OVERFLOW) & (torch.sign(ref) == torch.sign(got.double()))
    if bool((gi & ~ok_inf).any()):
        i = tuple(int(v) for v in (gi & ~ok_inf).nonzero()[0])
        raise AssertionError(f"{what}: got inf at {i} where the fp64 value is {ref[i].item()!r}")
    fin = ~gn & ~gi
    if bool((fin & torch.isinf(ref)).any()):
        i = tuple(int(v) for v in (fin & torch.isinf(ref)).nonzero()[0])
        raise AssertionError(f"{what}: got {got[i].item()!r} at {i} where the fp64 value is {ref[i].item()!r}")
    return check_near_tie(got[fin], ref[fin], bound[fin], what)


def check_swiglu_bwd(h: torch.Tensor, d: torch.Tensor, grad_h: torch.Tensor, what: str = "swiglu_bwd"
                     ) -> Tuple[int, float, int]:
    """``grad_h`` of ``xtb_swiglu_bwd``: grad_u bit-exact given ``s`` (either candidate at a near tie of ``s``),
    grad_g within the float64 bound.  Returns ``(near ties of s, largest |err| / bound of grad_g, near ties of
    grad_g)``."""
    I = h.shape[1] // 2
    g, u = h[:, :I], h[:, I:]
    gg, gu = grad_h[:, :I], grad_h[:, I:]
    s, alt, tie = s_candidates(g)
    want = _pick(gu, _mul_bf16(d, s), _mul_bf16(d, alt), tie)
    assert_bits_equal_nan(gu, want, f"{what} grad_u")
    ds = _mul_bf16(d, u)
    ref, bound = grad_g_ref(g, ds)
    ratio, ties_g = check_bf16_near_tie(gg, ref, bound, f"{what} grad_g")
    return int(tie.sum()), ratio, ties_g


# ---- SwiGLU: the backward's row split --------------------------------------------------------------------------------


def row_split_inverse(I8: int) -> int:
    """``inv_I8`` of ``xtb_swiglu_bwd``: ceil(2^32 / I8)."""
    return ((1 << 32) + I8 - 1) // I8


def umulhi(i, inv: int):
    """``__umulhi(i, inv)`` for numpy uint64 arrays (or ints) with i, inv < 2^32."""
    return (i * inv) >> 32


# ---- fp8 -------------------------------------------------------------------------------------------------------------


def e4m3_bits(v: torch.Tensor) -> torch.Tensor:
    """uint8 e4m3fn of float64 ``v`` (an fp32 value) with a saturating round to nearest even: the normal quantum is
    2^(e - 4) for 2^(e-1) <= |v| < 2^e, the subnormal one 2^-9; |v| past 448 (inf included) saturates, NaN gives
    0x7F with the sign bit of v."""
    a = v.abs()
    _, e = torch.frexp(a)
    q = torch.pow(2.0, (e - 4).clamp_min(-9).to(torch.float64))
    r = torch.where(torch.isfinite(a), torch.round(a / q) * q, a).clamp(max=E4M3_MAX)
    r = torch.where(torch.isnan(v), torch.zeros_like(r), r)
    _, er = torch.frexp(r)
    sub = r < 2.0 ** -6
    exp_field = torch.where(sub, torch.zeros_like(er), er - 1 + 7)
    mant = torch.where(sub, r / 2.0 ** -9, (r / torch.pow(2.0, (er - 1).to(torch.float64)) - 1) * 8)
    bits = (exp_field.to(torch.int32) << 3) | mant.round().to(torch.int32)
    bits = torch.where(torch.isnan(v), torch.full_like(bits, 0x7F), bits)
    bits = bits | (torch.signbit(v).to(torch.int32) << 7)
    return bits.to(torch.uint8)


def fp8_scale(amax: torch.Tensor) -> torch.Tensor:
    """fp32 scale from a float64 amax: max(amax, 1e-12) / 448 in float64 (NaN stays NaN)."""
    a = amax.double()
    return torch.where(a < FP8_EPS, torch.full_like(a, FP8_EPS), a).div(E4M3_MAX).float()


def tile_quant(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(q uint8 [M, K], scales fp32 [M, K/128])`` of ``xtb_fp8_per_tile_quant`` on bf16 ``x``."""
    M, K = x.shape
    t = x.float().view(M, K // 128, 128)
    s = fp8_scale(t.double().abs().amax(-1))
    return e4m3_bits((t / s[..., None]).double()).view(M, K), s


def block_scales(w: torch.Tensor) -> torch.Tensor:
    """fp32 [nw, dout/128, din/128] of ``xtb_fp8_block_scales`` on fp32 / bf16 ``w [nw, dout, din]``."""
    nw, dout, din = w.shape
    b = w.float().view(nw, dout // 128, 128, din // 128, 128).transpose(2, 3)
    return fp8_scale(b.double().abs().amax((-1, -2)))


def block_cast(w2d: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """uint8 [dout, din] of ``xtb_fp8_block_cast`` on one matrix and its [dout/128, din/128] scales."""
    dout, din = w2d.shape
    s = scales.float().reshape(dout // 128, 1, din // 128, 1).expand(-1, 128, -1, 128).reshape(dout, din)
    return e4m3_bits((w2d.float() / s).double())


def assert_fp8_equal(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """e4m3 bytes equal as uint8, NaN bytes (0x7F / 0xFF) compared as NaN-ness: the sign of a NaN is not pinned."""
    g, w = got.view(torch.uint8).int(), want.view(torch.uint8).int()
    gn, wn = (g & 0x7F) == 0x7F, (w & 0x7F) == 0x7F
    bad = (gn != wn) | (~gn & (g != w))
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} bytes differ; first at {i}: "
                             f"got 0x{int(g[i]):02x}, want 0x{int(w[i]):02x}")


def assert_scales_equal(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """fp32 scales equal (``torch.equal``) with NaN matched as NaN."""
    gn, wn = torch.isnan(got), torch.isnan(want)
    assert torch.equal(gn, wn), f"{what}: NaN scales at different positions"
    assert torch.equal(torch.where(gn, 0.0, got), torch.where(wn, 0.0, want)), f"{what}: scales differ"


def cast_sweep_values() -> torch.Tensor:
    """Every bf16 value in [-448, 448] (±0, subnormals, e4m3 ties and values below half the smallest e4m3 subnormal
    included), in bit-pattern order."""
    v = all_bf16()
    f = v.float()
    return v[torch.isfinite(f) & (f.abs() <= E4M3_MAX)]


def amax_one_tiles(vals: torch.Tensor, width: int = 128) -> torch.Tensor:
    """[n, width] rows whose element 0 is 448 and whose other elements are ``vals`` in order (padded with 448): every
    row's amax is exactly 448, its scale exactly 1, so the quotient is the value itself."""
    per = width - 1
    n = -(-vals.numel() // per)
    body = torch.full((n * per,), E4M3_MAX, dtype=vals.dtype)
    body[: vals.numel()] = vals
    return torch.cat([torch.full((n, 1), E4M3_MAX, dtype=vals.dtype), body.view(n, per)], 1)
