"""Golden vectors for the fused q/k RMSNorm + rotary embedding (``tests/golden/qk_norm_rope.pt``), made on the CPU by the
REFERENCE'S OWN modules (imported through ``ref_shim``): ``RMSNorm`` (module/rms_norm/rms_norm.py, ``F.rms_norm``),
``apply_rotary_pos_emb_cuda`` (ops/rotary_emb.py) and ``RotaryEmbedding`` (module/rope/rope.py, rope_theta = 1e6):

    python tests/golden/make_qk_norm_rope_golden.py

The steps are those of ``MultiHeadAttention.forward`` (module/attention/mha.py:335-363): the projections viewed as
[1, T, H, D] (q optionally as the first half of the ``with_gate`` chunk, head stride 2D), q_norm / k_norm, the transpose
to [1, H, T, D] and the rotary embedding, over T = 8 packed tokens of three documents whose position ids restart at 0.
Then autograd of sum(out * g) for a random bf16 g.  Stored per case, all as [T, H, D] (the transposes undone): the inputs,
the outputs, the gradient at the norm outputs (``gn``, from ``retain_grad``), the input gradients and the norm weight
gradients.  Cases: Hq = 8, Hkv = 2 at D = 128 and D = 64 with fp32 norm weights, D = 128 with bf16 norm weights, a
``with_gate`` q, and ``qk_norm=False``.
"""
from __future__ import annotations

import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402

ref_shim.apply_cpu_patches()

from make_golden import save  # noqa: E402
from xtuner.v1.module.rms_norm import RMSNorm  # noqa: E402
from xtuner.v1.module.rope.rope import RotaryEmbedding  # noqa: E402
from xtuner.v1.ops.rotary_emb import apply_rotary_pos_emb_cuda  # noqa: E402

T, HQ, HKV, EPS = 8, 8, 2, 1e-6
DOCS = [3, 4, 1]  # packed documents: position ids restart at each
CASES = {  # name: (D, norm weight dtype or None, with_gate)
    "d128": (128, torch.float32, False),
    "d64": (64, torch.float32, False),
    "d128_bf16w": (128, torch.bfloat16, False),
    "d128_gate": (128, torch.float32, True),
    "d128_nonorm": (128, None, False),
}


def cos_sin(D: int):
    cfg = types.SimpleNamespace(max_position_embeddings=4096, rope_parameters_cfg=None, rope_scaling_cfg=None,
                                rope_theta=1e6, head_dim=D, hidden_size=D * HQ, num_attention_heads=HQ)
    pos = torch.cat([torch.arange(n) for n in DOCS]).view(1, T)
    cos, sin = RotaryEmbedding(cfg).forward(torch.zeros(1, dtype=torch.bfloat16), pos)
    return cos, sin  # [1, T, D] bf16


def run_case(seed: int, D: int, wdtype, with_gate: bool) -> dict:
    g = torch.Generator().manual_seed(seed)
    q_cols = 2 * D if with_gate else D
    q_in = (torch.randn(1, T, HQ, q_cols, generator=g) * 3).to(torch.bfloat16).requires_grad_(True)
    k_in = (torch.randn(1, T, HKV, D, generator=g) * 0.5).to(torch.bfloat16).requires_grad_(True)
    cos, sin = cos_sin(D)
    q = torch.chunk(q_in, 2, dim=-1)[0] if with_gate else q_in
    k = k_in
    out = {}
    if wdtype is not None:
        q_norm, k_norm = RMSNorm(D, eps=EPS), RMSNorm(D, eps=EPS)
        with torch.no_grad():
            q_norm.weight.copy_(1.0 + 0.5 * torch.randn(D, generator=g))
            k_norm.weight.copy_(1.0 + 0.5 * torch.randn(D, generator=g))
        q_norm.to(wdtype), k_norm.to(wdtype)
        q, k = q_norm(q), k_norm(k)
        q.retain_grad(), k.retain_grad()
        nq, nk = q, k
        out["w_q"], out["w_k"] = q_norm.weight.detach(), k_norm.weight.detach()
    oq, ok = apply_rotary_pos_emb_cuda(q.transpose(1, 2), k.transpose(1, 2), cos, sin)
    gq = torch.randn(oq.shape, generator=g).to(torch.bfloat16)
    gk = torch.randn(ok.shape, generator=g).to(torch.bfloat16)
    ((oq.float() * gq.float()).sum() + (ok.float() * gk.float()).sum()).backward()
    out.update({
        "q": q_in.detach()[0], "k": k_in.detach()[0], "cos": cos[0], "sin": sin[0],
        "out_q": oq.detach()[0].transpose(0, 1).contiguous(), "out_k": ok.detach()[0].transpose(0, 1).contiguous(),
        "g_q": gq[0].transpose(0, 1).contiguous(), "g_k": gk[0].transpose(0, 1).contiguous(),
        "dx_q": q_in.grad[0], "dx_k": k_in.grad[0],
    })
    if wdtype is not None:
        out["gn_q"], out["gn_k"] = nq.grad[0], nk.grad[0]
        out["dw_q"], out["dw_k"] = q_norm.weight.grad.detach(), k_norm.weight.grad.detach()
    return out


def main():
    out = {"eps": EPS, "docs": torch.tensor(DOCS)}
    for i, (name, (D, wdtype, gate)) in enumerate(CASES.items()):
        for key, v in run_case(1000 + i, D, wdtype, gate).items():
            out[f"{name}.{key}"] = v
    save("qk_norm_rope", out)


if __name__ == "__main__":
    main()
