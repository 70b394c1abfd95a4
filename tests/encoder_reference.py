"""The ViT encoder of PARSeq and ViTSTR as an fp64 rounding-point model.  TEST HELPER.

`EncoderReference` rounds to bf16 at exactly the encoder's rounding points (DESIGN.md section 5): image patches and GEMM
weights (round-to-nearest-even, as `im2col_patch_kernel` and the weight conversion at load do), LayerNorm outputs,
QKV, the un-normalised softmax numerators P (the row sum is taken from the unrounded P, as `enc_attention_kernel`
does), the attention output and GELU(fc1), with the engine's polynomial erf-GELU (`engine_gelu`, the function of the
encoder GEMM's GELU epilogue and of `mlp_ln.cuh`).  Everything else, the fp32 residual stream included, is computed in
`accum` (fp64 by default).  `encode` gives what the engine's `encode` / `forward_features` returns (the final
LayerNorm in full precision); `tail` gives ViTSTR's logits, head(bf16(norm(x[:, 1 + j]))) for j < L, as `vitstr_tail`
computes them.  The model runs on the device its inputs are on.

`accum=torch.float32` is a CPU stand-in for the engine: the same rounding points with fp32 arithmetic.  Its distance
from the fp64 model is the noise a correct encoder shows.  `gelu="exact"` with fp32 accumulation is the oracle's
bf16 mode (`ParseqOracle(cfg, sd, "bf16").encode`), and `rounding=False` on top of that is its fp32 mode;
tests/test_encoder_budget_cpu.py pins both.

`bug=` injects one wrong detail (BUGS).  tests/test_encoder_budget_cpu.py shows each of them outside BOUNDS where it
can show and the fp32 stand-in inside, so the bounds that tests/test_gpu_encoder_isolated.py holds the engine to are
the ones that separate a correct encoder from these mistakes.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple, Union

import torch
import torch.nn.functional as F

from decoder_reference import engine_gelu

# Each entry changes exactly one thing in the model.
BUGS = {
    "patch_round_trunc": "image patches are rounded to bf16 by truncation",
    "weight_round_trunc": "the GEMM weights are rounded to bf16 by truncation at load",
    "patch_dx_dy_swap": "im2col walks a patch column by column (k = ch ph pw + dx ph + dy)",
    "pos_embed_shift": "patch token t gets pos_embed of token t + 1 (the last one wraps to the first)",
    "ln_eps": "the encoder LayerNorms use eps 1e-5 instead of 1e-6",
    "attn_drop_last_key": "the attention drops the last key",
    "attn_extra_zero_key": "the attention sees one extra key whose K and V are zero (a padding key not masked)",
    "attn_p_normalised_before_rounding": "P is divided by the row sum before it is rounded to bf16",
    "gelu_tanh": "the MLP uses the tanh approximation of GELU",
    "no_v_bias": "the V third of the qkv bias is dropped",
    "next_norm_from_own_block": "block i + 1's norm1 uses block i's norm1 parameters (the fused fc2 epilogue's tables)",
    "vitstr_cls_without_pos": "ViTSTR's class-token row is cls_token without pos_embed[0]",
    "vitstr_row_shift": "ViTSTR's head reads token j instead of 1 + j",
}

# Bounds on |engine - model| over the encoder output (PARSeq's memory, ViTSTR's forward_features) relative to the
# standard deviation sigma of the model's output, per (embed_dim, enc_depth); ("vitstr", 2) is ViTSTR-S's features at
# depth 2 and ("vitstr-tail", 2) its tail logits.  The median, the mean and the 99th percentile of |d| / sigma.
# A correct encoder's error is bf16 rounding flips: an fp32 sum on the other side of a rounding boundary than the fp64
# one.  Within one block they are sparse and most outputs see none (depth 1: medians 1e-7 to 1e-6 at D <= 384), so a
# wrong detail that moves every output a little (an eps, an extra key, the tanh GELU) stands out on the median by 10x or
# more.  The attention spreads every flip of block 0 over all the tokens of the image, so from depth 2 on every output
# carries some and the median of a correct encoder (6e-4 to 2.4e-3) is as large as those small bugs: at depth 2 the
# bounds catch the wrong wiring (positions, patches, norms, biases, keys) and the truncating roundings, and depth 1 the
# small bugs.  D = 768 (T = 240) flips more often already at depth 1.
# tests/test_encoder_budget_cpu.py is the reason for every number here: the fp32 stand-in stays within half of each
# bound, and every bug in BUGS exceeds one of them by 2x or more where it can show, save the exceptions it names with
# their numbers.  The engine's own figures (DESIGN.md section 5; H100 SXM, 700 W) stay below each bound by 1.3x or more.
BOUNDS: Dict[Tuple[Union[int, str], int], Dict[str, float]] = {
    (192, 1): {"p50": 1.0e-5, "mean": 6.0e-5, "p99": 1.0e-3},
    (384, 1): {"p50": 2.0e-5, "mean": 2.0e-4, "p99": 2.5e-3},
    (768, 1): {"p50": 8.0e-4, "mean": 1.1e-3, "p99": 5.3e-3},
    (192, 2): {"p50": 3.6e-4, "mean": 5.0e-4, "p99": 2.4e-3},
    (384, 2): {"p50": 1.3e-3, "mean": 1.65e-3, "p99": 6.2e-3},
    (768, 2): {"p50": 3.5e-3, "mean": 4.3e-3, "p99": 1.65e-2},
    ("vitstr", 2): {"p50": 1.45e-3, "mean": 1.85e-3, "p99": 7.2e-3},
    ("vitstr-tail", 2): {"p50": 2.75e-3, "mean": 3.3e-3, "p99": 1.15e-2},
}


def bug_shows(bug: str, key) -> bool:
    """Whether `bug` can change the output bounded by BOUNDS[key] at all."""
    vit = key[0] in ("vitstr", "vitstr-tail")
    if bug == "vitstr_cls_without_pos":
        return vit
    if bug == "vitstr_row_shift":
        return key[0] == "vitstr-tail"
    if bug == "next_norm_from_own_block":
        return key[1] >= 2
    return True


def sharpen_vitstr(state_dict, s: float):
    """weights._sharpen for ViTSTR's parameter names: the q and k rows of every qkv projection (and their biases) times
    s, i.e. every pre-softmax score times s^2 (peaked attention rows)."""
    sd = dict(state_dict)
    i = 0
    while f"blocks.{i}.attn.qkv.weight" in sd:
        for k in (f"blocks.{i}.attn.qkv.weight", f"blocks.{i}.attn.qkv.bias"):
            t = sd[k].clone()
            t[: 2 * t.shape[0] // 3] *= s
            sd[k] = t
        i += 1
    return sd


def _trunc_bf16(x: torch.Tensor) -> torch.Tensor:
    """fp32(x) rounded to bf16 toward zero, in the dtype of x."""
    f = x.to(torch.float32).contiguous()
    return (f.view(torch.int32) & -65536).view(torch.float32).to(x.dtype)


class EncoderReference:
    def __init__(self, cfg, state_dict, accum=torch.float64, device="cpu", bug: Optional[str] = None,
                 gelu: str = "engine", rounding: bool = True):
        from parseq_b200.weights import gemm_weight_keys
        if bug is not None and bug not in BUGS:
            raise KeyError(bug)
        assert gelu in ("engine", "exact")
        self.cfg, self.bug, self.dt, self.rounding = cfg, bug, accum, rounding
        self.device = torch.device(device)
        self.vit = cfg.arch == "vitstr"
        self.gelu = engine_gelu if gelu == "engine" else F.gelu
        if bug == "gelu_tanh":
            self.gelu = lambda x: F.gelu(x, approximate="tanh")
        # ViTSTR's parameters under the PARSeq encoder's names (as oracle/vitstr_oracle.py presents them)
        name = (lambda k: k if k.startswith("head.") else "encoder." + k) if self.vit else (lambda k: k)
        p = {name(k): v.detach().to(torch.float32) for k, v in state_dict.items()}
        p = {k: v for k, v in p.items() if k.startswith("encoder.") or (self.vit and k.startswith("head."))}
        for k in gemm_weight_keys(cfg):
            k = name(k)
            if k in p and rounding:
                p[k] = _trunc_bf16(p[k]) if bug == "weight_round_trunc" else p[k].to(torch.bfloat16).to(torch.float32)
        if bug == "no_v_bias":
            D = cfg.embed_dim
            for i in range(cfg.enc_depth):
                k = f"encoder.blocks.{i}.attn.qkv.bias"
                p[k] = torch.cat([p[k][: 2 * D], torch.zeros_like(p[k][2 * D:])])
        self.p = {k: v.to(device=self.device, dtype=accum) for k, v in p.items()}

    def r(self, x):
        return x.to(torch.bfloat16).to(x.dtype) if self.rounding else x

    def _ln(self, x, prefix):
        eps = 1e-5 if self.bug == "ln_eps" else 1e-6
        return F.layer_norm(x, (x.shape[-1],), self.p[prefix + ".weight"], self.p[prefix + ".bias"], eps)

    def _patches(self, img):
        """[B, 3, H, W] -> bf16 patches [B, T, 3 ph pw] with k = ch ph pw + dy pw + dx (the Conv2d weight flattened)."""
        B = img.shape[0]
        (ph, pw), (gh, gw) = self.cfg.patch_size, self.cfg.grid
        x = img.to(device=self.device, dtype=torch.float32).reshape(B, 3, gh, ph, gw, pw)
        x = x.permute(0, 2, 4, 1, 5, 3) if self.bug == "patch_dx_dy_swap" else x.permute(0, 2, 4, 1, 3, 5)
        x = x.reshape(B, gh * gw, 3 * ph * pw)
        if not self.rounding:
            return x.to(self.dt)
        return _trunc_bf16(x).to(self.dt) if self.bug == "patch_round_trunc" else x.to(torch.bfloat16).to(self.dt)

    def _attention(self, a, blk):
        cfg, p = self.cfg, self.p
        B, T, D = a.shape
        h = cfg.enc_num_heads
        d = D // h
        qkv = self.r(a @ p[blk + "attn.qkv.weight"].t() + p[blk + "attn.qkv.bias"])
        q, k, v = qkv.reshape(B, T, 3, h, d).permute(2, 0, 3, 1, 4)
        if self.bug == "attn_drop_last_key":
            k, v = k[:, :, :-1], v[:, :, :-1]
        elif self.bug == "attn_extra_zero_key":
            k = torch.cat([k, k.new_zeros((B, h, 1, d))], dim=2)
            v = torch.cat([v, v.new_zeros((B, h, 1, d))], dim=2)
        s = (q @ k.transpose(-1, -2)) * (d ** -0.5)
        e = torch.exp(s - s.amax(dim=-1, keepdim=True))
        if self.bug == "attn_p_normalised_before_rounding":
            o = self.r(e / e.sum(dim=-1, keepdim=True)) @ v
        else:
            o = (self.r(e) @ v) / e.sum(dim=-1, keepdim=True)
        return self.r(o.permute(0, 2, 1, 3).reshape(B, T, D))

    def residual(self, img: torch.Tensor) -> torch.Tensor:
        """The residual stream after the last block, [B, T (+1), D]."""
        cfg, p = self.cfg, self.p
        D = cfg.embed_dim
        B = img.shape[0]
        x = self._patches(img) @ p["encoder.patch_embed.proj.weight"].reshape(D, -1).t() + p["encoder.patch_embed.proj.bias"]
        pos = p["encoder.pos_embed"]
        if self.vit:
            cls = p["encoder.cls_token"] if self.bug == "vitstr_cls_without_pos" else p["encoder.cls_token"] + pos[:, :1]
            pos = pos[:, 1:]
        if self.bug == "pos_embed_shift":
            pos = torch.roll(pos, -1, dims=1)
        x = x + pos
        if self.vit:
            x = torch.cat([cls.expand(B, -1, -1), x], dim=1)
        for i in range(cfg.enc_depth):
            blk = f"encoder.blocks.{i}."
            n1 = f"encoder.blocks.{i - 1}.norm1" if self.bug == "next_norm_from_own_block" and i > 0 else blk + "norm1"
            o = self._attention(self.r(self._ln(x, n1)), blk)
            x = x + (o @ p[blk + "attn.proj.weight"].t() + p[blk + "attn.proj.bias"])
            a = self.r(self._ln(x, blk + "norm2"))
            hdn = self.r(self.gelu(a @ p[blk + "mlp.fc1.weight"].t() + p[blk + "mlp.fc1.bias"]))
            x = x + (hdn @ p[blk + "mlp.fc2.weight"].t() + p[blk + "mlp.fc2.bias"])
        return x

    def encode(self, img: torch.Tensor) -> torch.Tensor:
        """PARSeq's memory / ViTSTR's forward_features: encoder.norm of the residual stream, not rounded."""
        return self._ln(self.residual(img), "encoder.norm")

    def tail(self, img: torch.Tensor, L: int) -> torch.Tensor:
        """ViTSTR's logits [B, L, C]: head(bf16(norm(x[:, 1 + j]))) for j < L."""
        assert self.vit
        x = self.residual(img)
        rows = x[:, :L] if self.bug == "vitstr_row_shift" else x[:, 1: 1 + L]
        return self.r(self._ln(rows, "encoder.norm")) @ self.p["head.weight"].t() + self.p["head.bias"]
