"""The PARSeq decoder as an fp64 rounding-point model, fed a given encoder memory.  TEST HELPER.

`DecoderReference` (depth 1, a `ParseqOracle`) and `DepthDecoderReference` (any depth, a `DepthOracle`) round to bf16
at exactly the engine's rounding points (DESIGN.md section 5: LayerNorm outputs, the (position, token) K/V table, the
cross K/V, attention outputs, GELU) and compute everything else in `accum` (fp64 by default).  Two engine functions
are restated rather than the exact ones: the polynomial erf-GELU (`engine_gelu`) and, with `cluster=True`, the cluster
AR kernel's bf16 hi + lo cross-attention operands (`hi_lo`).  Fed `bf16(memory)` of
the engine's own encoder, the model differs from the engine only by the engine's fp32 summation order, so the
comparison sees the decoder's arithmetic alone, without the encoder's bf16 cascade.  The model runs on the device its
inputs are on (fp64 has no TF32 path, so a GPU computes it exactly as a CPU would, only faster).

Under teacher forcing every AR step is a fixed function of the memory and the context, so the whole AR loop is one
decode pass: query i over keys 0..i under the causal mask (`ar`).  `nar` and `refine` are the other two passes of
`PARSeq.forward` (model.py:148-166).

`accum=torch.float32` is a CPU stand-in for the engine: the same rounding points with fp32 arithmetic.  Its distance
from the fp64 model is the noise floor a correct decoder shows (rare bf16 rounding flips dominate it).

`bug=` injects one wrong detail into the model (BUGS).  tests/test_decoder_budget_cpu.py shows each of them outside
BOUNDS and the fp32 stand-in inside, so the bounds that tests/test_gpu_decoder_isolated.py holds the engine to are the
ones that separate a correct decoder from these mistakes.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import torch

from dec_depth_oracle import DepthOracle
from oracle.parseq_oracle import EOS_ID, ParseqOracle

# Each entry changes exactly one thing in the model.
BUGS = {
    "self_mask_leak": "the self-attention mask lets query i see key i + 1",
    "ln_eps": "the query stream's per-step LayerNorms (norm1, norm2, decoder.norm) use eps 1e-6 instead of 1e-5",
    "cross_extra_zero_key": "cross-attention sees one extra key whose K and V are zero (a padding row not masked)",
    "cross_drop_last_key": "cross-attention drops the last image token",
    "cross_q_bf16": "the cross-attention query is rounded to bf16 (the hi + lo split lost)",
    "eos_mask_off_by_one": "the refinement's padding mask starts one key after the first EOS",
    "pos_query_shift": "context row k adds pos_queries[k] instead of pos_queries[k - 1]",
    "no_linear2_bias": "the decoder MLP's linear2 bias is dropped",
    "no_head_bias": "the head bias is dropped",
    "self_extra_zero_key": "every self-attention query also sees one key whose K and V are zero (an unwritten cache slot, "
                           "or a lane past nkeys)",
    "self_drop_own_key": "AR query i >= 1 does not see key i (query 0 keeps BOS)",
    "cloze_mask_shift": "the refinement hides key i from query i >= 1 instead of key i + 1 (query 0 keeps every key)",
    "eos_mask_eos_only": "the refinement's padding mask hides the EOS keys only, not every key from the first EOS on",
    "norm_qc_eps": "norm_q and norm_c use eps 1e-6 instead of 1e-5 (every layer; at depth 1 the (position, token) table "
                   "and the query table)",
    "self_q_bf16": "the self-attention query (the pre-scaled query table; at depth >= 2 the query GEMM output) is rounded "
                   "to bf16",
}

# Bounds on |engine - model| over the logits of one decoder pass, relative to the standard deviation sigma of the model's
# logits, per (embed_dim, dec_depth): the median, the mean and the 99th percentile of |d| / sigma.  A correct decoder's
# error is bf16 rounding flips (an fp32 sum on the other side of a bf16 rounding boundary than the fp64 one), each carried
# into everything downstream of it.  While flips are rare (D = 192) most logits see none and the median is ~1e-7; a wrong
# detail moves every logit a little, so the median separates the small bugs (an eps, one extra or missing key, a rounded
# q) from the noise by a factor the mean cannot give.  The wider the decoder, the longer its sums and the more flips per
# row; from D = 384 on, and at depth 2, the engine's flips reach most rows and its median comes within 2x of those small
# bugs (its fp32 tensor-core sums flip more often than the fp32 stand-in's, so at D >= 384 the engine's measured figure,
# not the stand-in's, is the floor of a bound).  The mean and the p99 catch what touches few rows.
# tests/test_decoder_budget_cpu.py is the reason for every number here: the fp32 stand-in stays within half of each
# bound, and every bug in BUGS exceeds one of them by 2x or more, save the exceptions it names with their numbers.  The
# engine's own figures (DESIGN.md section 5) are below each bound by 1.3x or more.
BOUNDS: Dict[Tuple[int, int], Dict[str, float]] = {
    (192, 1): {"p50": 8.0e-4, "mean": 2.0e-3, "p99": 1.4e-2},
    (384, 1): {"p50": 1.6e-3, "mean": 2.9e-3, "p99": 2.0e-2},
    (768, 1): {"p50": 2.6e-3, "mean": 3.6e-3, "p99": 1.4e-2},
    (384, 2): {"p50": 3.5e-3, "mean": 4.4e-3, "p99": 1.8e-2},
}


def budget_stats(got: torch.Tensor, ref: torch.Tensor) -> Dict[str, float]:
    """sigma of the model's logits, and the median, mean, 99th percentile and max of |got - ref| relative to it."""
    ref = ref.double()
    d = (got.to(ref.device, torch.float64) - ref).abs().flatten()
    sigma = ref.std().item()
    n = d.numel()
    return {"sigma": sigma, "p50": d.kthvalue((n + 1) // 2).values.item() / sigma, "mean": d.mean().item() / sigma,
            "p99": d.kthvalue(max(1, math.ceil(0.99 * n))).values.item() / sigma, "max": d.max().item() / sigma}


def excess(stats: Dict[str, float], key: Tuple[int, int], bounds=None) -> Dict[str, float]:
    """stat / bound for every bounded statistic of BOUNDS[(embed_dim, dec_depth)] (or of bounds[key], another module's
    table): <= 1 inside the budget."""
    return {k: stats[k] / b for k, b in (BOUNDS if bounds is None else bounds)[key].items()}


def format_stats(name: str, s: Dict[str, float]) -> str:
    return (f"{name}: sigma {s['sigma']:.3f}  |d| / sigma: p50 {s['p50']:.2e}  mean {s['mean']:.2e}  p99 {s['p99']:.2e}  "
            f"max {s['max']:.2e}")


def forced_ar_ids(B, L, C, bos, seed):
    """AR teacher forcing [B, L] int32: BOS, then ids over all C classes with C - 1 and EOS at scattered positions."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, C, (B, L), generator=g, dtype=torch.int32)
    for b in range(B):
        pos = torch.randperm(L - 1, generator=g)[:4] + 1
        ids[b, pos[:2]] = C - 1
        ids[b, pos[2:]] = EOS_ID
    ids[:, 0] = bos
    return ids


def refine_context(B, L, C, bos, first_eos, seed):
    """Refinement contexts [B, L] int32: BOS, then ids over classes 1..C-1 (C - 1 included) and the first EOS of row b at
    position first_eos[b % len(first_eos)] (None: no EOS), followed by more ids and EOS."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, max(C, 2), (B, L), generator=g, dtype=torch.int32)
    ids[:, L // 2] = C - 1
    for b in range(B):
        e = first_eos[b % len(first_eos)]
        if e is not None and e < L:
            ids[b, e] = EOS_ID
            ids[b, e + 1:] = torch.randint(0, C, (L - e - 1,), generator=g, dtype=torch.int32)
    ids[:, 0] = bos
    return ids


# The engine's erf-GELU (ptx.cuh gelu_erf): x Phi(x) with Phi(-|x|) = 2^q(|x|), q a degree-8 polynomial on [0, 8.5]
_GELU_Q = (8.503329848e-03, -2.785826938e-02, 4.857975011e-02, -8.378244194e-02, 1.570760869e-01, -2.896217881e-01,
           -1.247551552e+01, -2.737368526e+01, -1.651358203e+01)


def engine_gelu(x: torch.Tensor) -> torch.Tensor:
    """The engine's GELU evaluated in the dtype of x.  It is within 1.2e-5 (relative) of the exact erf-GELU, yet that
    is enough to put ~0.04 % of its bf16-rounded outputs on the other side of a rounding boundary, i.e. one or two of the
    1536..3072 hidden values of a decoder row; the model therefore rounds the engine's function, not the exact one."""
    u = x.abs().clamp(max=8.5)
    t = u * (2.0 / 8.5) - 1.0
    q = torch.full_like(x, _GELU_Q[0])
    for c in _GELU_Q[1:]:
        q = q * t + c
    return x.clamp(min=0.0) - u * torch.exp2(q)


def _bf16(x):
    return x.to(torch.bfloat16).to(x.dtype)


def hi_lo(x: torch.Tensor) -> torch.Tensor:
    """x as the cluster AR kernel feeds it to the tensor cores: bf16(x) + bf16(x - bf16(x)), ~16 mantissa bits."""
    h = _bf16(x)
    return h + _bf16(x - h)


class _RoundingPointModel:
    def _setup(self, accum, device, bug, cluster):
        if bug is not None and bug not in BUGS:
            raise KeyError(bug)
        self.bug = bug
        self.cluster = cluster
        self.dt = accum                  # ParseqOracle.r rounds to bf16 and returns to self.dt
        self.device = torch.device(device)
        self.p = {k: v.to(device=self.device, dtype=accum) for k, v in self.p.items()}
        if bug == "no_linear2_bias":
            for k in self.p:
                if k.endswith(".linear2.bias"):
                    self.p[k] = torch.zeros_like(self.p[k])
        if bug == "no_head_bias":
            self.p["head.bias"] = torch.zeros_like(self.p["head.bias"])

    # -- the overrides that carry the bugs --------------------------------------------------------------------------
    def _ln(self, x, prefix, eps):
        if self.bug == "ln_eps" and prefix.startswith("decoder.") and prefix.endswith(("norm1", "norm2", "decoder.norm")):
            eps = 1e-6
        if self.bug == "norm_qc_eps" and prefix.endswith(("norm_q", "norm_c")):
            eps = 1e-6
        return super()._ln(x, prefix, eps)

    def _context(self, ids):
        if self.bug != "pos_query_shift":
            return super()._context(ids)
        D = self.cfg.embed_dim
        emb = math.sqrt(D) * self.p["text_embed.embedding.weight"][ids]
        j = ids.shape[1]
        if j > 1:
            emb = torch.cat([emb[:, :1], self.p["pos_queries"][:, 1:j] + emb[:, 1:]], dim=1)
        return emb

    def _mha(self, prefix, q_in, kv_in, mask):
        """ParseqOracle._mha with the cross- and self-attention bugs."""
        p, cfg = self.p, self.cfg
        D, h = cfg.embed_dim, cfg.dec_num_heads
        d = D // h
        W, b = p[prefix + ".in_proj_weight"], p[prefix + ".in_proj_bias"]
        B, nq, _ = q_in.shape
        q = (q_in @ W[:D].t() + b[:D]) * (1.0 / math.sqrt(d))
        kv = self.r(kv_in @ W[D:].t() + b[D:])
        if prefix.endswith("cross_attn"):
            if self.bug == "cross_q_bf16":
                q = self.r(q)
            elif self.bug == "cross_extra_zero_key":
                kv = torch.cat([kv, kv.new_zeros((B, 1, 2 * D))], dim=1)
            elif self.bug == "cross_drop_last_key":
                kv = kv[:, :-1]
        elif prefix.endswith("self_attn"):
            if self.bug == "self_q_bf16":
                q = self.r(q)
            elif self.bug == "self_extra_zero_key":
                kv = torch.cat([kv, kv.new_zeros((B, 1, 2 * D))], dim=1)
                if mask is not None:
                    mask = torch.cat([mask, mask.new_zeros((B, nq, 1))], dim=2)
        nk = kv.shape[1]
        k, v = kv[..., :D], kv[..., D:]
        q = q.reshape(B, nq, h, d).transpose(1, 2)
        k = k.reshape(B, nk, h, d).transpose(1, 2)
        v = v.reshape(B, nk, h, d).transpose(1, 2)
        if self.cluster and prefix.endswith("cross_attn"):
            # the cluster AR kernel: q and the un-normalised P = exp(s - max) enter the MMAs as hi + lo pairs, the row
            # sum is taken from P itself
            q = hi_lo(q)
        s = q @ k.transpose(-1, -2)
        if mask is not None:
            s = s.masked_fill(mask[:, None], float("-inf"))
        if self.cluster and prefix.endswith("cross_attn"):
            e = torch.exp(s - s.amax(dim=-1, keepdim=True))
            o = (hi_lo(e) @ v) / e.sum(dim=-1, keepdim=True)
        else:
            o = torch.softmax(s, dim=-1) @ v
        o = self.r(o.transpose(1, 2).reshape(B, nq, D))
        return o @ p[prefix + ".out_proj.weight"].t() + p[prefix + ".out_proj.bias"]

    @staticmethod
    def _mask(B, nq, nk, attn_mask, pad_mask):
        """DepthOracle._mask on the device of the masks."""
        if attn_mask is None and pad_mask is None:
            return None
        dev = (attn_mask if attn_mask is not None else pad_mask).device
        m = torch.zeros((B, nq, nk), dtype=torch.bool, device=dev)
        if attn_mask is not None:
            m = m | attn_mask[None]
        if pad_mask is not None:
            m = m | pad_mask[:, None, :]
        return m

    # -- the passes of PARSeq.forward under teacher forcing -----------------------------------------------------------
    def _memory(self, memory):
        return self.r(memory.to(device=self.device, dtype=self.dt))

    def _pos(self, B, L):
        return self.p["pos_queries"][:, :L].expand(B, -1, -1)

    def _causal(self, L):
        """Query i sees keys 0..i (model.py:130-136)."""
        m = torch.triu(torch.ones((L, L), dtype=torch.bool, device=self.device), 2 if self.bug == "self_mask_leak" else 1)
        if self.bug == "self_drop_own_key":
            i = torch.arange(1, L, device=self.device)
            m[i, i] = True
        return m

    def _cloze(self, L):
        """Query i sees every key but i + 1 (model.py:157)."""
        m = torch.zeros((L, L), dtype=torch.bool, device=self.device)
        if self.bug == "cloze_mask_shift":
            i = torch.arange(1, L, device=self.device)
            m[i, i] = True
        elif self.bug != "self_mask_leak":
            i = torch.arange(L - 1, device=self.device)
            m[i, i + 1] = True
        return m

    def ar(self, memory, forced_ids):
        """Logits [B, L, C] of the whole AR loop with step i fed forced_ids[:, i + 1] (forced_ids[:, 0] is BOS)."""
        ids = forced_ids.to(device=self.device, dtype=torch.long)
        B, L = ids.shape
        return self._decode(ids, self._memory(memory), self._pos(B, L), self._causal(L), None)

    def nar(self, memory, L):
        B = memory.shape[0]
        ids = torch.full((B, 1), self.cfg.num_tokens - 2, dtype=torch.long, device=self.device)
        return self._decode(ids, self._memory(memory), self._pos(B, L), None, None)

    def refine(self, memory, ctx_ids):
        """One cloze pass over the context ctx_ids [B, L] (BOS first), keys from the first EOS on masked."""
        ids = ctx_ids.to(device=self.device, dtype=torch.long)
        B, L = ids.shape
        pad = (ids == EOS_ID).int().cumsum(-1) > 0
        if self.bug == "eos_mask_eos_only":
            pad = ids == EOS_ID
        elif self.bug == "eos_mask_off_by_one":
            pad = torch.cat([pad.new_zeros((B, 1)), pad[:, :-1]], dim=1)
        return self._decode(ids, self._memory(memory), self._pos(B, L), self._cloze(L), pad)


class DecoderReference(_RoundingPointModel, ParseqOracle):
    """The depth-1 decoder (query stream only)."""

    def __init__(self, cfg, state_dict, accum=torch.float64, device="cpu", bug: Optional[str] = None,
                 cluster: bool = False):
        ParseqOracle.__init__(self, cfg, state_dict, "bf16")
        self._setup(accum, device, bug, cluster)

    def _decode(self, ids, memory_r, query, query_mask, pad_mask):
        """ParseqOracle._decode with its masks on the model's device."""
        p = self.p
        L = "decoder.layers.0"
        ctx = self._context(ids)
        qn = self.r(self._ln(query, L + ".norm_q", 1e-5))
        cn = self.r(self._ln(ctx, L + ".norm_c", 1e-5))
        mask = self._mask(query.shape[0], query.shape[1], ids.shape[1], query_mask, pad_mask)
        y = query + self._mha(L + ".self_attn", qn, cn, mask)
        y = y + self._mha(L + ".cross_attn", self.r(self._ln(y, L + ".norm1", 1e-5)), memory_r, None)
        hdn = self.r(engine_gelu(self.r(self._ln(y, L + ".norm2", 1e-5)) @ p[L + ".linear1.weight"].t()
                                 + p[L + ".linear1.bias"]))
        y = y + (hdn @ p[L + ".linear2.weight"].t() + p[L + ".linear2.bias"])
        out = self.r(self._ln(y, "decoder.norm", 1e-5))
        return out @ p["head.weight"].t() + p["head.bias"]


class DepthDecoderReference(_RoundingPointModel, DepthOracle):
    """Decoders of any depth: both streams, the content stream under the content mask of each pass."""

    def __init__(self, cfg, state_dict, accum=torch.float64, device="cpu", bug: Optional[str] = None,
                 cluster: bool = False):
        DepthOracle.__init__(self, cfg, state_dict, "bf16")
        self._setup(accum, device, bug, cluster)

    def _stream(self, l, x, xn, kvn, memory_r, mask):
        """DepthOracle._stream with the engine's GELU."""
        p = self.p
        L = f"decoder.layers.{l}"
        y = x + self._mha(L + ".self_attn", xn, kvn, mask)
        y = y + self._mha(L + ".cross_attn", self.r(self._ln(y, L + ".norm1", 1e-5)), memory_r, None)
        hdn = self.r(engine_gelu(self.r(self._ln(y, L + ".norm2", 1e-5)) @ p[L + ".linear1.weight"].t()
                                 + p[L + ".linear1.bias"]))
        return y + (hdn @ p[L + ".linear2.weight"].t() + p[L + ".linear2.bias"])
