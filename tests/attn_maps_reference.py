"""The cross-attention maps of the PARSeq decoder from the fp64 rounding-point model.  TEST HELPER.

`MapsReference` wraps tests/decoder_reference.py's `DecoderReference` (depth 1) or `DepthDecoderReference` (any depth)
and records, in every decode pass, the head-averaged cross-attention weights (`ca_weights` of nn.MultiheadAttention,
strhub/models/parseq/modules.py:74) of the query stream of the last decoder layer.  The weights are computed from the
model's own query (LayerNorm outputs rounded to bf16 as the engine rounds them, the projection and the 1/sqrt(head_dim)
scale in `accum`) and its bf16 K, so fed the engine's bf16 memory the maps differ from the engine's only by the fp32
summation order of the decoder.  The existing models are used as they are; only their `_mha` is observed.

The three passes give the maps of the three schedules of parseq_forward_args.attn_maps:
  * `ar(memory, ids)`: AR without refinement, one causal pass over [BOS, ids[:, :L-1]] (the returned ids);
  * `nar(memory, L)`: the NAR pass;
  * `refine(memory, contexts)`: the last of the cloze passes, contexts[r] the context of pass r.

`bug=` injects one wrong detail (BUGS); tests/test_attn_maps_budget_cpu.py shows each outside BOUNDS and the fp32
stand-in (accum=torch.float32) inside, so the bounds tests/test_gpu_attn_maps.py holds the engine to separate a correct
map from these mistakes.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Sequence

import torch

from decoder_reference import DecoderReference, DepthDecoderReference

BUGS = {
    "head0": "the map is head 0's weights instead of the mean over the heads",
    "first_refine": "the maps come from the first refinement pass instead of the last",
    "layer0": "the maps come from layer 0 of a depth-2 decoder instead of the last layer",
    "no_scale": "the scores miss the 1/sqrt(head_dim) scale",
    "key_shift": "map column t holds the weight of key t - 1",
    "col_major": "the map is laid out column-major over the patch grid",
    "ar_from_nar": "the rows of an AR-only schedule come from the NAR pass's queries",
}

# Bounds on |engine - model| * T over the map entries of one pass (T image tokens: the error relative to the uniform
# weight 1 / T): the median, the mean and the 99th percentile.  Enforced by tests/test_attn_maps_budget_cpu.py: the fp32
# stand-in stays within half of each bound, and every bug in BUGS exceeds one of them by 2x or more.  Measured there
# (not enforced): the stand-in's worst figures (PARSeq-S at depth 2, where a second layer carries the bf16 flips of the
# first into every row) are p50 7.6e-4, mean 2.0e-3, p99 1.8e-2, and the smallest bug figures p50 0.32, mean 0.49,
# p99 2.7.  The bounds leave the engine's fp32 tensor-core sums, which flip more bf16 roundings than the stand-in's,
# room above the stand-in.
BOUNDS: Dict[str, float] = {"p50": 2.0e-2, "mean": 5.0e-2, "p99": 5.0e-1}

# Bounds on |engine - reference| * T against the goldens of the reference's own modules (tests/golden/attention, fp64
# end to end): the engine's error there also carries its bf16 encoder, so they are wider than BOUNDS.  Enforced by
# tests/test_attn_maps_budget_cpu.py: every bug in BUGS exceeds one of them by 2x or more as well.  Measured on an H100
# (not enforced): the engine's worst golden figures are p50 3.1e-3, mean 7.2e-3, p99 5.9e-2.
GOLDEN_BOUNDS: Dict[str, float] = {"p50": 5.0e-2, "mean": 1.0e-1, "p99": 1.0}


def map_stats(got: torch.Tensor, ref: torch.Tensor) -> Dict[str, float]:
    """The median, mean, 99th percentile and max of |got - ref| * T (T = the last dimension)."""
    ref = ref.double()
    T = ref.shape[-1]
    d = ((got.to(ref.device, torch.float64) - ref).abs() * T).flatten()
    n = d.numel()
    return {"p50": d.kthvalue((n + 1) // 2).values.item(), "mean": d.mean().item(),
            "p99": d.kthvalue(max(1, math.ceil(0.99 * n))).values.item(), "max": d.max().item()}


def excess(stats: Dict[str, float], bounds: Optional[Dict[str, float]] = None) -> Dict[str, float]:
    return {k: stats[k] / b for k, b in (bounds or BOUNDS).items()}


def format_stats(name: str, s: Dict[str, float]) -> str:
    return f"{name}: |d| * T: p50 {s['p50']:.2e}  mean {s['mean']:.2e}  p99 {s['p99']:.2e}  max {s['max']:.2e}"


class _Recorder:
    """Observes every cross-attention call of the wrapped model and records its head-averaged weights."""

    def _mha(self, prefix, q_in, kv_in, mask):
        if prefix.endswith("cross_attn"):
            self.records.append(self._weights(prefix, q_in, kv_in))
        return super()._mha(prefix, q_in, kv_in, mask)

    def _weights(self, prefix, q_in, kv_in):
        p, cfg = self.p, self.cfg
        D, h = cfg.embed_dim, cfg.dec_num_heads
        d = D // h
        W, b = p[prefix + ".in_proj_weight"], p[prefix + ".in_proj_bias"]
        scale = 1.0 if self.map_bug == "no_scale" else 1.0 / math.sqrt(d)
        q = (q_in @ W[:D].t() + b[:D]) * scale
        k = self.r(kv_in @ W[D:2 * D].t() + b[D:2 * D])
        B, nq, nk = q.shape[0], q.shape[1], k.shape[1]
        s = q.reshape(B, nq, h, d).transpose(1, 2) @ k.reshape(B, nk, h, d).permute(0, 2, 3, 1)   # [B, h, nq, nk]
        a = torch.softmax(s, dim=-1)
        w = a[:, 0] if self.map_bug == "head0" else a.mean(dim=1)
        if self.map_bug == "key_shift":
            w = torch.roll(w, 1, dims=-1)
        elif self.map_bug == "col_major":
            gh, gw = cfg.grid
            w = w.reshape(B, nq, gh, gw).transpose(-1, -2).reshape(B, nq, nk)
        return w


class _Depth1(_Recorder, DecoderReference):
    pass


class _DepthN(_Recorder, DepthDecoderReference):
    pass


class MapsReference:
    def __init__(self, cfg, state_dict, accum=torch.float64, device="cpu", bug: Optional[str] = None):
        if bug is not None and bug not in BUGS:
            raise KeyError(bug)
        self.bug = bug
        self.m = (_DepthN if cfg.dec_depth > 1 else _Depth1)(cfg, state_dict, accum=accum, device=device)
        self.m.map_bug = bug
        self.bos = cfg.num_tokens - 2

    def _maps(self, run):
        """The last layer's query-stream maps of one pass: the last cross-attention call (the content stream is not
        updated in the last layer), or the first (layer 0's query stream) under bug "layer0"."""
        self.m.records = []
        run()
        return self.m.records[0 if self.bug == "layer0" else -1]

    def ar(self, memory, ids):
        """Maps [B, L, T] of an AR-only schedule whose returned ids are `ids` [B, L]."""
        B, L = ids.shape
        if self.bug == "ar_from_nar":
            return self._maps(lambda: self.m.nar(memory, L))
        ctx = torch.cat([torch.full((B, 1), self.bos, dtype=torch.long), ids[:, :L - 1].long().cpu()], dim=1)
        return self._maps(lambda: self.m.ar(memory, ctx))

    def nar(self, memory, L):
        return self._maps(lambda: self.m.nar(memory, L))

    def refine(self, memory, contexts: Sequence[torch.Tensor]):
        """Maps of the last cloze pass; contexts[r] [B, L] is the context (BOS first) of refinement pass r."""
        ctx = contexts[0] if self.bug == "first_refine" else contexts[-1]
        return self._maps(lambda: self.m.refine(memory, ctx))
