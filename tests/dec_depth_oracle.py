"""CPU oracle of PARSeq decoders of any depth (dec_depth >= 1).  TEST INFRASTRUCTURE ONLY.

`oracle.parseq_oracle.ParseqOracle` restates the depth-1 decoder (query stream only).  `DepthOracle` extends it to N
layers (strhub/models/parseq/modules.py:81-125): every layer runs the query stream, every layer but the last also
updates the content stream; both streams of layer l take their self-attention K/V from norm_c_l(content_l); the content
stream's own queries are norm_c_l(content_l) under the content mask `tgt_mask`.  `decoder.norm` and `head` follow the
last layer.  The precisions are those of ParseqOracle: "bf16" rounds, at the engine's points, the LayerNorm outputs, the
content K/V, the attention outputs and the GELU output of both streams.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.parseq_oracle import ParseqOracle

_FROM_QUERY_MASK = object()


def content_mask_of(query_mask, nk):
    """The content mask the reference's forward passes with a query mask (model.py:117,130-136,157-165): tgt_mask and
    query_mask are one tensor, of which the query mask is a row slice.  AR step i: query_mask = causal[i:j, :j], tgt_mask =
    causal[:j, :j]; refinement: both are the cloze mask; NAR: no mask (the context is BOS alone)."""
    if query_mask is None:
        return None
    if query_mask.shape[0] == nk:
        return query_mask
    return torch.triu(torch.ones((nk, nk), dtype=torch.bool), 1)


class DepthOracle(ParseqOracle):
    def __init__(self, cfg, state_dict, precision: str = "fp32"):
        depth, cfg.dec_depth = cfg.dec_depth, 1        # the base class checks for the depth it restates
        try:
            super().__init__(cfg, state_dict, precision)
        finally:
            cfg.dec_depth = depth
        if precision == "bf16":                        # the tensor-core weights of layers >= 1 too (rounding is idempotent)
            from parseq_b200.weights import gemm_weight_keys
            for k in gemm_weight_keys(cfg):
                self.p[k] = self.p[k].to(torch.bfloat16).to(self.dt)

    @staticmethod
    def _mask(B, nq, nk, attn_mask, pad_mask):
        if attn_mask is None and pad_mask is None:
            return None
        m = torch.zeros((B, nq, nk), dtype=torch.bool)
        if attn_mask is not None:
            m = m | attn_mask[None]
        if pad_mask is not None:
            m = m | pad_mask[:, None, :]
        return m

    def _stream(self, l, x, xn, kvn, memory_r, mask):
        """DecoderLayer.forward_stream (modules.py:55-79) of layer l: x the residual, xn its LayerNorm, kvn the keys."""
        p = self.p
        L = f"decoder.layers.{l}"
        y = x + self._mha(L + ".self_attn", xn, kvn, mask)
        y = y + self._mha(L + ".cross_attn", self.r(self._ln(y, L + ".norm1", 1e-5)), memory_r, None)
        hdn = self.r(F.gelu(self.r(self._ln(y, L + ".norm2", 1e-5)) @ p[L + ".linear1.weight"].t()
                            + p[L + ".linear1.bias"]))
        return y + (hdn @ p[L + ".linear2.weight"].t() + p[L + ".linear2.bias"])

    def decoder_out(self, ids, memory_r, query, query_mask, pad_mask, content_mask):
        """PARSeq.decode (model.py:86-103): Decoder output including decoder.norm, before the head."""
        ctx = self._context(ids)
        B, nq, nk = query.shape[0], query.shape[1], ids.shape[1]
        qm = self._mask(B, nq, nk, query_mask, pad_mask)
        cm = self._mask(B, nk, nk, content_mask, pad_mask)
        depth = self.cfg.dec_depth
        for l in range(depth):
            L = f"decoder.layers.{l}"
            cn = self.r(self._ln(ctx, L + ".norm_c", 1e-5))
            qn = self.r(self._ln(query, L + ".norm_q", 1e-5))
            query_next = self._stream(l, query, qn, cn, memory_r, qm)
            if l < depth - 1:
                ctx = self._stream(l, ctx, cn, cn, memory_r, cm)
            query = query_next
        return self._ln(query, "decoder.norm", 1e-5)

    def _decode(self, ids, memory_r, query, query_mask, pad_mask, content_mask=_FROM_QUERY_MASK):
        if content_mask is _FROM_QUERY_MASK:
            content_mask = content_mask_of(query_mask, ids.shape[1])
        out = self.r(self.decoder_out(ids, memory_r, query, query_mask, pad_mask, content_mask))
        return out @ self.p["head.weight"].t() + self.p["head.bias"]
