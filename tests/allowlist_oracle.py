"""Per-image class allowlists in the CPU oracles and in the reference's own modules.  TEST INFRASTRUCTURE ONLY.

The engine's allowlist (parseq_forward_args.class_mask) is specified as the reference model with its character head
wrapped: head'(x)[b, :, c] = head(x)[b, :, c] if c is allowed for image b, else -inf.  Everything else of
model.PARSeq.forward (AR loop, early exit, cloze refinement, NAR) and of ViTSTR's forward is unchanged, so every greedy
decision becomes the argmax of the masked row.  This module states that rule once, for three consumers:
  * `MaskedHead` wraps the reference's `head` module (tests/make_golden_allowlist.py builds the goldens with it);
  * `masked_oracle(cls)` subclasses an oracle restatement (ParseqOracle, DepthOracle) so that its `_decode` - the only
    producer of head outputs in `forward` - returns masked logits, and its margins are taken over allowed classes only;
  * `MaskedVitstrOracle` does the same for the ViTSTR restatement, whose head sees [B * s, D] rows: row r is image r // s.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import nn

from oracle.vitstr_oracle import VitstrOracle


def allowed_from_words(words: torch.Tensor, num_classes: int) -> torch.Tensor:
    """int32 [B, ceil(C / 32)] allowlist words -> bool [B, C] (bit c % 32 of word c / 32); EOS (class 0) always allowed."""
    w = words.to(torch.int64) & 0xFFFFFFFF
    bits = (w[:, :, None] >> torch.arange(32)) & 1
    allowed = bits.reshape(words.shape[0], -1)[:, :num_classes].bool()
    allowed[:, 0] = True
    return allowed


def allowed_from_strings(tokenizer, allowlist: Sequence[Optional[str]], num_classes: int) -> torch.Tensor:
    """bool [B, C] of one Optional[str] per image, independently of the engine's packing: None allows every class."""
    allowed = torch.zeros((len(allowlist), num_classes), dtype=torch.bool)
    for b, s in enumerate(allowlist):
        if s is None:
            allowed[b] = True
        else:
            allowed[b, 0] = True
            for ch in s:
                allowed[b, tokenizer._stoi[ch]] = True
    return allowed


def apply_mask(logits: torch.Tensor, allowed: torch.Tensor) -> torch.Tensor:
    """logits [B, ..., C] with the disallowed classes of each image set to -inf."""
    shape = (allowed.shape[0],) + (1,) * (logits.dim() - 2) + (allowed.shape[1],)
    return logits.masked_fill(~allowed.reshape(shape), float("-inf"))


class MaskedHead(nn.Module):
    """The reference's nn.Linear head, wrapped: [B, nq, D] rows (PARSeq) or [B * s, D] rows (ViTSTR, vitstr/model.py:26).
    It holds the head's own parameters (model.PARSeq._device reads them off `head`)."""

    def __init__(self, head: nn.Linear, allowed: torch.Tensor):
        super().__init__()
        self.weight, self.bias = head.weight, head.bias
        self.allowed = allowed

    def forward(self, x):
        out = F.linear(x, self.weight, self.bias)
        B = self.allowed.shape[0]
        if out.dim() == 2:                       # ViTSTR: row r of [B * s, C] belongs to image r // s
            return apply_mask(out, self.allowed.repeat_interleave(out.shape[0] // B, dim=0))
        return apply_mask(out, self.allowed)


def masked_oracle(base):
    """A subclass of the oracle class `base` whose head outputs are masked by `self.allowed` (bool [B, C])."""

    class Masked(base):
        allowed: torch.Tensor

        def _decode(self, *args, **kwargs):
            return apply_mask(super()._decode(*args, **kwargs), self.allowed)

        @staticmethod
        def _margin(logits):
            # top-1 minus top-2 of the masked row: a lone allowed class has no competitor (margin +inf)
            top2 = logits.topk(2, dim=-1).values
            m = top2[..., 0] - top2[..., 1]
            return torch.where(torch.isneginf(top2[..., 1]), torch.full_like(m, float("inf")), m)

    Masked.__name__ = "Masked" + base.__name__
    return Masked


class MaskedVitstrOracle(VitstrOracle):
    allowed: torch.Tensor

    def model_forward(self, img, seqlen: int = 25):
        return apply_mask(super().model_forward(img, seqlen), self.allowed)
