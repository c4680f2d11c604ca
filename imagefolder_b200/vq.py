"""Single-scale VectorQuantizer -- drop-in for tokenizer/tokenizer_image/xqgan_model.py:722-833.

Same constructor / attributes / return tuple / state_dict keys (`embedding.weight`,
`ema_vocab_hit_SV`).  The arithmetic is the fused search kernel of csrc/vq_kernels.cu.
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .quant import _allreduce_hist_, _world_size, record_hit_property

__all__ = ["VectorQuantizer"]


class VectorQuantizer(nn.Module):
    sync_usages: bool = False  # True: usages are python floats like the reference (one host sync)
    record_hit = record_hit_property

    def __init__(self, vocab_size=8192, z_channels=32, beta=0.25, codebook_norm=True):
        super().__init__()
        self.vocab_size = vocab_size
        self.z_channels = z_channels
        self.beta = beta
        self.codebook_norm = codebook_norm

        self.embedding = nn.Embedding(self.vocab_size, self.z_channels)
        self.embedding.weight.data.uniform_(-1.0 / self.vocab_size, 1.0 / self.vocab_size)
        if self.codebook_norm:
            self.embedding.weight.data = F.normalize(self.embedding.weight.data, p=2, dim=-1)

        self.register_buffer("ema_vocab_hit_SV", torch.full((self.vocab_size,), fill_value=0.0))
        self.register_buffer("_record_hit_dev", torch.zeros(2, dtype=torch.int64), persistent=False)

    def no_weight_decay(self):
        return ['embedding.weight', ]

    def forward(self, z, ret_usages=True, dropout=None):
        """-> (z_q, [codebook_usage], vq_loss, commit_loss, 0.0)      (xqgan_model.py:745-801)"""
        assert z.shape[1] == self.z_channels
        margin = _world_size() * (z.numel() / self.z_channels) / self.vocab_size * 0.08
        z_q, vq_loss, commit_loss, idx, hist = ops.vq_forward(z, self.embedding.weight, self.beta, self.codebook_norm)
        self.last_idx = idx
        if ret_usages and self.training:
            _allreduce_hist_(hist)
            usage = torch.ops.xqb200.usage_ema_(self.ema_vocab_hit_SV, hist, self._record_hit_dev, margin)[0]
        else:
            # the reference leaves `codebook_usage` unbound here (NameError); report the current EMA instead
            usage = (self.ema_vocab_hit_SV >= margin).float().mean() * 100
        codebook_usage = float(usage) if self.sync_usages else usage
        return z_q, [codebook_usage], vq_loss, commit_loss, 0.0

    def f_to_idxBl_or_fhat(self, z: torch.Tensor, to_fhat: bool, v_patch_nums=None) -> List[torch.Tensor]:
        """-> [z_q] or [idx (N,) int64]                                 (xqgan_model.py:803-833)"""
        z_q, idx = ops.vq_lookup(z, self.embedding.weight.data, self.codebook_norm)
        return [z_q if to_fhat else idx]

    def idx_to_fhat(self, idx_list, last_one=True):
        """token indices [B, hw] (or (N,)) -> normalised code map [B,C,h,w]."""
        idx = idx_list[0] if isinstance(idx_list, (list, tuple)) else idx_list
        B = idx.shape[0] if idx.dim() == 2 else 1
        q = self.embedding.weight.data[idx.reshape(B, -1)]
        if self.codebook_norm:
            q = F.normalize(q, p=2, dim=-1)
        hw = int(q.shape[1] ** 0.5)
        q = q.view(B, hw, hw, self.z_channels).permute(0, 3, 1, 2).contiguous()
        return q if last_one else [q]
