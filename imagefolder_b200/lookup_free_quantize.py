"""LFQ / BSQ multi-scale residual quantizer -- drop-in for the reference's
tokenizer/tokenizer_image/lookup_free_quantize.py (LFQ :83).

Same constructor, return 5-tuple and state_dict keys (`ema_vocab_hit_SV`, `scaler`,
`quant_resi.qresi_ls.*`; non-persistent `mask`, `codebook`).  The arithmetic runs in
libxqb200.so (csrc/ms_kernels.cu: ms_forward_kernel mode XQ_MS_BSQ + bsq_entropy_*_kernel, or mode
XQ_MS_BSQ_HARD + bsq_hard_*_kernel for soft_entropy=False).

Reference behaviour that is kept on purpose:
  * soft_entropy=True: the entropy term indexes the batch with an INT mask (`z[mask]`, :285) and therefore
    only ever looks at batch rows 0 and 1 -- reproduced exactly (and B >= 2 is required like there);
  * soft_entropy=False: entropy_loss over the 2^C-code softmax (:41-79, :220-229), a real masked mean over
    every image that still quantizes at the scale.  It is evaluated in closed form (per-bit sigmoids; the
    codebook distribution as a 2^(C/2) x 2^(C - C/2) contraction), so the [B, HW, 2^C] logits are never built.
    1 <= C <= 16; B == 1 raises like the reference (einops cannot reduce its 0-d masked mean);
  * all three losses are divided by SN (:238-240), unlike VectorQuantizer2;
  * the dead einsum + softmax over the 2^C codebook (:286-287, result overwritten) is NOT computed.
"""
from __future__ import annotations

from math import sqrt
from typing import Tuple

import torch
from torch import nn as nn
from torch.nn import functional as F

from . import _capi as C
from . import ops
from .quant import Phi, PhiNonShared, PhiPartiallyShared, PhiShared, _MultiScaleBase, build_quant_resi

__all__ = ["LFQ"]


class LFQ(_MultiScaleBase):
    def __init__(
            self, codebook_size, Cvae, using_znorm=False, beta: float = 0.25,
            default_qresi_counts=0, v_patch_nums=None, quant_resi=0.5, share_quant_resi=4,
            num_latent_tokens=256, codebook_drop=0.0, scale=1,
            sample_minimization_weight=1.0, batch_maximization_weight=1.0, entropy_weight=0.1, soft_entropy=True,
    ):
        super().__init__()
        self.Cvae: int = Cvae
        self.vocab_size: int = 2 ** self.Cvae
        assert self.vocab_size == codebook_size
        self.using_znorm: bool = using_znorm
        self.v_patch_nums: Tuple[int] = v_patch_nums
        self.num_latent_tokens = num_latent_tokens
        self.entropy_weight = entropy_weight
        self.soft_entropy = soft_entropy
        self.persample_entropy_compute = 'analytical'

        self.quant_resi_ratio = quant_resi
        self.quant_resi = build_quant_resi(Cvae, quant_resi, share_quant_resi, default_qresi_counts, self.v_patch_nums)

        self.register_buffer('ema_vocab_hit_SV', torch.full((len(self.v_patch_nums), self.vocab_size), fill_value=0.0))
        self.register_buffer('_record_hit_dev', torch.zeros(2, dtype=torch.int64), persistent=False)
        self.register_buffer('mask', 2 ** torch.arange(self.Cvae), persistent=False)
        self.beta: float = beta
        self.codebook_drop = codebook_drop

        scaler = scale ** torch.arange(len(self.v_patch_nums))
        if using_znorm:
            scaler = scaler / sqrt(self.Cvae)
        self.register_buffer('scaler', scaler)
        self._scaler_host = [float(s) for s in scaler.float().tolist()]

        self.sample_minimization_weight = sample_minimization_weight
        self.batch_maximization_weight = batch_maximization_weight

        all_codes = torch.arange(codebook_size)
        bits = self.indices_to_bits(all_codes)
        codebook = bits * 2.0 - 1.0
        self.register_buffer('codebook', codebook, persistent=False)
        self.prog_si = -1

    def extra_repr(self) -> str:
        return f'{self.v_patch_nums}, znorm={self.using_znorm}, beta={self.beta}  |  S={len(self.v_patch_nums)}, quant_resi={self.quant_resi_ratio}'

    def _load_from_state_dict(self, *args, **kwargs):
        super()._load_from_state_dict(*args, **kwargs)
        self._scaler_host = [float(s) for s in self.scaler.float().tolist()]

    def _desc(self, B, H, W, patch_nums=None):
        pns = list(patch_nums if patch_nums is not None else self.v_patch_nums)
        w, b, K = self._phi_params()
        SN = len(pns)
        pmap = self._phi_map(SN) if K else [-1] * SN
        d = C.make_ms_desc(B, self.Cvae, H, W, self.vocab_size, K, pns, pmap, C.XQ_MS_BSQ,
                           scaler=self._scaler_host[:SN], resi_ratio=abs(self.quant_resi_ratio), beta=self.beta,
                           loss_div_sn_all=True, channel_norm=self.using_znorm, entropy_weight=self.entropy_weight,
                           w_sample=self.sample_minimization_weight, w_batch=self.batch_maximization_weight)
        return d, w, b, pns

    def forward(self, f_BChw: torch.Tensor, ret_usages=False, dropout=None):
        """-> (f_hat, usages|None, vq, commit, entropy)   (lookup_free_quantize.py:149-250)"""
        if not self.training:
            # the reference's eval branch raises (list + int, :174)
            raise TypeError('can only concatenate list (not "int") to list')
        if not self.soft_entropy and self.Cvae > 16:
            raise NotImplementedError(f"soft_entropy=False is built for 1 <= Cvae <= 16 (got {self.Cvae})")
        if f_BChw.dtype != torch.float32:
            f_BChw = f_BChw.float()
        B, Cc, H, W = f_BChw.shape
        if B < 2:
            if self.soft_entropy:
                # soft_entropy_loss gathers batch rows with the int mask (values 0/1), :285
                raise IndexError(f"index 1 is out of bounds for dimension 0 with size {B}")
            # entropy_loss: mask.squeeze() is 0-d, masked_mean returns a 0-d tensor and einops' "... D -> D" raises (:62)
            raise RuntimeError('Error while processing mean-reduction pattern "... D -> D": expected >=1 dims, '
                               'received a 0-dim tensor (batch size 1)')
        d, w, b, pns = self._desc(B, H, W)
        if not self.soft_entropy:
            d.mode = C.XQ_MS_BSQ_HARD
        nq = self._n_quantizers(B, dropout, f_BChw.device, require_dropout=True)
        f_hat, vq, commit, ent, idx_all, hist = ops.ms_forward(f_BChw, None, w, b, nq, d, want_hist=True)
        usages = self._update_usage(hist, f_BChw.numel() / f_BChw.shape[1], ret_usages)
        self.last_idx_Bl = ops.split_scales(idx_all, B, pns)
        return f_hat, usages, vq, commit, ent

    def bits_to_indices(self, bits):
        """:254-268 -- bit c has weight 2^c."""
        assert bits.shape[-1] == self.Cvae
        indices = 2 ** torch.arange(0, self.Cvae, 1, dtype=torch.long, device=bits.device)
        return (bits * indices).sum(-1)

    def indices_to_bits(self, x, si=None):
        """:270-281."""
        mask = 2 ** torch.arange(self.Cvae, device=x.device, dtype=torch.long)
        x = (x.unsqueeze(-1) & mask) != 0
        if si is None:
            return x
        return torch.where(x, self.scaler[si], -self.scaler[si])
