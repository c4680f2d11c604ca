"""Multi-scale residual vector quantizer -- drop-in for the reference's
tokenizer/tokenizer_image/quant.py (VectorQuantizer2 :13, Phi :261, PhiShared :271,
PhiPartiallyShared :279, PhiNonShared :294).

Same constructor arguments, attributes, return tuples and state_dict keys
(`embedding.weight`, `ema_vocab_hit_SV`, `quant_resi.qresi_ls.{i}.{weight,bias}`); the arithmetic
runs in libxqb200.so (one fused CUDA kernel for the whole K-scale loop, csrc/ms_kernels.cu).

Differences from the reference, all host-side:
  * the SN per-scale histogram all-reduces (quant.py:104) are collapsed into ONE [SN,V] all-reduce;
  * `usages` are 0-dim device tensors unless `sync_usages=True` (the reference calls .item() per
    scale = SN host syncs per forward, quant.py:140); float(u) gives the reference value;
  * a process group is optional (the reference requires one even on 1 GPU, quant.py:137).
  * `record_hit` reads and writes a device counter that the usage-EMA kernel advances by SN per training forward.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import distributed as tdist, nn as nn
from torch.nn import functional as F

from . import _capi as C
from . import ops

__all__ = ["VectorQuantizer2", "Phi", "PhiShared", "PhiPartiallyShared", "PhiNonShared"]


def _world_size() -> int:
    return tdist.get_world_size() if (tdist.is_available() and tdist.is_initialized()) else 1


def _allreduce_hist_(hist: torch.Tensor) -> None:
    if tdist.is_available() and tdist.is_initialized() and tdist.get_world_size() > 1:
        tdist.all_reduce(hist)


def _set_record_hit(self, value: int) -> None:
    self._record_hit_dev.copy_(torch.tensor([int(value), 0]))


# The reference's `record_hit` (the usage EMA's step counter) as a view of the device buffer `_record_hit_dev` = [counter,
# kernel scratch word], which the usage-EMA kernel reads and advances without the host.  Reading it synchronises with the
# device, so no forward does; like the reference's plain attribute it is not part of the state_dict.
record_hit_property = property(lambda self: int(self._record_hit_dev[0]), _set_record_hit)


class Phi(nn.Conv2d):
    """quant.py:261-268.  Inside the quantizers the conv runs in the fused CUDA kernel; calling the
    module directly (VAR-side helpers) uses the library conv."""

    def __init__(self, embed_dim, quant_resi):
        ks = 3
        super().__init__(in_channels=embed_dim, out_channels=embed_dim, kernel_size=ks, stride=1, padding=ks // 2)
        self.resi_ratio = abs(quant_resi)

    def forward(self, h_BChw):
        return h_BChw.mul(1 - self.resi_ratio) + super().forward(h_BChw).mul_(self.resi_ratio)


class PhiShared(nn.Module):
    def __init__(self, qresi: Phi):
        super().__init__()
        self.qresi: Phi = qresi

    def __getitem__(self, _) -> Phi:
        return self.qresi

    def modules_list(self):
        return [self.qresi]

    def index_of(self, at_from_0_to_1: float) -> int:
        return 0


class PhiPartiallyShared(nn.Module):
    def __init__(self, qresi_ls: nn.ModuleList):
        super().__init__()
        self.qresi_ls = qresi_ls
        K = len(qresi_ls)
        self.ticks = np.linspace(1 / 3 / K, 1 - 1 / 3 / K, K) if K == 4 else np.linspace(1 / 2 / K, 1 - 1 / 2 / K, K)

    def index_of(self, at_from_0_to_1: float) -> int:
        return int(np.argmin(np.abs(self.ticks - at_from_0_to_1)).item())

    def __getitem__(self, at_from_0_to_1: float) -> Phi:
        return self.qresi_ls[self.index_of(at_from_0_to_1)]

    def modules_list(self):
        return list(self.qresi_ls)

    def extra_repr(self) -> str:
        return f'ticks={self.ticks}'


class PhiNonShared(nn.ModuleList):
    def __init__(self, qresi: List):
        super().__init__(qresi)
        K = len(qresi)
        self.ticks = np.linspace(1 / 3 / K, 1 - 1 / 3 / K, K) if K == 4 else np.linspace(1 / 2 / K, 1 - 1 / 2 / K, K)

    def index_of(self, at_from_0_to_1: float) -> int:
        return int(np.argmin(np.abs(self.ticks - at_from_0_to_1)).item())

    def __getitem__(self, at_from_0_to_1: float) -> Phi:
        return super().__getitem__(self.index_of(at_from_0_to_1))

    def modules_list(self):
        return [super(PhiNonShared, self).__getitem__(i) for i in range(len(self))]

    def extra_repr(self) -> str:
        return f'ticks={self.ticks}'


def build_quant_resi(Cvae, quant_resi, share_quant_resi, default_qresi_counts, v_patch_nums):
    """quant.py:28-39."""
    mk = lambda: (Phi(Cvae, quant_resi) if abs(quant_resi) > 1e-6 else nn.Identity())
    if share_quant_resi == 0:
        return PhiNonShared([mk() for _ in range(default_qresi_counts or len(v_patch_nums))])
    if share_quant_resi == 1:
        return PhiShared(mk())
    return PhiPartiallyShared(nn.ModuleList([mk() for _ in range(share_quant_resi)]))


class _MultiScaleBase(nn.Module):
    """host logic shared by VectorQuantizer2 and LFQ (descriptor, Phi stacking, EMA, usages)."""

    sync_usages: bool = False
    record_hit = record_hit_property

    def _phi_params(self):
        mods = self.quant_resi.modules_list()
        if len(mods) == 0 or not isinstance(mods[0], Phi):
            return None, None, 0
        w = torch.stack([m.weight for m in mods])
        b = torch.stack([m.bias for m in mods])
        return w, b, len(mods)

    def _phi_map(self, SN: int) -> List[int]:
        if SN == 1:
            return [0]  # quant.py:110-111: quant_resi[0]  (at 0.0 every container maps to module 0)
        return [self.quant_resi.index_of(si / (SN - 1)) for si in range(SN)]

    def _n_quantizers(self, B: int, dropout, device, require_dropout: bool) -> Optional[torch.Tensor]:
        """quant.py:79-86 / lookup_free_quantize.py:167-174 (the reference builds it on the CPU)."""
        SN = len(self.v_patch_nums)
        if not self.training:
            return None
        if dropout is None:
            if require_dropout:
                raise TypeError("'NoneType' object is not subscriptable")  # lookup_free_quantize.py:171
            return None
        nq = torch.ones((B,)) * (SN + 1)
        n_dropout = int(B * self.codebook_drop)
        nq[:n_dropout] = dropout[:n_dropout].to(nq.dtype).cpu() if torch.is_tensor(dropout) else dropout[:n_dropout]
        return nq.to(device, non_blocking=True)

    def _update_usage(self, hist: torch.Tensor, numel_per_channel: float, ret_usages: bool):
        SN = len(self.v_patch_nums)
        margin = _world_size() * numel_per_channel / self.vocab_size * 0.08
        if self.training:
            _allreduce_hist_(hist)
            usage = torch.ops.xqb200.usage_ema_(self.ema_vocab_hit_SV, hist, self._record_hit_dev, margin)
        else:
            usage = (self.ema_vocab_hit_SV >= margin).float().mean(dim=-1) * 100
        if not ret_usages:
            return None
        if self.sync_usages:
            return [float(u) for u in usage.tolist()]
        return list(usage.unbind(0))


    # ===================== feature-map helpers shared by VectorQuantizer2 and LFQ =====================
    def _decode_desc(self, B: int):
        """descriptor for building f_hat at the module's scales from codes or feature maps, which are used as they are
        (no channel normalisation)."""
        H = W = self.v_patch_nums[-1]
        d, w, b, pns = self._desc(B, H, W)
        d.channel_norm = 0
        return d, w, b, pns

    def _embed_steps(self, hs, si0: int, f_hat, want_scales: bool, want_next: bool):
        """scales [si0, si0+len(hs)) of  f_hat += Phi_si(bicubic_up(h_si))  in ONE fused kernel (xq_ms_embed)."""
        B = hs[0].shape[0]
        d, w, b, pns = self._decode_desc(B)
        for k, h in enumerate(hs):
            want = (B, self.Cvae, pns[si0 + k], pns[si0 + k])
            if tuple(h.shape) != want:
                raise ValueError(f"scale {si0 + k}: expected a feature map of shape {want}, got {tuple(h.shape)}")
        h_all = torch.cat([h.detach().to(torch.float32).reshape(-1) for h in hs])
        return ops.ms_embed(h_all, w, b, d, si0, si0 + len(hs), f_hat, want_scales, want_next)

    def embed_to_fhat(self, ms_h_BChw: List[torch.Tensor], all_to_max_scale=True, last_one=False):
        """quant.py:148-180 / lookup_free_quantize.py:311-343: per-scale feature maps -> cumulative f_hat(s)."""
        SN = len(self.v_patch_nums)
        if all_to_max_scale:
            if len(ms_h_BChw) != SN:
                raise ValueError(f"expected {SN} feature maps, got {len(ms_h_BChw)}")
            out, fs, _ = self._embed_steps(list(ms_h_BChw), 0, None, want_scales=not last_one, want_next=False)
            return out if last_one else list(fs.unbind(0))
        # experimental branch of the reference (f_hat grows with the scale; quant.py:167-179) -- library ops
        ls_f_hat_BChw = []
        B = ms_h_BChw[0].shape[0]
        f_hat = ms_h_BChw[0].new_zeros(B, self.Cvae, self.v_patch_nums[0], self.v_patch_nums[0], dtype=torch.float32)
        for si, pn in enumerate(self.v_patch_nums):
            f_hat = F.interpolate(f_hat, size=(pn, pn), mode='bicubic')
            h_BChw = self.quant_resi[si / (SN - 1)](ms_h_BChw[si])
            f_hat.add_(h_BChw)
            if last_one:
                ls_f_hat_BChw = f_hat
            else:
                ls_f_hat_BChw.append(f_hat)
        return ls_f_hat_BChw

    def get_next_autoregressive_input(self, si: int, SN: int, f_hat: torch.Tensor, h_BChw: torch.Tensor):
        """quant.py:247-258 / lookup_free_quantize.py:404-415: one VAR inference step; f_hat is updated in place.
        -> (f_hat, area-pooled f_hat at the next scale)  or  (f_hat, f_hat) at the last scale."""
        if (SN != len(self.v_patch_nums) or f_hat.dtype != torch.float32 or not f_hat.is_contiguous()
                or not f_hat.is_cuda):
            HW = self.v_patch_nums[-1]                     # unusual call: keep the reference's op sequence
            if si != SN - 1:
                h = self.quant_resi[si / (SN - 1)](F.interpolate(h_BChw, size=(HW, HW), mode='bicubic'))
                f_hat.add_(h)
                pn = self.v_patch_nums[si + 1]
                return f_hat, F.interpolate(f_hat, size=(pn, pn), mode='area')
            f_hat.add_(self.quant_resi[si / (SN - 1)](h_BChw))
            return f_hat, f_hat
        _, _, nxt = self._embed_steps([h_BChw], si, f_hat, want_scales=False, want_next=si != SN - 1)
        return f_hat, (nxt if si != SN - 1 else f_hat)

    # ===================== inference (VectorQuantizer2 / LFQ) =====================
    def _codebook(self) -> Optional[torch.Tensor]:
        """the codebook the kernels read: None for LFQ, whose codes are +-scaler per bit; VectorQuantizer2 returns its
        embedding."""
        return None

    def f_to_idxBl_or_fhat(self, f_BChw: torch.Tensor, to_fhat: bool,
                           v_patch_nums: Optional[Sequence[Union[int, Tuple[int, int]]]] = None):
        """quant.py:182-223 / lookup_free_quantize.py:345-380: list over scales of idx [B, pn*pn] (int64) or cumulative
        f_hat [B,C,H,W]."""
        B, Cc, H, W = f_BChw.shape
        pns = [pn if isinstance(pn, int) else pn[0] for pn in (v_patch_nums or self.v_patch_nums)]
        d, w, b, pns = self._desc(B, H, W, pns)
        _, idx_all, fs = ops.ms_lookup(f_BChw.detach(), self._codebook(), w, b, d, want_fhat_scales=to_fhat)
        if to_fhat:
            return list(fs.unbind(0))
        return ops.split_scales(idx_all, B, pns)

    def idx_to_fhat(self, gt_ms_idx_Bl: List[torch.Tensor], last_one=True):
        """token lists -> f_hat (fused decode kernel; used by VQModel.decode_tokens)."""
        d, w, b, _ = self._decode_desc(gt_ms_idx_Bl[0].shape[0])
        idx_all = torch.cat([t.reshape(-1) for t in gt_ms_idx_Bl]).to(torch.int64)
        out, fs, _ = ops.ms_decode(idx_all, self._codebook(), w, b, d, want_out=last_one, want_fhat_scales=not last_one)
        return out if last_one else list(fs.unbind(0))

    # ===================== idxBl_to_var_input: only used in VAR training =====================
    def idxBl_to_var_input(self, gt_ms_idx_Bl: List[torch.Tensor]) -> torch.Tensor:
        """quant.py:226-244 / lookup_free_quantize.py:383-401 -> [B, sum_{si>=1} pn^2, C] float32 (None for a single
        scale).  The reference's LFQ version reads a non-existent self.embedding; here LFQ uses its BSQ codes +-scaler[si],
        which is what indices_to_bits(idx, si) yields."""
        SN = len(self.v_patch_nums)
        if SN < 2:
            return None
        B = gt_ms_idx_Bl[0].shape[0]
        d, w, b, pns = self._decode_desc(B)
        lists = list(gt_ms_idx_Bl)
        if len(lists) < SN:  # the last scale's tokens are not needed for teacher forcing
            lists = lists + [torch.zeros(B, pns[-1] ** 2, dtype=torch.int64, device=lists[0].device)]
        idx_all = torch.cat([t.reshape(-1) for t in lists]).to(torch.int64)
        _, _, var = ops.ms_decode(idx_all, self._codebook(), w, b, d, want_out=False, want_var_input=True)
        return var


class VectorQuantizer2(_MultiScaleBase):
    # VQGAN originally use beta=1.0, never tried 0.25; SD seems using 0.25
    def __init__(
            self, vocab_size, Cvae, using_znorm=True, beta: float = 0.25,
            default_qresi_counts=0, v_patch_nums=None, quant_resi=0.5, share_quant_resi=4,
            num_latent_tokens=256, codebook_drop=0.0,
    ):
        super().__init__()
        self.vocab_size: int = vocab_size
        self.Cvae: int = Cvae
        self.using_znorm: bool = using_znorm
        self.v_patch_nums: Tuple[int] = v_patch_nums
        self.num_latent_tokens = num_latent_tokens

        self.quant_resi_ratio = quant_resi
        self.quant_resi = build_quant_resi(Cvae, quant_resi, share_quant_resi, default_qresi_counts, self.v_patch_nums)

        self.register_buffer('ema_vocab_hit_SV', torch.full((len(self.v_patch_nums), self.vocab_size), fill_value=0.0))
        self.register_buffer('_record_hit_dev', torch.zeros(2, dtype=torch.int64), persistent=False)

        self.beta: float = beta
        self.embedding = nn.Embedding(self.vocab_size, self.Cvae)
        self.codebook_drop = codebook_drop

        self.embedding.weight.data.uniform_(-1.0 / self.vocab_size, 1.0 / self.vocab_size)
        if self.using_znorm:
            self.embedding.weight.data = F.normalize(self.embedding.weight.data, p=2, dim=-1)

        self.prog_si = -1  # progressive training: not supported (same as the reference)

    def eini(self, eini):
        if eini > 0:
            nn.init.trunc_normal_(self.embedding.weight.data, std=eini)
        elif eini < 0:
            self.embedding.weight.data.uniform_(-abs(eini) / self.vocab_size, abs(eini) / self.vocab_size)

    def extra_repr(self) -> str:
        return f'{self.v_patch_nums}, znorm={self.using_znorm}, beta={self.beta}  |  S={len(self.v_patch_nums)}, quant_resi={self.quant_resi_ratio}'

    def _desc(self, B, H, W, patch_nums=None):
        pns = list(patch_nums if patch_nums is not None else self.v_patch_nums)
        w, b, K = self._phi_params()
        SN = len(pns)
        pmap = self._phi_map(SN) if K else [-1] * SN
        mode = C.XQ_MS_VQ_ZNORM if self.using_znorm else C.XQ_MS_VQ_L2
        d = C.make_ms_desc(B, self.Cvae, H, W, self.vocab_size, K, pns, pmap, mode,
                           resi_ratio=abs(self.quant_resi_ratio), beta=self.beta, loss_div_sn_all=False)
        return d, w, b, pns

    def _codebook(self):
        return self.embedding.weight.data

    # ===================== `forward` is only used in VAE training =====================
    def forward(self, f_BChw: torch.Tensor, ret_usages=False, dropout=None):
        """-> (f_hat, usages|None, mean_vq_loss, mean_commit_loss, 0)   (quant.py:64-144)"""
        if f_BChw.dtype != torch.float32:
            f_BChw = f_BChw.float()
        B, Cc, H, W = f_BChw.shape
        d, w, b, pns = self._desc(B, H, W)
        nq = self._n_quantizers(B, dropout, f_BChw.device, require_dropout=False)
        f_hat, vq, commit, _ent, idx_all, hist = ops.ms_forward(f_BChw, self.embedding.weight, w, b, nq, d,
                                                               want_hist=True)
        usages = self._update_usage(hist, f_BChw.numel() / f_BChw.shape[1], ret_usages)
        self.last_idx_Bl = ops.split_scales(idx_all, B, pns)
        return f_hat, usages, vq, commit, 0
