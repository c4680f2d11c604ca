"""Goldens of the giant (SwiGLU MLP, D = 1536) and four-register DINOv2 backbones from the REFERENCE'S OWN modules (CPU, fp32).

    XQ_REFERENCE=<checkout> python tests/golden/make_vit_giant_golden.py     # writes tests/golden/vit_giant_*.npz, vit_reg4_*.npz

Same recipe as make_vit_golden.py (whose timm stand-ins and name-seeded weights it reuses): VQModel.encode / decode of the
reference with dino_enc/dinov2.py and the vendored vision_transformer.py (vit_giant_patch14_dinov2 :2925,
vit_*_reg4_dinov2 :2942-2995).  One more timm piece is a stand-in here: SwiGLUPacked = GluMlp(act_layer=nn.SiLU,
gate_last=False) from timm 1.0.9's published code (fc1 -> chunk(2) -> act(x1) * x2 -> norm (Identity) -> fc2).

The giant cases keep the full width and cut the depth to GIANT_DEPTH blocks (the registry entry's kwargs override its
defaults, as timm's do).  vit_reg4_abs records that the reference's forward fails for a reg4 backbone with
abs_pos_embed=True: lvl1LC is sized for one prefix token (dinov2.py:91, 98, 266).
"""
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_vit_golden as mvg  # noqa: E402
from vit_det_init import golden_inputs  # noqa: E402

GIANT_DEPTH = 2
TOKEN_STRIDE = {"vit_giant_vq": 16, "vit_giant_relpos": 16, "vit_reg4_relpos": 4}


class GluMlp(nn.Module):
    """timm.layers.GluMlp (1.0.9); SwiGLUPacked is this with act_layer=nn.SiLU, gate_last=False."""

    def __init__(self, in_features, hidden_features=None, out_features=None, act_layer=nn.Sigmoid, norm_layer=None, bias=True,
                 drop=0.0, use_conv=False, gate_last=True):
        super().__init__()
        out_features = out_features or in_features
        hidden_features = hidden_features or in_features
        assert hidden_features % 2 == 0
        self.chunk_dim = -1
        self.gate_last = gate_last
        self.fc1 = nn.Linear(in_features, hidden_features, bias=bias)
        self.act = act_layer()
        self.drop1 = nn.Dropout(drop)
        self.norm = norm_layer(hidden_features // 2) if norm_layer is not None else nn.Identity()
        self.fc2 = nn.Linear(hidden_features // 2, out_features, bias=bias)
        self.drop2 = nn.Dropout(drop)

    def forward(self, x):
        x = self.fc1(x)
        x1, x2 = x.chunk(2, dim=self.chunk_dim)
        x = x1 * self.act(x2) if self.gate_last else self.act(x1) * x2
        return self.drop2(self.fc2(self.norm(self.drop1(x))))


def SwiGLUPacked(*args, **kwargs):
    kwargs["act_layer"] = nn.SiLU
    return GluMlp(*args, gate_last=False, **kwargs)


def create_model(model_name, pretrained=False, **kwargs):
    if "giant" in model_name:
        kwargs.setdefault("depth", GIANT_DEPTH)
    return mvg.create_model(model_name, pretrained=False, **kwargs)


_install_timm = mvg.install_stand_ins


def install_stand_ins():
    _install_timm()
    sys.modules["timm.layers"].SwiGLUPacked = SwiGLUPacked
    sys.modules["timm.models"].create_model = create_model


mvg.install_stand_ins = install_stand_ins         # make_vit_golden.build_reference installs these before importing the reference


def build_reference(cfg):
    return mvg.build_reference(cfg)


GIANT = "vit_giant_patch14_dinov2.lvd142m"
REG4 = "vit_small_patch14_reg4_dinov2.lvd142m"
BASE = dict(codebook_size=8192, codebook_embed_dim=32, v_patch_nums=[16], num_latent_tokens=256, product_quant=1)
CASES = {
    "vit_giant_vq": dict(BASE, abs_pos_embed=True, encoder_model=GIANT, decoder_model=GIANT),        # S = 513 / 514
    "vit_giant_relpos": dict(BASE, abs_pos_embed=False, encoder_model=GIANT, decoder_model=GIANT),   # S = 513 / 513
    "vit_reg4_relpos": dict(BASE, abs_pos_embed=False, encoder_model=REG4, decoder_model=REG4),      # S = 517 / 517
}
FAILING = {"vit_reg4_abs": dict(BASE, abs_pos_embed=True, encoder_model=REG4, decoder_model=REG4)}


def main():
    common = dict(mvg.COMMON)
    for name, c in CASES.items():
        cfg = dict(common, **c)
        model = build_reference(cfg)
        side = int(math.sqrt(model.config.num_latent_tokens))
        x, q = golden_inputs(cfg["codebook_embed_dim"], side)
        with torch.no_grad():
            tok = model.encoder(x)
            h = model.encode(x)
            dec = model.decode(q)
        st = TOKEN_STRIDE[name]
        np.savez_compressed(os.path.join(HERE, name + ".npz"), cfg_json=np.array(repr(cfg)), giant_depth=GIANT_DEPTH,
                            token_stride=st, x_sum=np.float64(x.double().sum()), q_sum=np.float64(q.double().sum()),
                            q_shape=np.array(q.shape), tok_sub=tok[:, ::st].numpy(), tok_sum=np.float64(tok.double().sum()),
                            tok_abs=np.float64(tok.double().abs().sum()), h_sub=h.flatten(2)[:, :, ::4].numpy(),
                            h_shape=np.array(h.shape), h_sum=np.float64(h.double().sum()),
                            dec_sub=dec[:, :, ::4, ::4].numpy(), dec_sum=np.float64(dec.double().sum()),
                            dec_abs=np.float64(dec.double().abs().sum()),
                            enc_S=model.encoder.num_img_tokens + model.encoder.num_prefix_tokens + model.encoder.num_latent_tokens)
        print(name, "tokens", tuple(tok.shape), "h", tuple(h.shape), "dec", tuple(dec.shape))
    for name, c in FAILING.items():
        cfg = dict(common, **c)
        model = build_reference(cfg)
        x, q = golden_inputs(cfg["codebook_embed_dim"], int(math.sqrt(model.config.num_latent_tokens)))
        errors = []
        for what, fn in (("encode", lambda: model.encode(x)), ("decode", lambda: model.decode(q))):
            try:
                with torch.no_grad():
                    fn()
                errors.append("")
            except Exception as e:          # the recorded outcome: which exception, and its message
                errors.append(f"{type(e).__name__}: {e}")
        np.savez_compressed(os.path.join(HERE, name + ".npz"), cfg_json=np.array(repr(cfg)), encode_error=np.array(errors[0]),
                            decode_error=np.array(errors[1]))
        print(name, errors)


if __name__ == "__main__":
    main()
