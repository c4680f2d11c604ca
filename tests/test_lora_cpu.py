"""LoRA tuning of the DINOv2 encoder / decoder (imagefolder_b200/dino_enc/lora.py), on the CPU: peft 0.13.0's module names,
state_dict keys, initialisation and trainable set for the reference's 'lora' and 'lora_unfreeze_patch_embed', the fp32
module path against 'full', finetine after a 'full' checkpoint, the state_dict round trip, the EMA copy's names, and the
argument refusals of the two LoRA GEMM entry points."""
import copy
import ctypes
import math

import pytest
import torch
import torch.nn as nn

from imagefolder_b200.dino_enc import DINOv2Decoder, DINOv2Encoder
from imagefolder_b200.dino_enc import lora

KW = {'img_size': 56, 'patch_size': 14, 'drop_path_rate': 0.0}      # 4 x 4 patch grid: small, every code path of ViT-S
DEPTH = 12
VIT_S = 'vit_small_patch14_dinov2.lvd142m'
P = 'model.base_model.model.'


def _enc(method, seed=0, **kw):
    torch.manual_seed(seed)
    return DINOv2Encoder(num_latent_tokens=4, model_name=VIT_S, model_kwargs=dict(KW), pretrained=False, tuning_method=method,
                         **kw)


def _dec(method, seed=0):
    torch.manual_seed(seed)
    return DINOv2Decoder(num_latent_tokens=4, model_name=VIT_S, model_kwargs=dict(KW), pretrained=False, tuning_method=method)


def _lora_keys(prefix, r_in=384, hidden=1536):
    keys = {}
    for i in range(DEPTH):
        for fc, (o, n) in (("fc1", (hidden, r_in)), ("fc2", (r_in, hidden))):
            b = f"{prefix}blocks.{i}.mlp.{fc}."
            keys[b + "base_layer.weight"] = (o, n)
            keys[b + "base_layer.bias"] = (o,)
            keys[b + "lora_A.default.weight"] = (8, n)
            keys[b + "lora_B.default.weight"] = (o, 8)
    return keys


def _expected_keys(full_sd, saved):
    """peft's naming applied to the 'full' model's state_dict: `model.` -> `model.base_model.model.`, mlp.fc1 / fc2 through
    base_layer plus their adapters, each saved module as original_module + modules_to_save.default"""
    out = {}
    for k, v in full_sd.items():
        if not k.startswith("model."):
            out[k] = tuple(v.shape)
            continue
        rest = k[len("model."):]
        mod, _, leaf = rest.rpartition(".")
        if ".mlp.fc" in mod:
            continue
        if mod in saved:
            out[f"{P}{mod}.original_module.{leaf}"] = tuple(v.shape)
            out[f"{P}{mod}.modules_to_save.default.{leaf}"] = tuple(v.shape)
        else:
            out[P + rest] = tuple(v.shape)
    out.update(_lora_keys(P))
    return out


@pytest.mark.parametrize("method,saved", [("lora", {"norm"}),
                                          ("lora_unfreeze_patch_embed", {"norm", "patch_embed.proj"})])
@pytest.mark.parametrize("side", ["encoder", "decoder"])
def test_state_dict_keys_follow_peft(side, method, saved):
    build = _enc if side == "encoder" else _dec
    full = {k: v for k, v in build("full").state_dict().items()}
    m = build(method)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    if side == "decoder":
        saved = saved - {"patch_embed.proj"}                # parameter-free in the decoder: no keys at all
    assert got == _expected_keys(full, saved)
    for k in ("model.base_model.model.blocks.11.mlp.fc2.lora_B.default.weight", "model.base_model.model.blocks.0.mlp.fc1.base_layer.bias",
              "model.base_model.model.norm.original_module.weight", "model.base_model.model.norm.modules_to_save.default.bias",
              "model.base_model.model.blocks.5.attn.qkv.weight", "model.base_model.model.pos_embed"):
        assert k in got, k
    if side == "decoder":
        assert not any(".patch_embed.proj" in k for k in got)


@pytest.mark.parametrize("method", ["lora", "lora_unfreeze_patch_embed"])
def test_trainable_set(method, capsys):
    m = _enc(method)
    trainable = {n for n, p in m.named_parameters() if p.requires_grad}
    want = {k for k in _lora_keys(P) if ".lora_" in k}
    want |= {P + "norm.modules_to_save.default.weight", P + "norm.modules_to_save.default.bias"}
    if method == "lora_unfreeze_patch_embed":
        want |= {P + "patch_embed.proj.modules_to_save.default.weight", P + "patch_embed.proj.modules_to_save.default.bias"}
    want |= {"latent_tokens", "latent_pos_embed"}           # outside the wrapped ViT: untouched
    assert trainable == want
    # peft's one-line report, printed by the constructor
    n_train = sum(p.numel() for n, p in m.model.named_parameters() if p.requires_grad)
    n_all = sum(p.numel() for p in m.model.parameters())
    line = f"trainable params: {n_train:,d} || all params: {n_all:,d} || trainable%: {100 * n_train / n_all:.4f}"
    m.model.print_trainable_parameters()
    assert capsys.readouterr().out.strip().splitlines()[-1] == line


def test_decoder_keeps_its_own_parameters_trainable():
    m = _dec("lora")
    for name in ("mask_token", "latent_pos_embed", "to_pixel.model.weight", "to_pixel.model.bias"):
        assert dict(m.named_parameters())[name].requires_grad, name
    assert not dict(m.named_parameters())[P + "blocks.0.mlp.fc1.base_layer.weight"].requires_grad


def test_modules_follow_peft():
    m = _enc("lora")
    assert isinstance(m.model, lora.PeftModel) and isinstance(m.model.base_model, lora.LoraModel)
    vit = m.model.base_model.model
    assert m.model.blocks is vit.blocks and m.model.patch_embed is vit.patch_embed     # peft's attribute fall-through
    assert m.model._pos_embed.__self__ is vit
    fc1 = vit.blocks[3].mlp.fc1
    assert isinstance(fc1, lora.Linear) and isinstance(fc1.base_layer, nn.Linear)
    assert fc1.weight is fc1.base_layer.weight and fc1.bias is fc1.base_layer.bias
    assert isinstance(fc1.lora_dropout["default"], nn.Identity)
    assert fc1.scaling == {"default": 1.0} and fc1.r == {"default": 8}
    assert not fc1.lora_B["default"].weight.any()
    # kaiming-uniform with a = sqrt(5): U(-1/sqrt(fan_in), 1/sqrt(fan_in))
    a = fc1.lora_A["default"].weight.detach()
    bound = 1.0 / math.sqrt(a.shape[1])
    assert float(a.abs().max()) <= bound and float(a.abs().max()) > 0.9 * bound
    assert sorted(m.model.base_model.targeted_module_names) == sorted(
        f"blocks.{i}.mlp.fc{j}" for i in range(DEPTH) for j in (1, 2))
    norm = vit.norm
    assert isinstance(norm, lora.ModulesToSaveWrapper) and not norm.original_module.weight.requires_grad
    assert torch.equal(norm.original_module.weight, norm.modules_to_save["default"].weight)
    assert norm.modules_to_save["default"].weight is not norm.original_module.weight
    # peft matches modules_to_save with str.endswith: the parameter-free q_norm / k_norm / fc_norm are wrapped too
    assert isinstance(vit.blocks[0].attn.q_norm, lora.ModulesToSaveWrapper) and isinstance(vit.fc_norm, lora.ModulesToSaveWrapper)
    assert not isinstance(vit.norm_pre, lora.ModulesToSaveWrapper)


def test_lora_config_rank_and_alpha():
    m = _enc("lora", tuning_kwargs={"r": 16, "lora_alpha": 32, "lora_dropout": 0.1})
    fc2 = m.model.blocks[0].mlp.fc2
    assert fc2.scaling["default"] == 2.0 and fc2.lora_A["default"].weight.shape == (16, 1536)
    assert isinstance(fc2.lora_dropout["default"], nn.Dropout) and fc2.lora_dropout["default"].p == 0.1


def _wrapped(full, method="lora"):
    """a copy of `full` with LoRA added (the constructors draw the adapters before the latent tokens: other values)"""
    m = copy.deepcopy(full)
    m.finetine(method)
    return m


def test_zero_lora_b_reproduces_full_model_bit_for_bit():
    torch.manual_seed(1)
    x = torch.randn(2, 3, 56, 56)
    full_e, full_d = _enc("full").eval(), _dec("full").eval()
    lora_e, lora_d = _wrapped(full_e).eval(), _wrapped(full_d).eval()
    with torch.no_grad():
        h_full, h_lora = full_e(x), lora_e(x)
        assert torch.equal(h_full, h_lora)
        assert torch.equal(full_d(h_full), lora_d(h_lora))


def test_nonzero_adapter_matches_explicit_formula():
    """with lora_B != 0 the module path is base(x) + B(A(x)) * scaling in every fc1 / fc2"""
    ref = _enc("full").eval()
    e = _wrapped(ref)
    torch.manual_seed(2)
    for mod in e.modules():
        if isinstance(mod, lora.Linear):
            nn.init.normal_(mod.lora_B["default"].weight, std=0.02)
    for blk, rblk in zip(e.model.blocks, ref.model.blocks):
        for name in ("fc1", "fc2"):
            f, rf = getattr(blk.mlp, name), getattr(rblk.mlp, name)
            rf.weight.data += f.scaling["default"] * (f.lora_B["default"].weight @ f.lora_A["default"].weight)
    x = torch.randn(2, 3, 56, 56)
    with torch.no_grad():
        torch.testing.assert_close(e(x), ref(x), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("method", ["lora", "lora_unfreeze_patch_embed"])
def test_finetine_after_full_checkpoint(method):
    src = _enc("full", seed=3)
    ckpt = src.state_dict()
    e = _enc("full", seed=4)
    e.load_state_dict(ckpt)
    e.finetine(method)
    sd = e.state_dict()
    assert set(sd) == set(_enc(method).state_dict())
    vit = e.model.base_model.model
    for k, v in ckpt.items():
        if k.startswith("model.blocks.") and ".mlp.fc" in k:
            k2 = P + k[len("model."):].replace(".weight", ".base_layer.weight").replace(".bias", ".base_layer.bias")
            assert torch.equal(sd[k2], v), k2
    assert torch.equal(vit.norm.modules_to_save["default"].weight, ckpt["model.norm.weight"])
    x = torch.randn(1, 3, 56, 56)
    with torch.no_grad():
        assert torch.equal(e.eval()(x), src.eval()(x))
    d = _dec("full")
    d.finetine(method)
    assert not any(".patch_embed.proj" in k for k in d.state_dict())


def test_state_dict_round_trip():
    a = _enc("lora", seed=5)
    for p in a.parameters():
        if p.requires_grad:
            p.data.add_(torch.randn_like(p) * 0.01)
    b = _enc("lora", seed=6)
    b.load_state_dict(a.state_dict())
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb), ka
    x = torch.randn(1, 3, 56, 56)
    with torch.no_grad():
        assert torch.equal(a.eval()(x), b.eval()(x))


def test_ema_copy_gets_the_same_parameter_names():
    """the trainer deep-copies the EMA model before `finetune`: only the same call on the copy gives it the LoRA names"""
    model = _enc("full")
    ema = copy.deepcopy(model)
    model.finetine("lora")
    assert set(dict(ema.named_parameters())) != set(dict(model.named_parameters()))
    ema.finetine("lora")
    assert list(dict(ema.named_parameters())) == list(dict(model.named_parameters()))


def test_lat_lora_and_unknown_methods_raise():
    with pytest.raises(NotImplementedError, match="LatentLoRALinear"):
        _enc("lat_lora")
    with pytest.raises(NotImplementedError, match="LatentLoRALinear"):
        _enc("full").finetine("lat_lora")
    with pytest.raises(NotImplementedError):
        _dec("dora")


# ---- C ABI: argument refusals of the LoRA GEMM entry points (no device work) -----------------------------------------------
XQ_ERR_ARG, XQ_ERR_CUDA = -1, -3
PTR = 1 << 20                              # non-null dummy device pointers, 256-byte aligned; never dereferenced
M, N, K = 256, 256, 128


def _fwd(L, u=PTR, bl=PTR, R=8, x=PTR):
    return L.xq_vit_fc1_lora_gelu_fwd(x, PTR, u, bl, ctypes.cast(PTR, ctypes.POINTER(ctypes.c_float)), PTR, PTR, M, N, K, R, None)


def _bwd(L, v=PTR, a2t=PTR, R=8, d_bias=PTR):
    f32 = lambda p: ctypes.cast(p, ctypes.POINTER(ctypes.c_float)) if p else None
    return L.xq_vit_fc2_lora_dgelu_bwd(PTR, PTR, v, a2t, PTR, f32(PTR), PTR, f32(d_bias), M, N, K, R, None)


@pytest.mark.skipif(torch.cuda.is_available(), reason="dummy device pointers must never reach a real GPU")
@pytest.mark.parametrize("call", [_fwd, _bwd])
def test_lora_entry_points_refuse_bad_arguments(call):
    from imagefolder_b200 import _capi
    L = _capi.lib()
    for kw in ({"R": 0}, {"R": 4}, {"R": 72}, {"R": 12}, {"R": -8}):
        assert call(L, **kw) == XQ_ERR_ARG, kw
    first, second = ("u", "bl") if call is _fwd else ("v", "a2t")
    for kw in ({first: None}, {second: None}, {first: PTR + 8}, {second: PTR + 2}):
        assert call(L, **kw) == XQ_ERR_ARG, kw
    if call is _fwd:
        assert call(L, x=None) == XQ_ERR_ARG
    else:
        assert call(L, d_bias=None) == XQ_ERR_ARG
    # valid arguments pass every check and fail only at the first CUDA call (no device here)
    for R in (8, 16, 64):
        assert call(L, R=R) == XQ_ERR_CUDA
