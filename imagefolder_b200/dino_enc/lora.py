"""LoRA adapters for the DINOv2 encoder / decoder: the part of peft 0.13.0 that the reference's tuning methods reach.

The reference builds `tuning_method='lora'` and `'lora_unfreeze_patch_embed'` (dino_enc/dinov2.py:54-66, 117-130, 244-250,
295-301) as

    peft.get_peft_model(vit, peft.LoraConfig(target_modules=r".*\\.mlp\\.fc\\d", modules_to_save=[...], r=8))

peft is not vendored in the reference, so this module restates that behaviour, the way vision_transformer.py restates timm:
the module nesting (`PeftModel -> LoraModel -> model`, state-dict prefix `base_model.model.`), the attribute fall-through to
the wrapped ViT, the LoRA `Linear` (`base_layer`, `lora_dropout`, `lora_A`, `lora_B` ModuleDicts keyed by the adapter name
`default`), its initialisation (lora_A kaiming-uniform with a = sqrt(5), lora_B zero, scaling = lora_alpha / r), the
`modules_to_save` wrappers (`original_module` frozen, `modules_to_save.default` a trainable copy that runs the forward) and the
trainable set.  Only what those calls use is built: one adapter, `bias='none'`, default initialisation, nn.Linear targets.

This boundary is parity-unpinned: nothing here is compared against peft itself, which is not installed.  The names and rules
follow peft 0.13.0's published source; tests/test_lora_cpu.py pins them as stated here.

On the fused ViT path (vit_ops.mlp_forward) a LoRA-wrapped fc1 / fc2 pair does not run `Linear.forward`: its rank-r term enters
the wgmma MLP GEMMs as one more K stage (csrc/gemm_kernel.cu).  `Linear.forward` is the path everywhere else (CPU, fp32,
lora_dropout active).
"""
from __future__ import annotations

import copy
import math
import re

import torch.nn as nn

ADAPTER = "default"


class LoraConfig:
    """peft.LoraConfig, the fields the reference sets.  `target_modules` is a regex matched with re.fullmatch against the
    wrapped model's module names; `modules_to_save` entries match every module whose name ends with them (peft's rule)."""

    def __init__(self, target_modules: str, modules_to_save=None, r: int = 8, lora_alpha: int = 8, lora_dropout: float = 0.0,
                 bias: str = "none", init_lora_weights=True):
        if not isinstance(target_modules, str):
            raise NotImplementedError("target_modules: only a regex string is built")
        if bias != "none":
            raise NotImplementedError(f"bias={bias!r}: only 'none' is built")
        if init_lora_weights is not True:
            raise NotImplementedError(f"init_lora_weights={init_lora_weights!r}: only the default initialisation is built")
        if r <= 0:
            raise ValueError(f"r={r}: the rank must be positive")
        self.target_modules, self.modules_to_save = target_modules, list(modules_to_save or [])
        self.r, self.lora_alpha, self.lora_dropout = r, lora_alpha, lora_dropout
        self.bias, self.init_lora_weights = bias, init_lora_weights


class Linear(nn.Module):
    """peft.tuners.lora.Linear around an nn.Linear: base_layer(x) + lora_B(lora_A(lora_dropout(x))) * scaling."""

    def __init__(self, base_layer: nn.Linear, r: int, lora_alpha: int, lora_dropout: float):
        super().__init__()
        self.base_layer = base_layer
        self.in_features, self.out_features = base_layer.in_features, base_layer.out_features
        self.r, self.lora_alpha = {ADAPTER: r}, {ADAPTER: lora_alpha}
        self.scaling = {ADAPTER: lora_alpha / r}
        self.active_adapter = ADAPTER
        self.lora_dropout = nn.ModuleDict({ADAPTER: nn.Dropout(p=lora_dropout) if lora_dropout > 0.0 else nn.Identity()})
        # peft's update_layer order: both Linears built (each draws its default init), then lora_A re-drawn, lora_B zeroed
        self.lora_A = nn.ModuleDict({ADAPTER: nn.Linear(self.in_features, r, bias=False)})
        self.lora_B = nn.ModuleDict({ADAPTER: nn.Linear(r, self.out_features, bias=False)})
        nn.init.kaiming_uniform_(self.lora_A[ADAPTER].weight, a=math.sqrt(5))
        nn.init.zeros_(self.lora_B[ADAPTER].weight)
        w = base_layer.weight
        for d in (self.lora_A, self.lora_B):
            d[ADAPTER].to(w.device, dtype=w.dtype)

    @property
    def weight(self):
        return self.base_layer.weight

    @property
    def bias(self):
        return self.base_layer.bias

    def lora_delta(self, x):
        """lora_B(lora_A(lora_dropout(x))) * scaling"""
        A = self.lora_A[ADAPTER]
        return self.lora_B[ADAPTER](A(self.lora_dropout[ADAPTER](x.to(A.weight.dtype)))) * self.scaling[ADAPTER]

    def forward(self, x):
        result = self.base_layer(x)
        return (result + self.lora_delta(x)).to(result.dtype)


class ModulesToSaveWrapper(nn.Module):
    """peft's modules_to_save wrapper: the original module frozen, a trainable deep copy that runs the forward."""

    def __init__(self, module_to_save: nn.Module):
        super().__init__()
        self.original_module = module_to_save
        self.modules_to_save = nn.ModuleDict({ADAPTER: copy.deepcopy(module_to_save)})
        self.active_adapter = ADAPTER
        self.original_module.requires_grad_(False)

    @property
    def active_module(self) -> nn.Module:
        return self.modules_to_save[self.active_adapter]

    def forward(self, *args, **kwargs):
        return self.active_module(*args, **kwargs)


def active_module(m: nn.Module) -> nn.Module:
    """the module that runs `m`'s forward: the trainable copy when `m` is a modules_to_save wrapper, else `m`"""
    return m.active_module if isinstance(m, ModulesToSaveWrapper) else m


class _FallThrough(nn.Module):
    """peft's attribute chain: what this wrapper does not have is looked up on the module it wraps (`_inner`)."""

    _inner = ""

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            if name == self._inner:
                raise
            return getattr(super().__getattr__(self._inner), name)


class LoraModel(_FallThrough):
    _inner = "model"

    def __init__(self, model: nn.Module, config: LoraConfig):
        super().__init__()
        self.model = model
        self.peft_config = {ADAPTER: config}
        self.targeted_module_names = []
        for key in [k for k, _ in model.named_modules()]:
            if not key:
                continue
            parent_key, _, name = key.rpartition(".")
            parent = model.get_submodule(parent_key)
            target = getattr(parent, name)
            # peft 0.13 tests modules_to_save first, with str.endswith: ['norm'] also matches q_norm, k_norm, fc_norm and
            # patch_embed.norm (parameter-free Identities in these ViTs)
            if any(key.endswith(m) for m in config.modules_to_save):
                if not isinstance(target, ModulesToSaveWrapper):
                    setattr(parent, name, ModulesToSaveWrapper(target))
                continue
            if not re.fullmatch(config.target_modules, key):
                continue
            if not isinstance(target, nn.Linear):
                raise ValueError(f"LoRA target {key}: {type(target).__name__} is not supported, only nn.Linear")
            setattr(parent, name, Linear(target, config.r, config.lora_alpha, config.lora_dropout))
            self.targeted_module_names.append(key)
        if not self.targeted_module_names:
            raise ValueError(f"Target modules {config.target_modules} not found in the base model")
        # peft's _mark_only_adapters_as_trainable (bias='none'), then the saved copies made trainable again
        for n, p in model.named_parameters():
            if "lora_" not in n:
                p.requires_grad = False
        for m in model.modules():
            if isinstance(m, ModulesToSaveWrapper):
                m.active_module.requires_grad_(True)

    def forward(self, *args, **kwargs):
        return self.model(*args, **kwargs)


class PeftModel(_FallThrough):
    _inner = "base_model"

    def __init__(self, model: nn.Module, config: LoraConfig):
        super().__init__()
        self.base_model = LoraModel(model, config)
        self.peft_config = self.base_model.peft_config
        self.active_adapter = ADAPTER

    def forward(self, *args, **kwargs):
        return self.base_model(*args, **kwargs)

    def get_nb_trainable_parameters(self):
        trainable = total = 0
        for p in self.parameters():
            total += p.numel()
            if p.requires_grad:
                trainable += p.numel()
        return trainable, total

    def print_trainable_parameters(self):
        trainable, total = self.get_nb_trainable_parameters()
        print(f"trainable params: {trainable:,d} || all params: {total:,d} || trainable%: {100 * trainable / total:.4f}")


def get_peft_model(model: nn.Module, config: LoraConfig) -> PeftModel:
    """wrap `model` in place (its Linears and saved modules are replaced) and return the PeftModel around it"""
    return PeftModel(model, config)
