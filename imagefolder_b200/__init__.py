"""imagefolder_b200 -- H100-native (sm_90a) hot path of the XQ-GAN / ImageFolder image tokenizer.

Public surface mirrors the reference modules (SURVEY.md section 8b):
    VectorQuantizer, VectorQuantizer2, LFQ, add_perturbation / add_perturb, VQModel, ModelArgs,
    VQ_models
"""
from .latent_perturbation import add_perturb, add_perturbation
from .lookup_free_quantize import LFQ
from .quant import Phi, PhiNonShared, PhiPartiallyShared, PhiShared, VectorQuantizer2
from .vq import VectorQuantizer

__all__ = ["VectorQuantizer", "VectorQuantizer2", "LFQ", "add_perturbation", "add_perturb", "Phi", "PhiShared",
           "PhiPartiallyShared", "PhiNonShared"]
