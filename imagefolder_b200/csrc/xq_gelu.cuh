// xq_gelu.cuh -- the exact-erf GELU, SiLU / SwiGLU and their derivatives as ONE set of device functions, shared by the
// stand-alone element-wise kernels (vit_kernels.cu) and the fused GELU GEMM epilogues (gemm_kernel.cu), so that both paths
// produce the same bits.
// Reference ops: nn.GELU() (erf form) inside timm's Mlp, tokenizer/tokenizer_image/dino_enc/vision_transformer.py:336-339, and
// nn.SiLU inside timm's SwiGLUPacked (GluMlp, gate_last=False) of the giant backbones, vision_transformer.py:2925-2937.
#pragma once
#include <cuda_runtime.h>

namespace xqv {

__device__ __forceinline__ float rcp_fast(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float ex2_fast(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// gelu(x) = x/2 * (1 + erf(x/sqrt2)) with erf(|z|) = 1 - r, r = (1 + a1|z| + ... + a6|z|^6)^-16 (A&S 7.1.28):
//   gelu(x) = h + |h| * (1 - r) = (h + |h|) - |h| * r ,  h = x/2.
// The 1/sqrt2 of z is folded into the coefficients (b_k = a_k * 2^(-k/2)) and the sign handling into the abs/neg operand
// modifiers, which takes 3 instructions off the previous form (the kernel is instruction-issue bound, not HBM bound).
__device__ __forceinline__ float gelu_f(float x) {
    const float a = fabsf(x);
    float p = fmaf(a, 5.382975000e-06f, 4.889063564e-05f);
    p = fmaf(p, a, 3.800357500e-05f);
    p = fmaf(p, a, 3.277626324e-03f);
    p = fmaf(p, a, 2.114100615e-02f);
    p = fmaf(p, a, 4.986734697e-02f);
    p = fmaf(p, a, 1.0f);
    p = p * p; p = p * p; p = p * p; p = p * p;
    const float h = 0.5f * x;
    return fmaf(-fabsf(h), rcp_fast(p), h + fabsf(h));
}
// gelu'(x) = Phi(x) + x phi(x).  Both need exp(-x^2/2): with A&S 7.1.26,  erf(z) = 1 - (a1 t + ... + a5 t^5) exp(-z^2),
// t = 1/(1 + p z), the SAME exponential serves Phi and phi (z = |x|/sqrt2), so the derivative costs one ex2 + one rcp +
// ~14 FP32 instructions (the 7.1.28 erf + a separate exp used before: ~20).  |abs err| 3e-7.
__device__ __forceinline__ float dgelu_f(float x) {
    const float ax = fabsf(x);
    const float t = rcp_fast(fmaf(ax, 0.23164189f, 1.0f));             // p / sqrt2 = 0.3275911 / 1.41421356
    float q = fmaf(t, 1.061405429f, -1.453152027f);
    q = fmaf(q, t, 1.421413741f);
    q = fmaf(q, t, -0.284496736f);
    q = fmaf(q, t, 0.254829592f);
    const float e = ex2_fast(x * x * -0.72134752044448170f);            // exp(-x^2 / 2)
    const float pe = q * t * e;                                          // 1 - erf(|x| / sqrt2)
    const float half = fmaf(-0.5f, pe, 0.5f);                           // Phi(|x|) - 1/2
    return fmaf(x * 0.3989422804014327f, e, 0.5f + copysignf(half, x));
}

// silu(x) = x / (1 + exp(-x)) with the accurate expf and an IEEE division: the formula and the fp32 operations of
// torch.nn.functional.silu's CUDA kernel.  Large negative x: exp overflows to +inf and the result is -0; x = -inf gives NaN,
// as torch does.
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
// silu'(x) = s (1 + x (1 - s)), s = sigmoid(x) = 1 / (1 + exp(-x))
__device__ __forceinline__ float dsilu_f(float x) {
    const float s = 1.0f / (1.0f + expf(-x));
    return s * fmaf(x, 1.0f - s, 1.0f);
}
// SwiGLU on one column pair (timm GluMlp, gate_last=False: the first half of fc1's output is the gate):
//   a = gate pre-activation + its bias, c = up pre-activation + its bias;  act = silu(a) * c
__device__ __forceinline__ float swiglu_f(float a, float c) { return silu_f(a) * c; }
// backward of act = silu(a) * c for the incoming gradient g:  d_a = g c silu'(a),  d_c = g silu(a)
__device__ __forceinline__ void dswiglu_f(float g, float a, float c, float &d_a, float &d_c) {
    d_a = g * c * dsilu_f(a);
    d_c = g * silu_f(a);
}

}  // namespace xqv
