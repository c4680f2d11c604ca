/*
 * xqb200.h -- C ABI of libxqb200.so: the H100 (sm_90a) quantizer hot path of the XQ-GAN /
 * ImageFolder image tokenizer.
 *
 * The reference (lxa9867/ImageFolder) is pure Python; its "operator boundary" for this path is
 * the nn.Module surface of its quantizers (SURVEY.md section 8b).  Each entry point below replaces
 * the arithmetic of one reference method and is what a binding for that method calls
 * (INTEGRATION.md shows the ctypes stubs; imagefolder_b200/_capi.py is the in-repo binding).
 *
 * Conventions
 *   - plain pointers and sizes only; every tensor pointer is a DEVICE pointer owned by the caller
 *     (PyTorch), contiguous, fp32 unless stated; indices are int64 like torch.long.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises.
 *   - no allocation, no global state: scratch memory is a caller-provided workspace whose size the
 *     matching *_workspace_bytes() call returns; calls are re-entrant across streams when the
 *     workspaces differ.
 *   - return value: 0 = ok, negative = error (xq_strerror()); the Python side maps it to
 *     RuntimeError / ValueError, mirroring the reference's exceptions/asserts.
 *   - tensors named `*_nchw` are [B, C, H*W] exactly as the reference passes them (B,C,H,W
 *     contiguous); "rows" n = b*HW + p follow the reference's 'b c h w -> b h w c' flattening
 *     (xqgan_model.py:750-751).
 */
#ifndef XQB200_H_
#define XQB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XQ_OK 0
#define XQ_ERR_ARG (-1)         /* bad shape / null pointer / unsupported size */
#define XQ_ERR_WORKSPACE (-2)   /* workspace too small */
#define XQ_ERR_CUDA (-3)        /* a CUDA runtime call or launch failed */
#define XQ_ERR_UNSUPPORTED (-4) /* valid in the reference, not built here */

#define XQ_MAX_SCALES 32

const char *xq_strerror(int code);
int xq_abi_version(void);
/* last CUDA error string recorded on this thread by a failed call (for diagnostics) */
const char *xq_last_cuda_error(void);

/* ------------------------------------------------------------------------------------------
 * Single-scale VectorQuantizer   (VQ-4096 / VQ-8192 / VP2-* / RobustTok)
 *   replaces VectorQuantizer.forward           tokenizer/tokenizer_image/xqgan_model.py:745-801
 *            VectorQuantizer.f_to_idxBl_or_fhat                      xqgan_model.py:803-833
 * ------------------------------------------------------------------------------------------ */
size_t xq_vq_workspace_bytes(int B, int C, int HW, int V);

/*
 * Fused normalise -> distance -> argmin -> gather -> normalise -> STE value -> MSE partials
 * -> usage histogram.  The N x V distance matrix is never written to memory.
 *   z_nchw        [B,C,HW]   encoder latent (input of the reference forward)
 *   E             [V,C]      embedding.weight (raw)
 *   codebook_norm 1: rows and codes are L2-normalised first (xqgan_model.py:753-756)
 *   ste_value     1: out = zn + (q - zn)  (forward, :796)   0: out = q  (f_to_idxBl_or_fhat :826-831)
 *   idx           [B*HW]     argmin index per row (first index on ties)
 *   out_nchw      [B,C,HW]
 *   loss          [2]        {vq_loss, commit_loss} = {mse, beta*mse} (:792-793); may be NULL
 *   hist          [V]        += bincount(idx) as float (:774); may be NULL
 */
int xq_vq_forward(const float *z_nchw, const float *E, int B, int C, int HW, int V, int codebook_norm,
                  int ste_value, float beta, int64_t *idx, float *out_nchw, float *loss, float *hist,
                  void *workspace, size_t workspace_bytes, void *stream);

/*
 * Backward of (out, vq_loss, commit_loss) wrt z and E (SURVEY.md Appendix A.3).
 *   g_out_nchw [B,C,HW] or NULL; g_vq / g_commit: device scalars or NULL (treated as 0)
 *   gz_nchw    [B,C,HW]  written;   gE [V,C] overwritten (zeroed, then scatter-added)
 */
int xq_vq_backward(const float *z_nchw, const float *E, const int64_t *idx, const float *g_out_nchw,
                   const float *g_vq, const float *g_commit, int B, int C, int HW, int V, int codebook_norm,
                   float beta, float *gz_nchw, float *gE, void *stream);

/* ------------------------------------------------------------------------------------------
 * Latent perturbation   (RobustTok)
 *   replaces add_perturbation      tokenizer/tokenizer_image/latent_perturbation.py:4-35
 * The two random tensors the reference draws (torch.rand(N) :21, torch.randint(0,delta,(N,)) :22)
 * are INPUTS, so the host keeps the reference's RNG stream.
 * ------------------------------------------------------------------------------------------ */
size_t xq_perturb_workspace_bytes(int B, int C, int HW, int V);
/*   n_perturb = int(B * beta) evaluated by the host (Python double arithmetic, :32)
 *   out_nchw [B,C,HW] = where(b < n_perturb, zn + (normalize(E[sel]) - zn), zq)
 *   sel      [n_perturb*HW] chosen code per perturbed row (may be NULL) */
int xq_perturb_forward(const float *z_nchw, const float *zq_nchw, const float *E, const float *rand_u,
                       const int64_t *rand_j, int B, int C, int HW, int V, int codebook_norm, float alpha,
                       int n_perturb, int delta, float *out_nchw, int64_t *sel, void *workspace,
                       size_t workspace_bytes, void *stream);
/*   g [B,C,HW] -> gz (through the normalisation Jacobian, perturbed samples only), gzq (the rest) */
int xq_perturb_backward(const float *z_nchw, const float *g_nchw, int B, int C, int HW, int codebook_norm,
                        int n_perturb, float *gz_nchw, float *gzq_nchw, void *stream);

/* ------------------------------------------------------------------------------------------
 * Multi-scale residual quantizers (MSVR*, MSBR*)
 *   replaces VectorQuantizer2.forward / f_to_idxBl_or_fhat   tokenizer/tokenizer_image/quant.py:64-223
 *            LFQ.forward / f_to_idxBl_or_fhat    tokenizer/tokenizer_image/lookup_free_quantize.py:149-380
 *            Phi.forward                                                   quant.py:261-268
 * One CTA owns one image: residual, accumulated f_hat and the upsampled code map stay in shared
 * memory across all scales.
 * ------------------------------------------------------------------------------------------ */
#define XQ_MS_VQ_ZNORM 0 /* VectorQuantizer2, using_znorm=True  (argmax cosine)        */
#define XQ_MS_VQ_L2 1    /* VectorQuantizer2, using_znorm=False (argmin L2)            */
#define XQ_MS_BSQ 2      /* LFQ: sign bits, code = +-scaler[si]                        */
/* LFQ(soft_entropy=False): the same quantizer, with the entropy term of entropy_loss (lookup_free_quantize.py:41-79,
 * 220-229), the softmax over all 2^C codes at temperature 0.01, evaluated in closed form instead of the soft path's
 * per-bit approximation.  Per scale si and masked row r (every position of every image b with si < n_quantizers[b]):
 *   q_rk = sigmoid(400 * scaler[si] * x_rk),  x = f (normalised when channel_norm) - f_hat before scale si
 *   sample entropy  S  = mean_r sum_k H_b(q_rk)
 *   codebook entropy Hc = -sum_j a_j log(a_j + 1e-5),  a_j = mean_r prod_k q_rk(bit k of j)  (bits little-endian),
 *     a = A^T Bm over the low floor(C/2) / high bits, contracted in fp32 on the CUDA cores in a fixed order
 *   entropy = mean_si (w_sample S - w_batch Hc) * entropy_weight / (n1 / B)
 * The backward carries the gradient to every image.  Deterministic: no atomics, fixed reduction order.
 * Refusals: C > 16 -> XQ_ERR_UNSUPPORTED (the 2^C code-probability table is kept per scale).  B == 1 is accepted here
 * (the reference module raises for it; imagefolder_b200 mirrors that in Python). */
#define XQ_MS_BSQ_HARD 3

typedef struct {
    int B, C, H, W;       /* f is [B,C,H,W]                                             */
    int V;                /* codebook size (BSQ: 2^C)                                   */
    int K;                /* number of Phi modules (0 = identity)                       */
    int SN;               /* number of scales                                           */
    int mode;             /* XQ_MS_*                                                    */
    int patch_nums[XQ_MAX_SCALES];
    int phi_map[XQ_MAX_SCALES]; /* scale -> Phi index (PhiPartiallyShared, quant.py:279-288) */
    float scaler[XQ_MAX_SCALES]; /* BSQ code magnitude per scale (lookup_free_quantize.py:124-128) */
    float resi_ratio;     /* Phi blend r (quant.py:265)                                 */
    float beta;           /* commit weight                                              */
    int loss_div_sn_all;  /* 0: only vq is divided by SN (quant.py:134)  1: all (LFQ :238-240) */
    int channel_norm;     /* 1: f is L2-normalised over C first (LFQ using_znorm, :153) */
    float entropy_weight, w_sample, w_batch; /* LFQ entropy term                        */
} xq_ms_desc;

size_t xq_ms_workspace_bytes(const xq_ms_desc *d);
size_t xq_ms_saved_bytes(const xq_ms_desc *d); /* bytes of `saved` (forward -> backward) */
int64_t xq_ms_total_tokens(const xq_ms_desc *d); /* sum_si B*pn^2 */

/*
 *   f            [B,C,H,W]
 *   E            [V,C] raw codebook (NULL for BSQ)
 *   phi_w/phi_b  [K,C,C,3,3] / [K,C]
 *   n_quantizers [B] float, scale si contributes to sample b iff si < n_quantizers[b]
 *                (quant.py:79-86,115); NULL = no quantizer dropout
 *   with_losses  0: inference (f_to_idxBl_or_fhat): no masks, no losses
 *   out          [B,C,H,W]  forward: (f_hat - f) + f (quant.py:135); inference: f_hat
 *   idx_all      [sum_si B*pn^2] int64, scale-major, then (b, y, x)
 *   fhat_scales  [SN,B,C,H,W] cumulative f_hat after each scale, or NULL (to_fhat=True lists)
 *   loss         [3] {vq, commit, entropy}
 *   hist         [SN,V] += bincount per scale, or NULL
 *   saved        xq_ms_saved_bytes(): state the backward needs (final masked f_hat, ...)
 * Refusals: XQ_ERR_UNSUPPORTED when one image's working set exceeds 227 KB of shared memory; with losses and `saved`
 * (training), also when the backward's would (it needs more: e.g. C = 32 fits the forward up to a 16 x 16 last
 * scale but the backward only up to 13 x 13), so that a forward never succeeds whose backward is refused.
 */
int xq_ms_forward(const xq_ms_desc *d, const float *f, const float *E, const float *phi_w, const float *phi_b,
                  const float *n_quantizers, int with_losses, float *out, int64_t *idx_all, float *fhat_scales,
                  float *loss, float *hist, void *saved, void *workspace, size_t workspace_bytes, void *stream);

/*
 * Backward wrt f, E, phi_w, phi_b (SURVEY.md Appendix A.2 / A.5).
 *   g_out [B,C,H,W] or NULL; g_vq/g_commit/g_entropy device scalars or NULL
 *   gf [B,C,H,W]; gE [V,C] (NULL for BSQ); gphi_w [K,C,C,3,3]; gphi_b [K,C]  -- all overwritten
 */
int xq_ms_backward(const xq_ms_desc *d, const float *f, const float *E, const float *phi_w, const float *phi_b,
                   const float *n_quantizers, const int64_t *idx_all, const void *saved, const float *g_out,
                   const float *g_vq, const float *g_commit, const float *g_entropy, float *gf, float *gE,
                   float *gphi_w, float *gphi_b, void *workspace, size_t workspace_bytes, void *stream);

/*
 * VAR-side helpers built from the same primitives (quant.py:148-180, 226-258):
 * given token indices per scale, rebuild f_hat (all scales) and the next-scale inputs.
 *   var_input [B, sum_{si>=1} pn_si^2, C] (idxBl_to_var_input) or NULL
 *   fhat_scales [SN,B,C,H,W] or NULL ; out [B,C,H,W] final f_hat or NULL
 */
int xq_ms_decode(const xq_ms_desc *d, const int64_t *idx_all, const float *E, const float *phi_w,
                 const float *phi_b, float *out, float *fhat_scales, float *var_input, void *stream);

/*
 * The same step in FEATURE-MAP form (the VAR generator's per-step loop and the VAE's embed_to_fhat):
 *   VectorQuantizer2.embed_to_fhat(all_to_max_scale=True)  quant.py:148-166   -> si0 = 0, si1 = SN, fhat_scales / out
 *   VectorQuantizer2.get_next_autoregressive_input         quant.py:247-258   -> si1 = si0 + 1, fhat_in = out (in place), next
 *   (LFQ: lookup_free_quantize.py:311-343, 404-415)
 * for si in [si0, si1):  f_hat += Phi_si(bicubic_up(h_si))   (no interpolation at the last scale)
 *   h_all       scales si0..si1-1 packed back to back, each [B,C,pn_si,pn_si] fp32
 *   fhat_in     [B,C,H,W] running f_hat or NULL (= zeros); may alias out
 *   out         [B,C,H,W] f_hat after scale si1-1, or NULL
 *   fhat_scales [si1-si0,B,C,H,W] cumulative f_hat after every scale, or NULL
 *   next        [B,C,pn_si1,pn_si1] = area-pool of the final f_hat (ignored when si1 == SN), or NULL
 */
int xq_ms_embed(const xq_ms_desc *d, int si0, int si1, const float *h_all, const float *phi_w, const float *phi_b,
                const float *fhat_in, float *out, float *fhat_scales, float *next, void *stream);

/* ------------------------------------------------------------------------------------------
 * Codebook-usage EMA (xqgan_model.py:777-788, quant.py:121-127,137-141)
 *   ema[rows,V], hit[rows,V]: row i <- copy | 0.9/0.1 | 0.99/0.01 blend of hit[i], chosen by
 *   (record_hit + i) == 0 | < 100 | otherwise  (the reference bumps record_hit once per scale).
 *   usage_out[rows] (device, may be NULL) = 100 * mean(ema[i] >= margin)
 * The step counter is on the device: record_hit_dev[0] = `record_hit` (read, then advanced by `rows` by the kernel),
 * record_hit_dev[1] = scratch (zero-initialised once).  The host neither reads nor writes the counter, which keeps the call
 * CUDA-graph capturable and lets torch.compile trace the module without specialising on a Python int.
 * ------------------------------------------------------------------------------------------ */
int xq_usage_ema_dev(float *ema, const float *hit, int rows, int V, int64_t *record_hit_dev, float margin,
                     float *usage_out, void *stream);

/* ------------------------------------------------------------------------------------------
 * ViT block glue (DINOv2Encoder / DINOv2Decoder blocks)
 *   replaces the non-GEMM ops of Block.forward   tokenizer/tokenizer_image/dino_enc/vision_transformer.py:336-339
 *   (LayerNorm :301,316 ; LayerScale :280-292 ; DropPath ; residual add) and Mlp's GELU.
 * Residual stream fp32 [M,D], GEMM operands bf16 (what bf16 autocast gives the reference).
 * D in {384, 768, 1024}.  `branch`, `y`, `g_y`, `g_branch` are bf16 [M,D].
 *
 * fp16 autocast: every ViT entry point below that takes or returns 16-bit data has an `_f16` twin with the same argument
 * list, the same checks and return codes, in which those tensors are fp16 instead of bf16 (the same kernel instantiated for
 * the other element type).  fp32 -> fp16 roundings are round-to-nearest-even and give +-inf on overflow (no saturation),
 * so a gradient scaler sees an overflow as inf / NaN.
 * ------------------------------------------------------------------------------------------ */
/*   x_out = x + rowscale[row / rows_per_sample] * ls_gamma[d] * (branch + branch_bias[d])
 *           (branch may be NULL: x_out = x; branch_bias = bias of the GEMM that produced `branch`, folded here
 *            so that its gradient is a free column sum of the backward kernel; may be NULL)
 *   y     = LayerNorm(x_out; eps) * ln_w + ln_b   (bf16; may be NULL)   mean / rstd [M] saved for backward
 *   rowscale [B] = DropPath keep mask / keep_prob (NULL = 1);  x_out may alias x or be NULL */
int xq_vit_residual_ln_fwd(const float *x, const void *branch, const float *branch_bias, const float *ls_gamma,
                           const float *rowscale, int rows_per_sample, const float *ln_w, const float *ln_b, float eps,
                           int M, int D, float *x_out, void *y, float *mean, float *rstd, void *stream);
int xq_vit_residual_ln_fwd_f16(const float *x, const void *branch, const float *branch_bias, const float *ls_gamma,
                               const float *rowscale, int rows_per_sample, const float *ln_w, const float *ln_b, float eps,
                               int M, int D, float *x_out, void *y, float *mean, float *rstd, void *stream);
/* workspace of xq_vit_residual_ln_bwd on the current device; 0 when the device cannot be queried (the cause is in
 * xq_last_cuda_error()), and xq_vit_residual_ln_bwd refuses a workspace that small */
size_t xq_vit_ln_bwd_workspace_bytes(int D);
/*   G = g_xout + LayerNorm^T(g_y)  -> g_x [M,D] fp32 ; g_branch = G * rowscale * ls_gamma (bf16)
 *   g_ln_w, g_ln_b, g_ls_gamma, g_branch_bias [D] overwritten (any may be NULL) */
int xq_vit_residual_ln_bwd(const float *g_xout, const void *g_y, const float *x_out, const float *mean,
                           const float *rstd, const float *ln_w, const void *branch, const float *branch_bias,
                           const float *ls_gamma, const float *rowscale, int rows_per_sample, int M, int D, float *g_x,
                           void *g_branch, float *g_ln_w, float *g_ln_b, float *g_ls_gamma, float *g_branch_bias,
                           void *workspace, size_t workspace_bytes, void *stream);
int xq_vit_residual_ln_bwd_f16(const float *g_xout, const void *g_y, const float *x_out, const float *mean,
                               const float *rstd, const float *ln_w, const void *branch, const float *branch_bias,
                               const float *ls_gamma, const float *rowscale, int rows_per_sample, int M, int D, float *g_x,
                               void *g_branch, float *g_ln_w, float *g_ln_b, float *g_ls_gamma, float *g_branch_bias,
                               void *workspace, size_t workspace_bytes, void *stream);
/*   im2col of the patch embedding (timm PatchEmbed = Conv2d(kernel = stride = p), vision_transformer.py PatchEmbed.forward):
 *   x fp32 [B,Cin,H,W] -> patches bf16 [B*(H/p)*(W/p), Cin*p*p] (K index = (c*p + ky)*p + kx = the flattened conv
 *   weight), so that tokens = patches @ weight.view(D,-1)^T + bias is a plain GEMM.  p % 4 == 0, H % p == W % p == 0. */
int xq_vit_patchify(const float *x, void *patches, int B, int Cin, int H, int W, int p, void *stream);
int xq_vit_patchify_f16(const float *x, void *patches, int B, int Cin, int H, int W, int p, void *stream);
/*   token assembly of the ViT encoder / decoder input (dino_enc/dinov2.py:151-170, 318-336):
 *     out[b,t,:] = table[t,:] + (t0 <= t < t0+Ls ? src[b,t-t0,:] : 0)   out fp32 [B,T,D], table fp32 [T,D] (the batch-
 *   independent part: cls / mask / latent tokens + positional + level embeddings), src [B,Ls,D] fp32, bf16 or fp16.
 *   src_type: XQ_ASSEMBLE_FP32 (0), XQ_ASSEMBLE_BF16 (1; any other value but 2 reads as bf16, as before fp16 existed) or
 *   XQ_ASSEMBLE_F16 (2).
 *   backward: d_src = g[:, t0:t0+Ls] in the source dtype (may be NULL), d_table = sum_b g (may be NULL); one read of g. */
#define XQ_ASSEMBLE_FP32 0
#define XQ_ASSEMBLE_BF16 1
#define XQ_ASSEMBLE_F16 2
int xq_vit_assemble_fwd(const void *src, int src_type, const float *table, int B, int Ls, int T, int D, int t0, float *out,
                        void *stream);
int xq_vit_assemble_bwd(const float *g, int B, int Ls, int T, int D, int t0, void *d_src, int src_type, float *d_table,
                        void *stream);
/*   y = GELU(x + bias) exact-erf form (timm Mlp act_layer=nn.GELU), x / y bf16 [M,C], bias fp32 [C] or NULL,
 *   C % 8 == 0.  Backward also returns g_bias [C] = column sums of gx (may be NULL). */
int xq_vit_gelu_fwd(const void *x, const float *bias, void *y, int M, int C, void *stream);
int xq_vit_gelu_bwd(const void *x, const float *bias, const void *gy, void *gx, float *g_bias, int M, int C,
                    void *stream);
int xq_vit_gelu_fwd_f16(const void *x, const float *bias, void *y, int M, int C, void *stream);
int xq_vit_gelu_bwd_f16(const void *x, const float *bias, const void *gy, void *gx, float *g_bias, int M, int C,
                        void *stream);

/*   Flash attention of the ViT blocks, head_dim 64, no mask, no dropout (Attention.forward,
 *   tokenizer/tokenizer_image/dino_enc/vision_transformer.py:173-197: F.scaled_dot_product_attention on
 *   qkv.reshape(B,N,3,H,hd).permute(2,0,3,1,4), then x.transpose(1,2).reshape(B,N,C)).  wgmma / TMA kernel.
 *     qkv   bf16 [B,N,3,H,64]  the packed projection, read in place (no q/k/v copies)
 *     out   bf16 [B,N,H*64]    head-merged attention output (what `proj` consumes)
 *     lse2  fp32 [B,H,N]       base-2 log-sum-exp of the scaled scores (scale*log2(e)*q.k), saved for backward
 *   scale = head_dim^-0.5 (Attention.scale).  Any N >= 1; qkv / out 16-byte aligned. */
int xq_vit_attn_fwd(const void *qkv, void *out, float *lse2, int B, int N, int H, int head_dim, float scale, void *stream);
int xq_vit_attn_fwd_f16(const void *qkv, void *out, float *lse2, int B, int N, int H, int head_dim, float scale, void *stream);

/*   Backward of xq_vit_attn_fwd: d_out bf16 [B,N,H*64] -> dqkv bf16 [B,N,3,H,64] (the gradient of the packed projection,
 *   written in place of autograd's three permuted tensors + stack).  `out` and `lse2` are the forward's results.
 *   workspace (256-byte aligned, xq_vit_attn_bwd_workspace_bytes): fp32 dQ accumulator [B*H,N,64] (atomic adds across
 *   the key blocks) + the padded statistics.  g_bias fp32 [3*H*64] (may be NULL) receives the column sums of dqkv = the
 *   gradient of the qkv bias (nn.Linear's backward `sum(0)` pass, fused into the epilogues).  3 launches + memsets. */
size_t xq_vit_attn_bwd_workspace_bytes(int B, int N, int H);
int xq_vit_attn_bwd(const void *qkv, const void *out, const void *d_out, const float *lse2, void *dqkv, float *g_bias, int B, int N,
                    int H, int head_dim, float scale, void *workspace, size_t workspace_bytes, void *stream);
/*   fp16 twins: qkv / out / d_out / dqkv fp16; P and dS are rounded to fp16 as the operands of their MMAs (scores and the
 *   dQ accumulator stay fp32).  The workspace is the same as the bf16 call's. */
int xq_vit_attn_bwd_f16(const void *qkv, const void *out, const void *d_out, const float *lse2, void *dqkv, float *g_bias, int B,
                        int N, int H, int head_dim, float scale, void *workspace, size_t workspace_bytes, void *stream);

/*
 * ---- loss stack (SURVEY.md section 8 row f-1) -------------------------------------------------------------------
 * LPIPS stage distance (tokenizer/tokenizer_image/lpips.py:79-90): for one VGG stage with feature maps f0, f1
 * [B,C,H*W] (fp32, or bf16 when is_bf16) and the stage's `lin` weights lin_w [C]:
 *   out[b] (+)= mean_p sum_c lin_w[c] * ( f0/(|f0|_c + eps) - f1/(|f1|_c + eps) )^2      (accumulate != 0: add to out)
 * backward returns the gradient w.r.t. f1 (swap the maps for f0); g_out [B] is d loss / d out.
 * The fp64 per-CTA partials live in the caller's workspace (xq_lpips_workspace_bytes).
 */
size_t xq_lpips_workspace_bytes(int B, int HW);
int xq_lpips_layer_forward(const void *f0, const void *f1, int is_bf16, const float *lin_w, int B, int C, int HW, float eps,
                           int accumulate, float *out, void *workspace, size_t workspace_bytes, void *stream);
int xq_lpips_layer_backward(const void *f0, const void *f1, int is_bf16, const float *lin_w, int B, int C, int HW, float eps,
                            const float *g_out, void *g_f1, void *stream);
/*
 * DiffAug.aug without the warm-up blur (tokenizer/tokenizer_image/diffaug.py:60-118): translation (zero fill), colour
 * (brightness, saturation about the per-pixel channel mean, contrast about the per-sample mean) and cutout.
 *   x, y, g, gx  [B,C,H,W] fp32, C <= 8 ;  rand01 [7,B] = the reference's torch.rand(7,B,1,1) (:64) ;
 *   flags: bit0 translation, bit1 colour, bit2 cutout (the reference's three `torch.rand(3) <= prob` draws, :61) ;
 *   cut_h, cut_w = round(H*cutout), round(W*cutout) ; sums [B] scratch.
 * backward is the exact transpose of the (per-sample affine) forward map.
 */
int xq_diffaug_forward(const float *x, const float *rand01, int B, int C, int H, int W, int flags, int cut_h, int cut_w,
                       float *y, float *sums, void *stream);
int xq_diffaug_backward(const float *g, const float *rand01, int B, int C, int H, int W, int flags, int cut_h, int cut_w,
                        float *gx, float *sums, void *stream);

/* ---- ViT MLP with the element-wise work fused into a hand-written wgmma GEMM (csrc/gemm_kernel.cu) ----------------------
 * Replaces, inside timm's Mlp as called by Block.forward (tokenizer/tokenizer_image/dino_enc/vision_transformer.py:336-339):
 *   forward   F.linear(y, W1) [cuBLAS] + GELU(. + b1) [xq_vit_gelu_fwd]            -> xq_vit_fc1_gelu_fwd
 *   backward  d_act = d_out W2 [cuBLAS] + d_act * GELU'(pre + b1), d_b1 [xq_vit_gelu_bwd] -> xq_vit_fc2_dgelu_bwd
 * All matrices row-major bf16; bias / d_bias fp32.  N % 128 == 0, N / 128 <= SM count, K % 64 == 0 (else XQ_ERR_UNSUPPORTED),
 * any M.  pre / act / d_pre apply the same device functions to the same rounded bf16 GEMM results as that two-call sequence
 * (equal up to the GEMM's fp32 accumulation order); d_bias is summed with fp32 atomics, in no fixed order.
 * One kernel, three roles per CTA: MMA warpgroups that hand each 128 x 128 tile, rounded to bf16, to an epilogue warpgroup
 * through shared memory and go on to the next tile; the epilogue warpgroup; a TMA producer warp.  pre / act / d_pre are
 * written by TMA stores (and pre read by TMA loads in the backward), so they must be 16-byte aligned like the operands.
 *   x [M,K], w [N,K] (fc1.weight as bf16)  ->  pre [M,N] = x w^T ,  act [M,N] = GELU(pre + bias)                               */
int xq_vit_fc1_gelu_fwd(const void *x, const void *w, const float *bias, void *pre, void *act, int M, int N, int K, void *stream);
/*  d_out [M,K] (gradient of the fc2 output), w2t [N,K] (fc2.weight TRANSPOSED, bf16), pre [M,N] (saved by the forward)
 *   ->  d_pre [M,N] = (d_out w2t^T) * GELU'(pre + bias) ,  d_bias [N] = column sums of the rounded d_pre                      */
int xq_vit_fc2_dgelu_bwd(const void *d_out, const void *w2t, const void *pre, const float *bias, void *d_pre, float *d_bias,
                         int M, int N, int K, void *stream);
/* LoRA forms of the two calls above, for fc1 / fc2 wrapped with rank-R adapters (imagefolder_b200/dino_enc/lora.py, peft's
 * `base_layer(x) + lora_B(lora_A(x)) * scaling`).  The caller forms the rank-R activation; the kernel adds its product with
 * the adapter as one more K stage, into the same fp32 accumulators, before the single rounding of the GEMM result:
 *   u [M,R] = s x A1^T (bf16), b_lora [N,R] = lora_B of fc1 (bf16)
 *     ->  pre [M,N] = x w^T + u b_lora^T ,  act [M,N] = GELU(pre + bias)
 *   v [M,R] = s d_out B2 (bf16), a2t [N,R] = lora_A of fc2 TRANSPOSED (bf16)
 *     ->  d_pre [M,N] = (d_out w2t^T + v a2t^T) * GELU'(pre + bias) ,  d_bias [N] = column sums of the rounded d_pre
 * Equal, bit for bit, to xq_vit_fc1_gelu_fwd / xq_vit_fc2_dgelu_bwd on the operands concatenated along K and zero-padded to
 * K + 64 ([x | u], [w | b_lora]) up to the fp32 accumulation order.  Same checks and codes as those two, plus
 * 8 <= R <= 64 with R % 8 == 0 and u / v, b_lora / a2t non-NULL and 16-byte aligned (else XQ_ERR_ARG).  A refused call writes
 * nothing. */
int xq_vit_fc1_lora_gelu_fwd(const void *x, const void *w, const void *u, const void *b_lora, const float *bias, void *pre, void *act,
                             int M, int N, int K, int R, void *stream);
int xq_vit_fc2_lora_dgelu_bwd(const void *d_out, const void *w2t, const void *v, const void *a2t, const void *pre, const float *bias,
                              void *d_pre, float *d_bias, int M, int N, int K, int R, void *stream);
/* fp16 twins of the four calls above: every 16-bit matrix is fp16 (fp16 autocast), everything else as above. */
int xq_vit_fc1_gelu_fwd_f16(const void *x, const void *w, const float *bias, void *pre, void *act, int M, int N, int K,
                            void *stream);
int xq_vit_fc2_dgelu_bwd_f16(const void *d_out, const void *w2t, const void *pre, const float *bias, void *d_pre, float *d_bias,
                             int M, int N, int K, void *stream);
int xq_vit_fc1_lora_gelu_fwd_f16(const void *x, const void *w, const void *u, const void *b_lora, const float *bias, void *pre,
                                 void *act, int M, int N, int K, int R, void *stream);
int xq_vit_fc2_lora_dgelu_bwd_f16(const void *d_out, const void *w2t, const void *v, const void *a2t, const void *pre,
                                  const float *bias, void *d_pre, float *d_bias, int M, int N, int K, int R, void *stream);

/* ---- input pipeline: the training / validation image transforms (SURVEY.md section 8 row f-4, csrc/img_kernels.cu) ---------
 * Replaces the per-image CPU transform of the reference's DataLoader workers:
 *   train  Compose([random_crop_arr, RandomHorizontalFlip(), ToTensor(), Normalize(0.5, 0.5)])  xqgan_train.py:225-230
 *   val    Compose([center_crop_arr, ToTensor(), Normalize(0.5, 0.5)])                          xqgan_train.py:250-254
 *   random_crop_arr / center_crop_arr                                                  dataset/augmentation.py:29-50 / :8-26
 * bit-identically (Pillow 8-bit Image.resize arithmetic for the BOX halvings and the BICUBIC resize).  The workers only decode
 * (np.asarray(Image.open(f).convert('RGB'))) and draw the random numbers; imagefolder_b200/data.py makes the plan.
 *   src     uint8, every image [h, w, 3] (HWC) packed back to back; src_bytes = its length
 *   offs    int64 [B, 2]: {byte offset of image i in src, byte offset of its halving buffers in the workspace}
 *   plan    int32 [B, XQ_IMG_PLAN_COLS]: {h, w, levels (BOX halvings, augmentation.py:37-40 / :13-16), rs_h, rs_w (BICUBIC size,
 *           :42-45 / :18-21), crop_y, crop_x (:48-49 / :24-25), flip (RandomHorizontalFlip's torch.rand(1) < 0.5)}
 *   out     fp32 [B, 3, S, S] = (u / 255 - 0.5) / 0.5 of the cropped (and flipped) uint8 pixels
 * A plan row is valid when h, w >= 1, (h, w) >> levels >= 1, rs_h, rs_w >= S, the crop lies inside the resized image, flip is 0/1
 * and the BICUBIC resize has at most XQ_IMG_MAX_TAPS taps per axis (a downscale by less than 4 after the halvings).  The kernels
 * re-check every row and every buffer bound and leave the output of an invalid image unwritten.
 * ------------------------------------------------------------------------------------------------------------------------------ */
#define XQ_IMG_PLAN_COLS 8
#define XQ_IMG_MAX_TAPS 17
#define XQ_IMG_MAX_SIZE 4096   /* largest crop side S */
/* host-side: validates the plan (a HOST copy) for crop side S and lays out the halving buffers: ws_off_host [B] (may be NULL)
 * receives each image's workspace offset.  Returns the workspace bytes (>= 16), or 0 when an argument or a plan row is invalid. */
size_t xq_img_workspace_bytes(const int32_t *plan_host, int B, int S, int64_t *ws_off_host);
/* one BOX halving level (1-based) for every image with levels >= level: (h, w) >> (level-1) -> (h, w) >> level, into the
 * workspace.  Call it for level = 1 .. max(levels); max_out_h / max_out_w (the largest output at this level) only size the grid. */
int xq_img_box_halve(const uint8_t *src, size_t src_bytes, const int64_t *offs, const int32_t *plan, int B, int S, int level,
                     int max_out_h, int max_out_w, void *workspace, size_t workspace_bytes, void *stream);
/* the final BICUBIC resize, evaluated only on the crop window, then flip, ToTensor and Normalize.  workspace may be NULL when no
 * image has levels > 0. */
int xq_img_resize_crop_normalize(const uint8_t *src, size_t src_bytes, const int64_t *offs, const int32_t *plan, int B, int S,
                                 const void *workspace, size_t workspace_bytes, float *out, void *stream);

/* ---- weight EMA of the trainer (csrc/ema_kernel.cu) ------------------------------------------------------------------------
 * Replaces update_ema (utils/ema.py:4-14, called after every optimizer step at xqgan_train.py:461-462): for i < n
 *   ema[i][k] <- ema[i][k] * decay + one_minus_decay * param[i][k]      k < numel[i], fp32
 * bit-identical to torch's `ema.mul_(decay); ema.add_(param, alpha=one_minus_decay)` on the same GPU (fma(param, a, ema * d)).
 *   ema, param, numel   HOST arrays of n entries; the pointers in ema / param are device pointers (4-byte aligned)
 * The table travels in the kernel's parameter space: one launch per XQ_EMA_MAX_TENSORS entries, in order, on `stream`.
 * n == 0 is a no-op; entries with numel 0 are skipped (their pointers may be NULL).  Every entry is validated before the first
 * launch, so XQ_ERR_ARG (n < 0, NULL arrays, a negative numel, a NULL or misaligned pointer) means nothing was written.
 * ------------------------------------------------------------------------------------------------------------------------------ */
#define XQ_EMA_MAX_TENSORS 1020
int xq_ema_update(float *const *ema, const float *const *param, const int64_t *numel, int n, float decay, float one_minus_decay,
                  void *stream);

/* ---- AdamW step of the trainer (csrc/adamw_kernel.cu) ----------------------------------------------------------------------
 * Replaces optimizer.step() / optimizer_disc.step() (torch.optim.AdamW, xqgan_train.py:344-347, 459, 474): for i < n, k < numel[i]
 *   p = p * wd_factor  (skipped when wd_factor == 1);  m = lerp(m, g, one_minus_beta1);  v = v * beta2 + one_minus_beta2 * g * g
 *   p = p + step_size[i] * m / (sqrt(v) / bc2_sqrt[i] + eps)
 * bit-identical to torch's foreach AdamW (_multi_tensor_adam) for a tensor at step t, with the host values
 *   wd_factor = 1 - lr * weight_decay, one_minus_beta1 = 1 - beta1, one_minus_beta2 = 1 - beta2,
 *   step_size[i] = -(lr / (1 - beta1 ** t_i)), bc2_sqrt[i] = (1 - beta2 ** t_i) ** 0.5          (all doubles, t_i after the increment)
 * each rounded once to fp32 here, as torch rounds its Scalar and scalar-list arguments.
 *   param, grad, exp_avg, exp_avg_sq, numel, step_size, bc2_sqrt   HOST arrays of n entries; the tensor pointers are fp32 device
 *   pointers (4-byte aligned).  The table travels in the kernel's parameter space: one launch per XQ_ADAMW_MAX_TENSORS entries, in
 *   order, on `stream`.
 * n == 0 is a no-op; entries with numel 0 are skipped (their pointers may be NULL).  Every entry and scalar is validated before the
 * first launch, so XQ_ERR_ARG (n < 0, NULL arrays, a negative numel, a NULL or misaligned pointer, a non-finite scalar) means
 * nothing was written.
 * ------------------------------------------------------------------------------------------------------------------------------ */
#define XQ_ADAMW_MAX_TENSORS 584
int xq_adamw_step(float *const *param, const float *const *grad, float *const *exp_avg, float *const *exp_avg_sq,
                  const int64_t *numel, const double *step_size, const double *bc2_sqrt, int n, double wd_factor,
                  double one_minus_beta1, double beta2, double one_minus_beta2, double eps, void *stream);

/* ---- gradient-norm clipping of the trainer (csrc/clip_kernel.cu) ----------------------------------------------------------
 * The two streaming passes of torch.nn.utils.clip_grad_norm_(params, max_norm) (xqgan_train.py:456-458, 471-473, with
 * --max_grad_norm set); the steps between them are torch's own ops on `norms` (imagefolder_b200/optim.py::clip_grad_norm_).
 *
 * xq_grad_norm: norms[i] = ||grad[i]||_2 for i < n, fp32, bit-identical to torch.stack(torch._foreach_norm(grads)) on the same
 *   GPU (the same per-chunk partials, trees and sqrt).  norms is a device array of n floats (4-byte aligned); entries with
 *   numel 0 get 0.  The per-chunk partials go to the caller's workspace of xq_grad_norm_workspace_bytes(n, numel) bytes.
 *   Two launches per XQ_CLIP_MAX_TENSORS entries (chunk partials, then one block per tensor), in order, on `stream`.
 * xq_grad_scale: grad[i][k] <- grad[i][k] * (*coef) for i < n, k < numel[i]: torch's _foreach_mul_(grads, coef) with coef a
 *   0-dim fp32 device tensor, read on the device (the host never synchronises).  One launch per XQ_CLIP_MAX_TENSORS entries.
 *   grad, numel   HOST arrays of n entries; the pointers in grad are fp32 device pointers (4-byte aligned).
 * n == 0 is a no-op; entries with numel 0 are not read (their pointers may be NULL).  Every entry is validated before the first
 * launch, so XQ_ERR_ARG (n < 0, NULL arrays, a negative numel, a NULL or misaligned pointer) and XQ_ERR_WORKSPACE mean nothing
 * was written.
 * ------------------------------------------------------------------------------------------------------------------------------ */
#define XQ_CLIP_MAX_TENSORS 1360
/* bytes of the partial-sum workspace of xq_grad_norm (4 per 65 536-float chunk); 0 when an argument is out of range */
size_t xq_grad_norm_workspace_bytes(int n, const int64_t *numel);
int xq_grad_norm(const float *const *grad, const int64_t *numel, int n, float *norms, void *workspace, size_t workspace_bytes,
                 void *stream);
int xq_grad_scale(float *const *grad, const int64_t *numel, int n, const float *coef, void *stream);

/* ---- reconstruction metrics: PSNR and SSIM per image (csrc/metric_kernels.cu) ---------------------------------------------
 * Replaces the scikit-image calls of the reference's reconstruction evaluation (tokenizer/vqgan/reconstruction_vqgan_ddp.py:
 * 155-169), per image b of rec [B,C,H,W] (the clamped reconstruction, fp32, or bf16 when rec_is_bf16) and x [B,C,H,W] fp32 (the
 * model input in [-1, 1]):
 *   g = (x + 1) / 2 ;  r = uint8(clamp(127.5 * rec + 128, 0, 255)) / 255                   (fp32)
 *   psnr[b] = peak_signal_noise_ratio(r, g)                     10 log10(1 / mse), mse in fp64; +inf when mse == 0
 *   ssim[b] = structural_similarity(r, g, data_range=2.0, channel_axis=-1)
 *             7x7 uniform window, sample covariance, K1 = 0.01, K2 = 0.03; per channel the fp64 mean of S over the windows
 *             inside the image, then the mean over channels
 * psnr, ssim: fp64 device arrays [B].  Deterministic (fixed-order fp64 reductions, no atomics).  C >= 1, H, W >= 7; the
 * workspace (16-byte aligned) holds two fp64 partials per (image, channel, strip of XQ_METRIC_STRIP_ROWS rows, column tile).
 * XQ_ERR_ARG (a bad size or flag, a NULL or misaligned pointer) and XQ_ERR_WORKSPACE are returned before anything is written.
 * ------------------------------------------------------------------------------------------------------------------------------ */
#define XQ_METRIC_STRIP_ROWS 32
/* 0 when an argument is out of range */
size_t xq_recon_psnr_ssim_workspace_bytes(int B, int C, int H, int W);
int xq_recon_psnr_ssim(const void *rec, int rec_is_bf16, const float *x, int B, int C, int H, int W, double *psnr, double *ssim,
                       void *ws, size_t ws_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* XQB200_H_ */
