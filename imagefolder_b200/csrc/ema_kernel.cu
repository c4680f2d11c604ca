// ema_kernel.cu -- the weight EMA of the tokenizer trainer on the GPU (sm_90a).
//
// Replaces update_ema (utils/ema.py:4-14), which the reference calls after every optimizer step
// (tokenizer/tokenizer_image/xqgan_train.py:461-462): for every parameter tensor
//   ema.mul_(decay).add_(param, alpha = 1 - decay)
// i.e. two elementwise kernels and two HBM passes per tensor.  Here one launch updates every tensor of the call in a
// single pass (read ema, read param, write ema: 12 bytes per element).
//
// Arithmetic: bit-identical to those two torch ops on the same GPU.  mul_ rounds e * d to fp32; ATen's CUDA add with
// alpha evaluates `self + other * alpha` in fp32 and nvcc contracts it to one fma.  Both steps are written as
// intrinsics so that the -fmad flag of this translation unit cannot change them.
//
// Work split: the tensor table travels in the kernel's parameter space and a persistent grid streams its 64 KiB chunks
// (xq_chunks.cuh): four float4 pairs in flight per thread when both bases are 16-byte aligned, eight floats otherwise.
#include <cuda_runtime.h>
#include <stdint.h>

#include "xq_chunks.cuh"

namespace xqe {

using xqc::THREADS;
constexpr int U4 = 4;                        // float4 pairs in flight per thread (2 x 64 B)
constexpr int U1 = 8;                        // floats in flight per thread on the scalar path

struct Scalars {
    float d, a;                              // decay, 1 - decay
};
using EmaTable = xqc::Table<2, XQ_EMA_MAX_TENSORS, Scalars>;   // arrays: ema (written), param
static_assert(sizeof(EmaTable) <= xqc::PARAM_BYTES, "the tensor table must fit in the kernel parameter space");

__global__ void __launch_bounds__(THREADS) ema_update_kernel(const __grid_constant__ EmaTable tab) {
    const float d = tab.own.d, a = tab.own.a;
    xqc::stream_table<0b01, U4, U1>(tab, [=](float (&x)[2]) { x[0] = __fmaf_rn(x[1], a, __fmul_rn(x[0], d)); });
}

}  // namespace xqe

using namespace xqe;

extern "C" {

int xq_ema_update(float *const *ema, const float *const *param, const int64_t *numel, int n, float decay,
                  float one_minus_decay, void *stream) {
    if (n < 0) return XQ_ERR_ARG;
    if (n == 0) return XQ_OK;
    int64_t chunks = 0;                      // every entry is checked before the first launch: a refused call writes nothing
    if (xqc::check_entries({ema, param}, numel, n, &chunks) != XQ_OK) return XQ_ERR_ARG;
    if (chunks == 0) return XQ_OK;
    EmaTable tab;
    tab.own.d = decay;
    tab.own.a = one_minus_decay;
    return xqc::launch_tables(ema_update_kernel, THREADS, "ema_update_kernel", tab, {ema, param}, numel, n, stream);
}

}  // extern "C"
