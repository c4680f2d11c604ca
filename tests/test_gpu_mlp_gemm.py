"""The fused MLP GEMMs xq_vit_fc1_gelu_fwd / xq_vit_fc2_dgelu_bwd (csrc/gemm_kernel.cu), checked bit for bit through the C ABI.

Exact-grid operands: every A entry (x, d_out) is in {-1, 0, 1} * 2^-3 and every B entry (w1, w2t) in {-1, 0, 1} * 2^-2, so
each product is an integer multiple of 2^-5 and each partial sum of a dot product has magnitude <= K units of 2^-5
(K <= 1024 < 2^11).  An fp32 accumulator (24-bit significand) holds every such partial sum exactly, in any order, so the
GEMM result is exact and the kernel's bf16 `pre` / rounded `d_act` must equal bf16 of an fp64 GEMM to the last bit.

Three kinds of fc1-bias columns, interleaved (column % 3) so that every 128-column block and every column % 8 lane position
has all three:
  b1 = +40: with |pre| < 16, gelu_f(pre + b1) is exactly pre + b1 (the p^16 of xq_gelu.cuh overflows, its reciprocal is 0)
            and dgelu_f is exactly 1 (ex2.approx.ftz of -x^2 / (2 ln 2) flushes to 0): act and d_pre are known exactly;
  b1 = -40: both functions are exactly 0;
  b1 ~ N(0, 1): the transcendental epilogue, checked bit for bit against the stand-alone xq_vit_gelu_fwd / _bwd kernels run
            on the fused kernel's own `pre` (the header's "same bits" claim) and against an fp64 erf-GELU.
Every output is NaN-filled and followed by 128 guard rows holding a sentinel, so an unwritten element or a write past row M
fails.  The inputs x / d_out carry 128 extra rows of nonzero values after row M: a tensor map that reached past M would feed
them into the backward's bias gradient.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

XQ_ERR_UNSUPPORTED = -4
GUARD = 128                   # guard rows after every input and output
SENTINEL = -12345             # int16 bit pattern of the output guard rows
CHUNK = 8192                  # rows per fp64 reference chunk (caps the reference's memory)
SAT = 40.0                    # |b1| of the saturated columns
TRAIN_S = (513, 514, 769, 499, 379)   # encoder / decoder sequence lengths of the shipped configs (DESIGN.md section 3)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _lib():
    from imagefolder_b200 import _capi
    return _capi, _capi.lib()


def _grid(rows, cols, scale, gen):
    """entries in {-1, 0, 1} * scale, bf16 (scale a power of two: exact)"""
    return torch.randint(-1, 2, (rows, cols), device="cuda", generator=gen).to(torch.bfloat16) * scale


def _bias(N, gen):
    b = torch.randn(N, device="cuda", generator=gen)
    kind = torch.arange(N, device="cuda") % 3
    b[kind == 0] = SAT
    b[kind == 1] = -SAT
    return b


def _guarded(M, N):
    """bf16 [M + GUARD, N]: rows < M NaN, the guard rows a sentinel bit pattern"""
    t = _nan((M + GUARD, N), torch.bfloat16)
    t[M:].view(torch.int16).fill_(SENTINEL)
    return t


def _assert_guard(t, M, what):
    bad = t[M:].view(torch.int16) != SENTINEL
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} guard elements after row {M} overwritten"


def _first_bad(bad):
    return tuple(int(i) for i in bad.nonzero()[0])


def _assert_bits(a, b, what):
    """bf16 a, b identical bit for bit (a NaN in a never-written output fails)"""
    bad = a.view(torch.int16) != b.view(torch.int16)
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements differ, first at {_first_bad(bad)}"


def _assert_bits_but_zero_sign(a, b, what):
    """bit for bit, except that +0 and -0 match: neither the fp64 reference GEMM nor the tensor cores fix the sign of an
    exactly cancelling sum, and 0 times a negative number is -0"""
    bad = (a.view(torch.int16) != b.view(torch.int16)) & ~((a == 0) & (b == 0))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} of {bad.numel()} elements differ, first at {_first_bad(bad)}"


def _assert_within(a, ref, tol, what):
    """|a - ref| <= tol elementwise; NaN fails"""
    err = (a.double() - ref).abs()
    ok = err <= tol
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} of {ok.numel()} out of tolerance, max err {err.max().item():.3e}"


def _gelu64(u):
    return 0.5 * u * (1.0 + torch.erf(u / math.sqrt(2.0)))


def _per_col(M, N):
    """CTAs per 128-column block (gm_launch): the SMs shared among the column blocks, at most one per row block"""
    return min(_sms() // (N // 128), (M + 127) // 128)


def _check(x, w1, b1, d_out, w2t, M, N, K):
    """Run xq_vit_fc1_gelu_fwd on rows [0, M) of x, then xq_vit_fc2_dgelu_bwd on rows [0, M) of d_out with the forward's own
    `pre`, and check every output.  x / d_out must hold at least M + GUARD rows."""
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr(x.device)
    assert x.shape[0] >= M + GUARD and d_out.shape[0] >= M + GUARD
    pos, neg = b1 == SAT, b1 == -SAT
    pre, act = _guarded(M, N), _guarded(M, N)
    _capi.check(L.xq_vit_fc1_gelu_fwd(p(x), p(w1), p(b1), p(pre), p(act), M, N, K, s), "xq_vit_fc1_gelu_fwd")
    d_pre, d_bias = _guarded(M, N), _nan((N,))          # d_bias NaN: the entry point zeroes it itself
    _capi.check(L.xq_vit_fc2_dgelu_bwd(p(d_out), p(w2t), p(pre), p(b1), p(d_pre), p(d_bias), M, N, K, s), "xq_vit_fc2_dgelu_bwd")

    w1d, w2d, b1d = w1.double(), w2t.double(), b1.double()
    sum_pos = torch.zeros(int(pos.sum()), dtype=torch.float64, device="cuda")   # exact column sums of bf16(d_act) on +40
    abs_pos = torch.zeros_like(sum_pos)
    sum_all = torch.zeros(N, dtype=torch.float64, device="cuda")                 # column sums of the kernel's d_pre
    abs_all = torch.zeros_like(sum_all)
    for r0 in range(0, M, CHUNK):
        r1 = min(M, r0 + CHUNK)
        rows = r1 - r0
        pre_c, act_c, dp_c = pre[r0:r1], act[r0:r1], d_pre[r0:r1]

        # ---- forward
        ref = x[r0:r1].double() @ w1d.t()
        assert float(ref[:, pos | neg].abs().max()) < 16, "precondition: |pre| < 16 on the saturated columns"
        _assert_bits_but_zero_sign(pre_c, ref.to(torch.bfloat16), "pre vs bf16(fp64 GEMM)")
        del ref
        # +40: act = bf16(pre + 40) -- the fp32 sum is exact (pre is a multiple of 2^-5 below 16); -40: act = 0
        _assert_bits(act_c[:, pos], (pre_c[:, pos].float() + SAT).to(torch.bfloat16), "act on b1 = +40")
        assert bool((act_c[:, neg] == 0).all()), "act on b1 = -40"
        g_fwd = _nan((rows, N), torch.bfloat16)
        _capi.check(L.xq_vit_gelu_fwd(p(pre_c), p(b1), p(g_fwd), rows, N, s), "xq_vit_gelu_fwd")
        _assert_bits(act_c, g_fwd, "act vs xq_vit_gelu_fwd on the same pre")
        del g_fwd
        # vs fp64 erf-GELU: bf16 rounding (2^-8 relative) + gelu_f's |abs err| <= 7.1e-7 (A&S 7.1.28 in fp32)
        u = pre_c.double() + b1d
        gref = _gelu64(u)
        del u
        _assert_within(act_c, gref, 2 ** -8 * gref.abs() + 1e-6, "act vs fp64 GELU(pre + b1)")
        del gref

        # ---- backward: d_act is exact in fp32, so the kernel's rounded d_act is bf16(fp64 d_act)
        gy = (d_out[r0:r1].double() @ w2d.t()).to(torch.bfloat16)
        gx = _nan((rows, N), torch.bfloat16)
        _capi.check(L.xq_vit_gelu_bwd(p(pre_c), p(b1), p(gy), p(gx), None, rows, N, s), "xq_vit_gelu_bwd")
        _assert_bits_but_zero_sign(dp_c, gx, "d_pre vs xq_vit_gelu_bwd on the same pre and d_act")
        del gx
        _assert_bits_but_zero_sign(dp_c[:, pos], gy[:, pos], "d_pre on b1 = +40")
        assert bool((dp_c[:, neg] == 0).all()), "d_pre on b1 = -40"
        t = gy[:, pos].double()
        sum_pos += t.sum(0)
        abs_pos += t.abs().sum(0)
        t = dp_c.double()
        sum_all += t.sum(0)
        abs_all += t.abs().sum(0)
        del gy, t

    # d_bias on the saturated columns, by equality: the terms are multiples of 2^-5, and with sum |terms| < 2^24 units every
    # partial sum is exact in fp32, whatever the order -- a row block dropped, counted twice or lost from an atomic fails
    assert float(abs_pos.max()) < 2 ** 24 * 2 ** -5, "precondition: the +40 column sums are exact in fp32"
    assert torch.equal(d_bias[pos].double(), sum_pos), "d_bias on b1 = +40 differs from the exact column sums"
    assert bool((d_bias[neg] == 0).all()), "d_bias on b1 = -40"
    # d_bias on every column, against the fp64 column sums of the kernel's own rounded d_pre.  A column's value passes
    # through at most 2 ceil(nM / per_col) sequential fp32 adds in a thread (rows r and r + 8 of each of its CTA's row
    # blocks), 3 shuffle-tree adds, and one atomicAdd per consumer warp of each CTA on the column (8 per_col); each add
    # rounds by at most 2^-24 relative, so the error is at most depth * 2^-24 * sum |terms| (first order).
    nM, per_col = (M + 127) // 128, _per_col(M, N)
    depth = 2 * -(-nM // per_col) + 3 + 8 * per_col
    _assert_within(d_bias, sum_all, depth * 2 ** -24 * abs_all, "d_bias vs fp64 column sums of d_pre")
    for t, what in ((pre, "pre"), (act, "act"), (d_pre, "d_pre")):
        _assert_guard(t, M, what)


def _operands(M, N, K, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = _grid(M + GUARD, K, 2 ** -3, gen)
    w1 = _grid(N, K, 2 ** -2, gen)
    d_out = _grid(M + GUARD, K, 2 ** -3, gen)
    w2t = _grid(N, K, 2 ** -2, gen)
    return x, w1, _bias(N, gen), d_out, w2t


def _run(M, N, K, seed):
    x, w1, b1, d_out, w2t = _operands(M, N, K, seed)
    _check(x, w1, b1, d_out, w2t, M, N, K)


@pytest.mark.parametrize("B", [128, 64, 1, 3])
@pytest.mark.parametrize("S", TRAIN_S)
def test_training_rows_vit_base(B, S):
    """The ViT-B MLP (C = 768, hidden 3072: 24 column blocks) at the training rows: at B = 128 each CTA walks ~100 row blocks
    through the ring; at B = 64 an odd S leaves M % 128 = 64 (the tail tile ends where the second warpgroup starts); at B = 1
    and 3 the tail ends inside either warpgroup (M % 128 = 1, 2, 3, 6, 89, 113, 115, 123)."""
    _run(B * S, 3072, 768, seed=B * 1000 + S)


@pytest.mark.parametrize("C,H", [(384, 1536), (1024, 4096)])
@pytest.mark.parametrize("M", [128 * 513, 3 * 499])
def test_other_widths(C, H, M):
    """ViT-S (12 column blocks, K = 384) and ViT-L (32 column blocks, K = 1024) widths at a training and a ragged M."""
    _run(M, H, C, seed=C + M)


@pytest.mark.parametrize("M", [1, 8, 9, 63, 64, 65, 120, 127, 128, 129, 191, 192, 193])
def test_row_tails(M):
    """Tail tiles that end inside the first warpgroup's rows, at its end, inside the second's, and on tile boundaries."""
    _run(M, 3072, 768, seed=M)


@pytest.mark.parametrize("K", [64, 256, 320, 384, 448])
def test_ring_depth(K):
    """nk = K / 64 against the 5-stage ring: one stage per tile, a ring that never fills, exactly fills, and wraps inside a
    tile.  Each CTA walks 6-7 row blocks, so with nk % 5 != 0 every tile starts at a different stage and parity."""
    N = 3072
    M = 128 * _per_col(1 << 30, N) * 6 + 100
    _run(M, N, K, seed=K)


def test_one_column_block_grid_clamped_to_row_blocks():
    """N = 128: one column block, fewer row blocks than SMs, so the grid is nM CTAs of one row block each."""
    M = 128 * (_sms() // 2) + 77
    assert _per_col(M, 128) == (M + 127) // 128 < _sms()
    _run(M, 128, 256, seed=1)


def test_one_cta_per_column_block():
    """N = 128 * SMs: per_col = 1, each CTA walks every row block of its column."""
    N = 128 * _sms()
    assert _per_col(1 << 30, N) == 1
    _run(128 * 8 + 5, N, 128, seed=2)


def test_more_column_blocks_than_sms_is_refused_without_writing():
    """N = 128 * (SMs + 1) cannot keep one CTA per column block: XQ_ERR_UNSUPPORTED, and no output is touched."""
    _capi, L = _lib()
    p, s = _capi.ptr, _capi.stream_ptr()
    M, N, K = 8, 128 * (_sms() + 1), 64
    x, w1, b1, d_out, w2t = _operands(M, N, K, seed=3)
    pre, act, d_pre, d_bias = _guarded(M, N), _guarded(M, N), _guarded(M, N), _nan((N,))
    assert L.xq_vit_fc1_gelu_fwd(p(x), p(w1), p(b1), p(pre), p(act), M, N, K, s) == XQ_ERR_UNSUPPORTED
    assert L.xq_vit_fc2_dgelu_bwd(p(d_out), p(w2t), p(pre), p(b1), p(d_pre), p(d_bias), M, N, K, s) == XQ_ERR_UNSUPPORTED
    for t in (pre, act, d_pre):
        assert bool(t[:M].isnan().all())
        _assert_guard(t, M, "refused call")
    assert bool(d_bias.isnan().all()), "a refused call zeroed d_bias"


def _attn_check(qkv, g):
    """xq_vit_attn_fwd / _bwd on qkv [1, N, 192] (one head) against fp32 autograd, at tests/test_gpu_attn.py's tolerances"""
    from imagefolder_b200 import vit_ops
    q32 = qkv.float().requires_grad_(True)
    q, k, v = q32.view(1, -1, 3, 64).unbind(2)
    s = (q @ k.transpose(-1, -2)) * 0.125
    o_ref = torch.softmax(s, -1) @ v
    (o_ref * g.float()).sum().backward()
    out, lse2 = vit_ops.attn_tc_forward(qkv, 1)
    dqkv = vit_ops.attn_tc_backward(qkv, out, lse2, g, 1)
    assert (out.float() - o_ref).abs().max().item() <= 8e-3 * max(1.0, o_ref.abs().max().item())
    gr, d = q32.grad.view(-1, 3, 64), dqkv.float().view(-1, 3, 64)
    for i in range(3):
        assert (d[:, i] - gr[:, i]).abs().max().item() <= 1e-2 * max(1e-3, gr[:, i].abs().max().item())


def test_tensor_map_cache_eviction_and_reuse():
    """One cache of 128 tensor maps (xqtc::tensor_map, round-robin) serves the GEMMs, the attention kernels and the VQ
    search.  Each of 64 distinct (pointer, M) GEMM combinations adds two maps (the A operands of the forward and the
    backward call), and an attention forward + backward on a fresh slice of a qkv buffer, interleaved after it, adds three
    more: 320 new maps wrap the cache twice, and the GEMMs' B maps and the attention maps evict one another.  Then the first
    combination again, and the same buffers with a smaller M.  A map reused for the wrong M would read the nonzero rows
    after M, which changes the bias gradient; a stale attention map would read another slice."""
    N, K = 256, 128
    gen = torch.Generator(device="cuda").manual_seed(4)
    combos = [(8 * i, 37 + 11 * i) for i in range(64)]          # (row offset, M)
    rows = max(o + m for o, m in combos) + GUARD
    x, d_out = _grid(rows, K, 2 ** -3, gen), _grid(rows, K, 2 ** -3, gen)
    w1, w2t = _grid(N, K, 2 ** -2, gen), _grid(N, K, 2 ** -2, gen)
    b1 = _bias(N, gen)
    S = 128                                                      # attention sequence length
    qkv = torch.randn(8 * len(combos) + S, 3 * 64, device="cuda", generator=gen).to(torch.bfloat16)
    g = torch.randn(8 * len(combos) + S, 64, device="cuda", generator=gen).to(torch.bfloat16)
    for i, (off, M) in enumerate(combos + [combos[0], (combos[0][0], combos[0][1] - 30), (combos[-1][0], 5)]):
        _check(x[off:], w1, b1, d_out[off:], w2t, M, N, K)
        j = 8 * (i % len(combos))
        _attn_check(qkv[j:j + S].unsqueeze(0), g[j:j + S].unsqueeze(0))


def _mlp(C, H, O, seed):
    torch.manual_seed(seed)
    mlp = torch.nn.Module()
    mlp.fc1 = torch.nn.Linear(C, H).cuda()
    mlp.fc2 = torch.nn.Linear(H, O).cuda()
    return mlp


def _run_mlp(mlp, y0, g, fused):
    from imagefolder_b200 import vit_ops
    vit_ops.MLP_TC_ENABLED[0] = fused
    try:
        for prm in mlp.parameters():
            prm.grad = None
        y = y0.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = vit_ops.mlp_forward(mlp, y)
        out.backward(g)
    finally:
        vit_ops.MLP_TC_ENABLED[0] = True
    return out.detach(), y.grad, mlp.fc1.weight.grad, mlp.fc1.bias.grad, mlp.fc2.weight.grad


def test_gate_sends_out_features_not_multiple_of_64_to_library_path():
    """out = 72 is a valid fc2 width the backward kernel refuses (its K = out must be a multiple of 64): the gate must send the
    whole node to the library GEMMs + stand-alone GELU kernels, whose results it then equals."""
    from imagefolder_b200 import vit_ops
    mlp = _mlp(64, 256, 72, seed=5)
    y0 = torch.randn(300, 64, device="cuda").to(torch.bfloat16)
    g = torch.randn(300, 72, device="cuda").to(torch.bfloat16)
    on, off = _run_mlp(mlp, y0, g, True), _run_mlp(mlp, y0, g, False)
    assert not vit_ops.mlp_tc_ok(y0, mlp.fc1, mlp.fc2)
    for n, u, v in zip(["branch", "d_y", "d_W1", "d_W2"], on[:3] + on[4:], off[:3] + off[4:]):
        assert torch.equal(u, v), n
    # d_b1: xq_vit_gelu_bwd's fp32 atomics add in no fixed order
    assert bool(((on[3] - off[3]).abs() <= 1e-4 * off[3].abs().max()).all()), "d_b1"


def test_gate_hidden_width_limit_is_one_column_block_per_sm():
    """hidden / 128 <= SM count is the kernel's limit: the widest hidden the gate takes runs forward and backward; the next
    multiple of 256 is refused."""
    from imagefolder_b200 import vit_ops
    sms = _sms()
    widest = sms // 2 * 256
    y0 = torch.randn(300, 64, device="cuda").to(torch.bfloat16)
    assert not vit_ops.mlp_tc_ok(y0, torch.nn.Linear(64, widest + 256), torch.nn.Linear(widest + 256, 64))
    mlp = _mlp(64, widest, 64, seed=6)
    assert vit_ops.mlp_tc_ok(y0, mlp.fc1, mlp.fc2)
    g = torch.randn(300, 64, device="cuda").to(torch.bfloat16)
    on, off = _run_mlp(mlp, y0, g, True), _run_mlp(mlp, y0, g, False)
    # same device functions on the same rounded values; the GEMMs differ in accumulation order (bf16 resolution)
    for n, u, v in zip(["branch", "d_y", "d_W1", "d_b1", "d_W2"], on, off):
        scale = max(1e-6, v.float().abs().max().item())
        assert (u.float() - v.float()).abs().max().item() <= 8e-3 * scale, n


def test_fused_mlp_node_at_training_shape_matches_fp64():
    """_FusedMLP (vit_ops.mlp_forward under bf16 autocast) at the encoder's training rows, M = 128 x 513, C = 768, hidden 3072,
    against an fp64 timm Mlp (erf GELU, no fc2 bias) on the same bf16-rounded operands: pins the host wiring at the real
    shape (W2t transpose, saved tensors, casts).

    Each tolerance is a first-order bound built from the roundings on the fused path: u = 2^-8 for a bf16 rounding, and
    gam(n) = n 2^-23 for an fp32 sum of n terms (twice the round-to-nearest figure, so a truncating tensor-core accumulator
    is covered too), pushed through the GEMMs with absolute values.  A per-element bound is split into r_* (roundings) and
    s_* (the fixed approximation errors of gelu_f, dgelu_f).  Row-local outputs (branch, d_y) take the worst case.  The
    weight and bias gradients sum one element of every row over M = 65,664 rows, where the worst case grows like M while
    the values grow like sqrt(M); there the roundings, independent and zero-mean from row to row, are bounded with
    Hoeffding's inequality: P(|sum_i X_i| > LAM sqrt(sum_i b_i^2)) <= 2 exp(-LAM^2 / 2) = 2.5e-14 for |X_i| <= b_i, and the
    fp32 accumulation error likewise by LAM sqrt(n) 2^-23 sum |terms| (Higham & Mary, 2019).  The s_* terms stay worst
    case."""
    from imagefolder_b200 import vit_ops
    M, C, H = 128 * 513, 768, 3072
    u, LAM = 2.0 ** -8, 8.0

    def gam(n):
        return n * 2.0 ** -23

    mlp = _mlp(C, H, C, seed=7)
    with torch.no_grad():
        mlp.fc1.bias.normal_()
    y0 = torch.randn(M, C, device="cuda").to(torch.bfloat16)
    g = torch.randn(M, C, device="cuda").to(torch.bfloat16)
    assert vit_ops.mlp_tc_ok(y0, mlp.fc1, mlp.fc2)
    y = y0.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = vit_ops.mlp_forward(mlp, y)
    assert type(out.grad_fn).__name__ == "_FusedMLPBackward", type(out.grad_fn).__name__
    out.backward(g)
    branch, d_y = out.detach().view(M, C), y.grad
    d_W1, d_b1, d_W2 = mlp.fc1.weight.grad, mlp.fc1.bias.grad, mlp.fc2.weight.grad
    assert branch.dtype == d_y.dtype == torch.bfloat16

    W1 = mlp.fc1.weight.detach().to(torch.bfloat16).double()
    W2 = mlp.fc2.weight.detach().to(torch.bfloat16).double()
    b1 = mlp.fc1.bias.detach().double()
    aW1, aW2 = W1.abs(), W2.abs()
    nM = (M + 127) // 128
    per_col = _per_col(M, H)
    depth_b1 = 2 * -(-nM // per_col) + 3 + 8 * per_col          # the kernel's fp32 adds per d_b1 column, see _check
    acc = {k: torch.zeros(s, dtype=torch.float64, device="cuda") for k, s in
           [(f"dW1{t}", (H, C)) for t in ("", "_s", "_r2", "_abs")] + [(f"dW2{t}", (C, H)) for t in ("", "_s", "_r2", "_abs")]
           + [(f"db1{t}", (H,)) for t in ("", "_s", "_r2", "_abs")]}
    for r0 in range(0, M, CHUNK):
        r1 = min(M, r0 + CHUNK)
        yc, gc = y0[r0:r1].double(), g[r0:r1].double()
        ayc, agc = yc.abs(), gc.abs()
        # forward.  pre = bf16(fp32 y W1^T): r_z.  act = bf16(gelu_f(pre + b1)): r_h, s_h (|gelu'| <= 1.129; gelu_f's
        # |abs err| <= 7.1e-7, A&S 7.1.28 in fp32)
        z = yc @ W1.t()
        r_z = u * z.abs() + gam(C) * (ayc @ aW1.t())
        s = z + b1
        h = _gelu64(s)
        r_h, s_h = u * h.abs() + 1.129 * r_z, 1e-6
        # branch = bf16(fp32 act W2^T)
        ref = h @ W2.t()
        tol = u * ref.abs() + (r_h + s_h) @ aW2.t() + gam(H) * (h.abs() @ aW2.t())
        _assert_within(branch[r0:r1], ref, tol, "branch")
        # backward.  d_act = bf16(fp32 g W2): r_a.  d_pre = bf16(d_act dgelu_f(pre + b1)): r_d, s_d (|gelu''| <= 0.798;
        # dgelu_f's |abs err| <= 5e-7, A&S 7.1.26 with approximate ex2 / rcp)
        a = gc @ W2
        r_a = u * a.abs() + gam(C) * (agc @ aW2)
        D = a * (0.5 * (1.0 + torch.erf(s / math.sqrt(2.0))) + s * torch.exp(-0.5 * s * s) / math.sqrt(2.0 * math.pi))
        r_d, s_d = u * D.abs() + 1.129 * r_a + 0.798 * a.abs() * r_z, 5e-7 * a.abs()
        del s, z, r_z, a, r_a
        aD = D.abs()
        # d_y = bf16(fp32 d_pre W1)
        ref = D @ W1
        tol = u * ref.abs() + (r_d + s_d) @ aW1 + gam(H) * (aD @ aW1)
        _assert_within(d_y[r0:r1], ref, tol, "d_y")
        del ref, tol
        # d_W1 = bf16(fp32 d_pre^T y), d_W2 = bf16(fp32 g^T act), d_b1 = fp32 column sums of d_pre: sums over all rows
        acc["dW1"] += D.t() @ yc
        acc["dW1_s"] += s_d.t() @ ayc
        acc["dW1_r2"] += (r_d * r_d).t() @ (yc * yc)
        acc["dW1_abs"] += aD.t() @ ayc
        acc["dW2"] += gc.t() @ h
        acc["dW2_s"] += agc.sum(0).unsqueeze(1) * s_h
        acc["dW2_r2"] += (gc * gc).t() @ (r_h * r_h)
        acc["dW2_abs"] += agc.t() @ h.abs()
        acc["db1"] += D.sum(0)
        acc["db1_s"] += s_d.sum(0)
        acc["db1_r2"] += (r_d * r_d).sum(0)
        acc["db1_abs"] += aD.sum(0)
        del D, aD, r_d, s_d, h, r_h
    for out_, k in ((d_W1, "dW1"), (d_W2, "dW2")):
        R = acc[k]
        tol = u * R.abs() + acc[k + "_s"] + LAM * acc[k + "_r2"].sqrt() + LAM * math.sqrt(M) * 2.0 ** -23 * acc[k + "_abs"]
        _assert_within(out_, R, tol, k)
    # d_b1: the kernel's fp32 adds are few (depth_b1), so their bound is the worst case
    tol = acc["db1_s"] + LAM * acc["db1_r2"].sqrt() + depth_b1 * 2.0 ** -24 * acc["db1_abs"]
    _assert_within(d_b1, acc["db1"], tol, "d_b1")
