"""numpy model of the screening decisions of `vq_search_tc_kernel` (imagefolder_b200/csrc/vq_tc_kernel.cu), and seeded
builders of the codebooks that drive each of its branches.

The kernel cannot be instrumented from a test, so this model is how the suite shows that the GPU inputs reach the
branches they are built for: the candidate-list overflow, compaction when the running maximum rises late, the
"several codes of one group within W" flag, last-tile padding masking and the fast path.

Model of one row (the kernel's epilogue thread):
  * operands truncated to TF32 (low 13 mantissa bits cleared: the worst case the kernel's error bound assumes),
    products accumulated in fp64;
  * score s = dot (`fold_ee=False`, the kernel) or s = dot - ee / 2 (`fold_ee=True`, the alternative design that folds
    the code norm into every score); padded codes (ee = +inf) score 0 without the fold and -inf with it;
  * `ee_flag=True` (the kernel): when any real code has |ee - 1| > 1e-5 (a zero row, or one of norm < XQ_EPS), the
    prep kernel raises a flag and every row takes the full canonical scan (reported as OVERFLOW);
  * 128-code tiles of 32-code groups, the running maximum, thr = runmax - W and `cand_push` with TC_CAP slots,
    compaction and the sticky overflow flag;
  * the second slot (m1 when more than one code of the group is within W of the group maximum);
  * after the scan: fast path when exactly one live group and no flag, otherwise canonical rescoring of the live
    groups, or of every code after an overflow.  Rescoring uses the oracle's canonical fp32 search, so the model's
    index is exact whenever the screening kept the true argmin.

The switches `W`, `fold_ee`, `ee_flag`, `mask_padding`, `check_multi`, `honour_overflow` turn each safeguard off
(mutants); `fold_ee=False, ee_flag=False` is the kernel before the flag.
"""
from __future__ import annotations

import numpy as np

from oracle import xq_oracle as xo

TC_BN = 128
GROUP = 32
TC_CAP = 16
TC_EPS = 2.5e-3
TC_W = float(np.float32(2.0 * np.float32(TC_EPS) + np.float32(2e-6)))

FAST, RESCORED, OVERFLOW = 0, 1, 2


def tf32(x: np.ndarray) -> np.ndarray:
    """Truncate fp32 values to TF32 (clear the low 13 mantissa bits)."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return u.view(np.float32)


def normalise(x: np.ndarray) -> np.ndarray:
    """F.normalize in the canonical fp32 chain (what the kernels and the oracle compute)."""
    return xo.l2norm_rows(np.ascontiguousarray(x, np.float32))[0]


def screen(z_rows, E, *, W=TC_W, fold_ee=False, ee_flag=True, mask_padding=True, check_multi=True,
           honour_overflow=True):
    """z_rows [N, C] (raw rows), E [V, C] (raw codebook, normalised like codebook_norm=True).

    Returns (idx [N] int64, path [N] in {FAST, RESCORED, OVERFLOW}, compacted [N] bool, multi [N] bool); `compacted`
    marks rows whose list was compacted with at least one entry dropped, `multi` rows whose final set had a live
    group with the second slot set."""
    zn, En = normalise(z_rows), normalise(E)
    N, C = zn.shape
    V = En.shape[0]
    Vp = (V + TC_BN - 1) // TC_BN * TC_BN
    G = Vp // GROUP
    ee = np.full(Vp, np.inf)
    ee[:V] = (En.astype(np.float64) ** 2).sum(1)
    Ep = np.zeros((Vp, C), np.float32)
    Ep[:V] = En
    S = tf32(zn).astype(np.float64) @ tf32(Ep).astype(np.float64).T          # [N, Vp]
    if fold_ee:
        S = S - ee / 2.0
    Sm = S.copy()
    if mask_padding:
        Sm[:, V:] = -np.inf
    Sg = Sm.reshape(N, G, GROUP)
    m1 = Sg.max(2)                                                          # group maxima (padding masked)
    i1 = Sg.argmax(2)                                                       # first index of the maximum
    nW = (Sg >= (m1 - W)[:, :, None]).sum(2)
    runmax = np.maximum.accumulate(m1, axis=1)
    thr_after = runmax - W
    thr_before = np.concatenate([np.full((N, 1), -np.inf), thr_after[:, :-1]], 1)
    pushed = m1 >= thr_before
    idx = np.empty(N, np.int64)
    path = np.empty(N, np.int64)
    compacted = np.zeros(N, bool)
    multi_out = np.zeros(N, bool)
    full_rows = []
    degenerate = ee_flag and bool((np.abs(ee[:V] - 1.0) > 1e-5).any())
    for n in range(N):
        c1, c2, cv = [], [], []
        overflow = False
        for g in np.nonzero(pushed[n])[0]:
            thr = thr_after[n, g]
            if len(c1) == TC_CAP:
                keep = [e for e in range(TC_CAP) if c1[e] >= thr]
                if len(keep) < TC_CAP:
                    compacted[n] = True
                c1, c2, cv = [c1[e] for e in keep], [c2[e] for e in keep], [cv[e] for e in keep]
            if len(c1) < TC_CAP:
                c1.append(m1[n, g])
                c2.append(m1[n, g] if nW[n, g] > 1 else -np.inf)
                cv.append(g * GROUP + i1[n, g])
            else:
                overflow = True
        thr = thr_after[n, -1]
        live = [e for e in range(len(c1)) if c1[e] >= thr]
        multi = any(c2[e] >= thr for e in live)
        multi_out[n] = multi
        overflow = (overflow and honour_overflow) or degenerate
        need = overflow or (multi and check_multi) or len(live) != 1
        if not need:
            idx[n], path[n] = cv[live[0]], FAST
        elif overflow:
            path[n] = OVERFLOW
            full_rows.append(n)
        else:
            path[n] = RESCORED
            codes = np.concatenate([np.arange((cv[e] // GROUP) * GROUP, (cv[e] // GROUP + 1) * GROUP) for e in live])
            codes = np.unique(codes[codes < V])
            idx[n] = codes[xo.search(zn[n:n + 1], En[codes], 0)[0][0]]
    if full_rows:
        idx[full_rows] = xo.search(zn[full_rows], En, 0)[0]
    return idx, path, compacted, multi_out


def oracle_idx(z_rows, E):
    return xo.search(normalise(z_rows), normalise(E), 0)[0]


def rows_to_nchw(rows: np.ndarray, B: int, hw: int) -> np.ndarray:
    """[B*hw*hw, C] rows (row n = b*hw*hw + p) -> [B, C, hw, hw]."""
    C = rows.shape[1]
    return np.ascontiguousarray(rows.reshape(B, hw * hw, C).transpose(0, 2, 1).reshape(B, C, hw, hw))


# ----------------------------------------------------------------------------------------------------------------
# input families.  Every builder takes (V, C, N, seed) and returns (z_rows [N, C], E [V, C]) in float32.
# ----------------------------------------------------------------------------------------------------------------
def _unit(rng, n, C):
    x = rng.standard_normal((n, C))
    return x / np.linalg.norm(x, axis=1, keepdims=True)


def _with_dot(rng, r, a):
    """unit vector whose dot with the unit vector r is a."""
    u = rng.standard_normal(r.shape)
    u -= (u @ r) * r
    u /= np.linalg.norm(u)
    return a * r + np.sqrt(max(0.0, 1.0 - a * a)) * u


def f1_zero_tiny(V, C, N, seed=1):
    """F1: zero rows and rows of norm ~1e-13 (< XQ_EPS) in a Gaussian codebook at group / tile boundaries; a few z rows
    exactly zero or of norm ~1e-13.  F.normalize leaves such vectors with norm < 1, so ee < 1 (0 for a zero row):
    the zero code is the nearest code of every row whose best dot is below 1/2."""
    rng = np.random.default_rng(seed)
    E = rng.standard_normal((V, C)).astype(np.float32)
    special = sorted({v for v in (0, 31, 32, 127, 128, V - 1) if 0 <= v < V})
    for j, v in enumerate(special):
        E[v] = 0.0 if j % 2 == 0 else (_unit(rng, 1, C)[0] * 1e-13)
    z = rng.standard_normal((N, C)).astype(np.float32)
    nz = max(2, N // 64)
    z[:nz // 2] = 0.0
    z[nz // 2:nz] = _unit(rng, nz - nz // 2, C) * 1e-13
    return z.astype(np.float32), E.astype(np.float32)


def f2_clusters(V, C, N, seed=2, n_centres=4, sigma=None):
    """F2: the whole codebook is n_centres collapsed clusters (members c + sigma u, >= 40 each), interleaved by index
    (member j of cluster k at index j * n_centres + k), so each cluster spans every group and tile.  Rows are the
    centres plus small noise: every group holds a code within ~1e-3 of the row's best -> more than TC_CAP live groups."""
    rng = np.random.default_rng(seed)
    assert V >= 40 * n_centres
    if sigma is None:
        sigma = 0.02 / np.sqrt(C)
    cen = _unit(rng, n_centres, C)
    E = cen[np.arange(V) % n_centres] + sigma * rng.standard_normal((V, C))
    k = rng.integers(0, n_centres, N)
    z = cen[k] + (0.2 * sigma) * rng.standard_normal((N, C))
    return z.astype(np.float32), E.astype(np.float32)


def f3_late_winner(V, C, N, seed=3):
    """F3: per design row r (unit), codes at dot d0 + jitter (|jitter| <= W/8) in consecutive groups of the first tiles,
    and one code in the last tile.  Three kinds of rows (round-robin over the designs):
      'late3W'  16 near-tie groups, then a code 3W better in the last tile: the list is full, the winner's push
                compacts it to nothing and the row takes the fast path;
      'lateW4'  20 near-tie groups (overflow), then a code W/4 better: the winner is dropped from the full list, only
                the overflow's full scan finds it;
      'reverse' the winner first (group 0), then 20 groups 3W below: none of them is ever pushed."""
    rng = np.random.default_rng(seed)
    G = V // GROUP
    assert G >= 48, "F3 needs V >= 1536"
    W = TC_W
    d0 = 0.9
    n_design = GROUP                   # one slot per design in every group
    kinds = ("late3W", "lateW4", "reverse")
    R = _unit(rng, n_design, C)
    # filler: random unit codes with a low dot with every design row
    E = np.empty((V, C))
    filled = 0
    while filled < V:
        cand = _unit(rng, 2 * V, C)
        ok = cand[np.abs(cand @ R.T).max(1) < 0.45]
        take = min(V - filled, len(ok))
        E[filled:filled + take] = ok[:take]
        filled += take
    last_group = G - 1
    for j in range(n_design):
        kind = kinds[j % 3]
        r = R[j]
        if kind == "reverse":
            E[0 * GROUP + j] = _with_dot(rng, r, d0 + 3 * W)
            for g in range(1, 21):
                E[g * GROUP + j] = _with_dot(rng, r, d0 + rng.uniform(-W / 8, W / 8))
        else:
            ng = 16 if kind == "late3W" else 20
            for g in range(ng):
                E[g * GROUP + j] = _with_dot(rng, r, d0 + rng.uniform(-W / 8, W / 8))
            E[last_group * GROUP + j] = _with_dot(rng, r, d0 + (3 * W if kind == "late3W" else W / 4 + W / 8))
    z = R[np.arange(N) % n_design]
    return z.astype(np.float32), E.astype(np.float32)


def _exact_unit(v: np.ndarray, fix: int) -> np.ndarray:
    """Adjust component `fix` of the fp32 vector v (the other components are kept bit for bit) so that the canonical
    fp32 norm is exactly 1: F.normalize then returns v unchanged, so the bit patterns built into v are the ones the
    kernel multiplies."""
    v = v.astype(np.float32).copy()
    rest = float((v.astype(np.float64) ** 2).sum() - float(v[fix]) ** 2)
    assert rest < 1.0
    f0 = np.float32(np.sqrt(1.0 - rest))
    base = f0.view(np.int32)
    cands = np.repeat(v[None], 257, 0)
    cands[:, fix] = (base + np.arange(-128, 129, dtype=np.int32)).view(np.float32)
    y, den = xo.l2norm_rows(cands)
    ok = np.nonzero((den == 1.0) & (y == cands).all(1))[0]
    assert len(ok), "no exact-unit completion"
    return cands[ok[len(ok) // 2]]


_LOSSY = np.float32(0.25 * (1.0 + 8191.0 * 2.0 ** -23))        # 0.25 with the low 13 mantissa bits set


def _reversal_design(rng, C):
    """(z, A, B): unit fp32 vectors, exactly normalised.  z and B share 8 components of 0.25 with the low 13 bits set
    (TF32 truncation loses 2^-10 of each), z and A share 8 TF32-exact components.  dot(z, B) - dot(z, A) is a small
    positive gap while the TF32 scores rank A above B by ~2^-10 - gap."""
    assert C >= 19
    perm = rng.permutation(C)
    SB, SA, fz, fa, fb = perm[:8], perm[8:16], perm[16], perm[17], perm[18]
    sB = rng.choice([-1.0, 1.0], 8).astype(np.float32)
    sA = rng.choice([-1.0, 1.0], 8).astype(np.float32)
    za = np.float32(0.25 - 2.0 ** -10)                           # TF32-exact
    z = np.zeros(C, np.float32)
    z[SB] = sB * _LOSSY
    z[SA] = sA * za
    z[fz] = 0.05
    z = _exact_unit(z, fz)
    B = np.zeros(C, np.float32)
    B[SB] = sB * _LOSSY
    B[fb] = 0.7
    B = _exact_unit(B, fb)
    dotB = float(z.astype(np.float64) @ B.astype(np.float64))
    # A: 8 TF32-exact magnitudes 0.25 + k * 2^-12 on SA, k chosen per component so that dot(z, A) is just below dot(z, B)
    k = np.zeros(8, np.int64)
    step = float(za) * 2.0 ** -12
    target = dotB - 1e-5
    base = 8 * float(za) * 0.25
    total = int(np.floor((target - base) / step))
    k[:] = total // 8
    k[: total % 8] += 1
    A = np.zeros(C, np.float32)
    A[SA] = sA * (0.25 + k * 2.0 ** -12).astype(np.float32)
    A[fa] = 0.7
    A = _exact_unit(A, fa)
    return z, A, B


def _filler(rng, V, C, rows, bound):
    E = np.empty((V, C))
    filled = 0
    while filled < V:
        cand = _unit(rng, 2 * V + 64, C)
        ok = cand[np.abs(cand @ rows.T.astype(np.float64)).max(1) < bound]
        take = min(V - filled, len(ok))
        E[filled:filled + take] = ok[:take]
        filled += take
    return E.astype(np.float32)


def _reversal_family(V, C, N, seed, same_group):
    rng = np.random.default_rng(seed)
    G = V // GROUP
    n_design = min(16, G if same_group else G // 2)
    assert n_design >= 1
    designs = [_reversal_design(rng, C) for _ in range(n_design)]
    Z = np.stack([d[0] for d in designs])
    E = _filler(rng, V, C, Z, 0.3)
    for j, (z, A, B) in enumerate(designs):
        if same_group:          # F4: A and B in group j, in either order
            a, b = (j * GROUP + 3, j * GROUP + 17) if j % 2 == 0 else (j * GROUP + 17, j * GROUP + 3)
        else:                   # F5: A and B in different groups (and tiles when V allows), in either order
            g2 = G - 1 - j
            a, b = (j * GROUP + 5, g2 * GROUP + 9) if j % 2 == 0 else (g2 * GROUP + 9, j * GROUP + 5)
        E[a], E[b] = A, B
    z = Z[np.arange(N) % n_design]
    return z.astype(np.float32), E


def f4_in_group_tie(V, C, N, seed=4):
    """F4: two codes of one 32-code group, true dots < 2^-9 apart, whose order TF32 truncation reverses (one code has
    TF32-exact components on its support, the other the low 13 bits set).  Only the `nW > 1` second slot sends the row
    to rescoring; without it the fast path returns the TF32 maximum, which is the wrong code."""
    return _reversal_family(V, C, N, seed, same_group=True)


def f5_worst_truncation(V, C, N, seed=5):
    """F5: the true argmin B loses ~2^-10 to truncation on each operand (its components and the row's share the low 13
    bits set), the competitor A is TF32-exact and ~1e-5 below B in true dot, in another group: the TF32 scores put A
    ~0.96e-3 above B, so B survives only if W covers that reversal.  (For unit vectors at dot 1/2 this is close to the
    largest reversal a competitor at equal true dot can reach.)"""
    return _reversal_family(V, C, N, seed, same_group=False)


def f6_negative(V, C, N, seed=6):
    """F6: every real dot is negative (codes in the negative orthant, rows in the positive one); a padded code (dot 0,
    ee = +inf) would win the screening if the last tile's padding were not masked."""
    rng = np.random.default_rng(seed)
    E = -np.abs(rng.standard_normal((V, C))) - 0.05
    z = np.abs(rng.standard_normal((N, C))) + 0.05
    return z.astype(np.float32), E.astype(np.float32)


def f7_exact_ties(V, C, N, seed=7, run=300):
    """F7: exact duplicates at (31, 32), (127, 128) and (0, V-1); a run of `run` identical codes (when V allows); codes
    that differ from a duplicate by 1 ulp in one component.  Rows sit on the duplicated codes (plus tiny noise for half
    of them) so that the tie rule (lowest index) decides."""
    rng = np.random.default_rng(seed)
    E = rng.standard_normal((V, C)).astype(np.float32)
    pairs = [(a, b) for a, b in ((31, 32), (127, 128), (0, V - 1)) if b < V and a != b]
    for a, b in pairs:
        E[b] = E[a]
    anchors = [a for a, _ in pairs]
    if V >= run + 400:
        start = 200
        E[start:start + run] = E[start]
        anchors.append(start)
    # 1-ulp neighbours of the duplicated codes, one component changed
    for a in list(anchors):
        for off in (2, 3):
            v = a + off
            if v < V and v not in (b for _, b in pairs) and not (V >= run + 400 and 200 <= v < 200 + run):
                E[v] = E[a]
                k = int(rng.integers(0, C))
                E[v, k] = np.nextafter(E[a, k], np.float32(np.inf) if off == 2 else np.float32(-np.inf))
    if not anchors:
        anchors = [0]
    z = E[np.array(anchors)[np.arange(N) % len(anchors)]].copy()
    half = np.arange(N) % 2 == 1
    z[half] += (1e-4 * rng.standard_normal((int(half.sum()), C))).astype(np.float32)
    return z.astype(np.float32), E.astype(np.float32)


FAMILIES = {"F1": f1_zero_tiny, "F2": f2_clusters, "F3": f3_late_winner, "F4": f4_in_group_tie,
            "F5": f5_worst_truncation, "F6": f6_negative, "F7": f7_exact_ties}
