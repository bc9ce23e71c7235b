# coding=utf-8
"""What K4 (tfgk_gemm_proj_f32, the 3xTF32 wgmma projection) must compute, checked element by element.

* Dispatch: the shared-memory plan runs a ring of 4, 3 or 2 A stages (K <= 152, 153..168, 169..184) and refuses
  K > ops.GEMM_PROJ_MAX_K.  The raw ABI is called here, so a refusal cannot hide behind the SIMT fallback of ops.gemm_proj.
* Accuracy against float64: |got - ref| <= (K 2^-23 + 2^-19) S + 2^-23 |ref| for every entry, S = |A| @ |W| + |bias|.
  That is a worst-case bound (three truncating k8 accumulations per k-step, lo cut to TF32 inside the MMA), not a fit.
  The "coherent-lo" inputs give every lo the same sign, so a lost lo product moves the result by ~2^-12 S, far outside it.
* Bits: a row's result does not depend on M, the blocks, the grid, the part layout, the weight layout or the epilogue.
* Routing of tfgk_gemm_f32: the M K threshold, N cut into blocks, split-K of the transposed-A products.
* Non-finite and extreme inputs: the same NaN / +inf / -inf entries as IEEE fp32 and the SIMT kernel."""
import ctypes

import numpy as np
import pytest
import torch

from tf_geometric_b200 import _ffi, ops

pytestmark = pytest.mark.gpu

MAX_K = ops.GEMM_PROJ_MAX_K
FLT_MAX = float(np.finfo(np.float32).max)


def dev(a):
    return ops.as_device(a)


def ring_depth(k):
    """A stages of gemm_proj_kernel<STAGES> for K (proj::Plan: W hi | lo costs 1024 Kpad bytes of the 227 KB)."""
    return 4 if k <= 152 else 3 if k <= 168 else 2


def proj(a, blocks, m=None, parts=None, part_rows=0, first_part=0, max_ctas=0):
    """One raw tfgk_gemm_proj_f32 call, no fallback: TfgkError(ERR_UNSUPPORTED) surfaces.  `blocks` holds
    (w, bias or None, act, out[, trans_b]) with w [K, n] (or [n, K] with trans_b); `a` gives K, lda and, without
    `parts`, the rows.  Returns the outputs."""
    m = a.shape[0] if m is None else m
    structs = (_ffi.ProjBlock * len(blocks))()
    for i, blk in enumerate(blocks):
        w, bias, act, out = blk[:4]
        tb = len(blk) > 4 and bool(blk[4])
        structs[i] = _ffi.ProjBlock(w.data_ptr(), w.stride(0), w.shape[0] if tb else w.shape[1], int(tb),
                                    None if bias is None else bias.data_ptr(), act, out.data_ptr(), out.stride(0))
    ptrs = [a.data_ptr()] if parts is None else [p.data_ptr() for p in parts]
    _ffi.call("tfgk_gemm_proj_f32", (ctypes.c_void_p * len(ptrs))(*ptrs), len(ptrs), part_rows, a.stride(0), m,
              a.shape[1], structs, len(blocks), first_part, max_ctas,
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return [blk[3] for blk in blocks]


def simt_gemm(monkeypatch, *args, **kwargs):
    """ops.gemm with the tensor-core route switched off (TFGK_GEMM_TC=0): the exact-fp32 FMA kernel."""
    with monkeypatch.context() as mp:
        mp.setenv("TFGK_GEMM_TC", "0")
        out = ops.gemm(*args, **kwargs)
        torch.cuda.synchronize()
    return out


def nan_like(m, n):
    return torch.full((m, n), float("nan"), device="cuda")


def reference(a, w, bias=None, c=None):
    """float64 pre-activation a @ w + bias (+ c) and its scale S = |a| @ |w| + |bias| (+ |c|)."""
    a64, w64 = a.astype(np.float64), w.astype(np.float64)
    pre, scale = a64 @ w64, np.abs(a64) @ np.abs(w64)
    for extra in (bias, c):
        if extra is not None:
            pre = pre + extra.astype(np.float64)
            scale = scale + np.abs(extra.astype(np.float64))
    return pre, scale


def check_bound(got, pre, scale, k, act=ops.ACT_NONE, what="", mask=None):
    """|got - ref| <= (K 2^-23 + 2^-19) S + 2^-23 |pre| everywhere (or where `mask`); returns max |got - ref| / bound."""
    got = got.cpu().numpy().astype(np.float64) if torch.is_tensor(got) else np.asarray(got, np.float64)
    ref = np.maximum(pre, 0.0) if act == ops.ACT_RELU else pre
    bound = (k * 2.0 ** -23 + 2.0 ** -19) * scale + 2.0 ** -23 * np.abs(pre)
    err = np.abs(got - ref)
    ok = err <= bound                                   # a NaN in `got` fails
    if mask is not None:
        ok, err, bound = ok | ~mask, np.where(mask, err, 0.0), np.where(mask, bound, 1.0)
    if not np.all(ok):
        bad = np.argwhere(~ok)
        i = tuple(bad[0])
        raise AssertionError("{}: {} of {} entries outside the bound, first at {}: got {!r}, ref {!r}, bound {:.3e}, "
                             "largest err / bound {:.3g}".format(what, len(bad), ok.size, i, got[i], ref[i], bound[i],
                                                                 np.max(err / np.maximum(bound, 1e-300))))
    return float(np.max(err / np.maximum(bound, 1e-300))) if err.size else 0.0


# ---- a. dispatch boundary ------------------------------------------------------------------------------------------

def _one_block_call(k, m=4, n=8, lda=None, a_offset=0):
    lda = k if lda is None else lda
    buf = dev(np.random.RandomState(k).randn(m, lda).astype(np.float32))
    a = buf[:, a_offset:a_offset + k]
    w = dev(np.ones((k, n), np.float32))
    return proj(a, [(w, None, ops.ACT_NONE, nan_like(m, n))])[0]


@pytest.mark.parametrize("k", list(range(1, 9)) + [31, 32, 33, 152, 153, 168, 169, 184])
def test_tensor_core_kernel_takes_k(k):
    lda = (k + 3) // 4 * 4
    buf = dev(np.random.RandomState(k).randn(4, lda).astype(np.float32))
    w = np.random.RandomState(k + 1).randn(k, 8).astype(np.float32)
    got = proj(buf[:, :k], [(dev(w), None, ops.ACT_NONE, nan_like(4, 8))])[0]
    pre, scale = reference(buf[:, :k].cpu().numpy(), w)
    check_bound(got, pre, scale, k, what="K={}".format(k))


@pytest.mark.parametrize("k", [MAX_K + 1, 192, 333, 512])
def test_tensor_core_kernel_refuses_k(k):
    with pytest.raises(_ffi.TfgkError) as err:
        _one_block_call(k, lda=(k + 3) // 4 * 4)
    assert err.value.code == _ffi.ERR_UNSUPPORTED


def test_gemm_proj_max_k_is_the_dispatch_limit():
    """A change to proj::Plan (stage bytes, budget, W layout) has to move ops.GEMM_PROJ_MAX_K with it."""
    assert MAX_K == 184
    _one_block_call(MAX_K)
    with pytest.raises(_ffi.TfgkError) as err:
        _one_block_call(MAX_K + 1, lda=MAX_K + 4)
    assert err.value.code == _ffi.ERR_UNSUPPORTED


@pytest.mark.parametrize("case", ["lda_not_multiple_of_4", "a_not_16_byte_aligned", "ncols_129"])
def test_tensor_core_kernel_refuses_layouts(case):
    with pytest.raises(_ffi.TfgkError) as err:
        if case == "lda_not_multiple_of_4":
            _one_block_call(8, lda=9)
        elif case == "a_not_16_byte_aligned":
            _one_block_call(8, lda=12, a_offset=1)
        else:
            _one_block_call(8, n=129)
    assert err.value.code == _ffi.ERR_UNSUPPORTED


# ---- b. accuracy against float64 -----------------------------------------------------------------------------------

SWEEP_K = list(range(1, 41)) + list(range(96, 137, 4)) + list(range(148, MAX_K + 1))
SWEEP_M = (1, 127, 128, 129, 1000)
WIDTHS = (1, 7, 8, 127, 128)
_WORST = {}


def randn(rs, shape):
    return rs.randn(*shape).astype(np.float32)


def coherent_lo(rs, shape):
    """Positive values in [0.25, 2) that are a TF32 number plus a remainder of 0.44 to 0.5 TF32 ulp: rna rounds them
    down, so every lo = a - rna_tf32(a) is positive and about 2^-12 a."""
    n = int(np.prod(shape))
    bits = (rs.randint(125, 128, n).astype(np.uint32) << 23) | (rs.randint(0, 1 << 10, n).astype(np.uint32) << 13) \
        | rs.randint(0xE00, 0x1000, n).astype(np.uint32)
    return bits.view(np.float32).reshape(shape)


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratio():
    yield
    if _WORST:
        print("\nK4 largest |got - ref| / bound by ring depth: " + ", ".join(
            "{} stages {}: {:.4f}".format(d, kind, r) for (d, kind), r in sorted(_WORST.items())))


@pytest.mark.parametrize("kind", ["randn", "coherent_lo"])
@pytest.mark.parametrize("k", SWEEP_K)
def test_projection_within_float64_bound(k, kind):
    """Every ring depth, every K tail mod 8 and mod 32; M tails around the 128-row tile; 1 to 4 blocks of ragged widths,
    bias and relu on alternate blocks, some weights transposed."""
    gen = coherent_lo if kind == "coherent_lo" else randn
    rs = np.random.RandomState(2 * k + (kind == "coherent_lo"))
    a_host = gen(rs, (max(SWEEP_M), k))
    lda = (k + 3) // 4 * 4                  # the kernel takes rows of whole 16-byte chunks; the columns past K are NaN
    a = dev(np.pad(a_host, ((0, 0), (0, lda - k)), constant_values=np.nan))[:, :k]
    worst = 0.0
    for mi, m in enumerate(SWEEP_M):
        blocks, host = [], []
        for b in range(1 + (k + mi) % 4):
            n = WIDTHS[(k + 2 * mi + 3 * b) % len(WIDTHS)]
            w = gen(rs, (k, n))
            bias = gen(rs, (n,)) if (b + mi) % 2 == 0 else None
            act = ops.ACT_RELU if (b + k) % 2 == 1 else ops.ACT_NONE
            tb = (k + mi + b) % 3 == 0
            blocks.append((dev(w.T.copy()) if tb else dev(w), None if bias is None else dev(bias), act, nan_like(m, n), tb))
            host.append((w, bias, act))
        outs = proj(a[:m], blocks)
        for b, ((w, bias, act), got) in enumerate(zip(host, outs)):
            pre, scale = reference(a_host[:m], w, bias)
            worst = max(worst, check_bound(got, pre, scale, k, act, what="K={} M={} block {} ({} x {}, transB={})".format(
                k, m, b, k, w.shape[1], blocks[b][4])))
    key = (ring_depth(k), kind)
    _WORST[key] = max(_WORST.get(key, 0.0), worst)


# ---- c. bit-invariants at each ring depth --------------------------------------------------------------------------

DEPTH_K = (100, 160, 184)


def _problem(k, m=1000, widths=(128, 40, 7), seed=0):
    rs = np.random.RandomState(seed + k)
    a = dev(randn(rs, (m, k)))
    blocks = []
    for i, n in enumerate(widths):
        blocks.append((dev(randn(rs, (k, n)) / np.float32(np.sqrt(k))), dev(randn(rs, (n,))) if i % 2 == 0 else None,
                       ops.ACT_RELU if i % 2 == 1 else ops.ACT_NONE))
    return a, blocks


def _run(a, blocks, m=None, **kw):
    m = a.shape[0] if m is None else m
    return proj(a, [(w, b, act, nan_like(m, w.shape[1])) for w, b, act in blocks], m=m, **kw)


def _assert_same_bits(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and torch.equal(g, w), "{}: block {} changed bits".format(what, i)


@pytest.mark.parametrize("k", DEPTH_K)
def test_row_bits_do_not_depend_on_m(k):
    a, blocks = _problem(k)
    full = _run(a, blocks)
    for m in (1, 127, 128, 129, 640):
        _assert_same_bits(_run(a[:m], blocks), [f[:m] for f in full], "M={}".format(m))


@pytest.mark.parametrize("k", DEPTH_K)
def test_row_bits_do_not_depend_on_blocks_or_their_order(k):
    a, blocks = _problem(k)
    full = _run(a, blocks)
    for i, blk in enumerate(blocks):
        _assert_same_bits(_run(a, [blk]), [full[i]], "block {} alone".format(i))
    _assert_same_bits(_run(a, blocks[::-1]), full[::-1], "reversed blocks")
    _assert_same_bits(_run(a, blocks + [blocks[0]]), full + [full[0]], "four blocks")


@pytest.mark.parametrize("k", DEPTH_K)
def test_row_bits_do_not_depend_on_grid(k):
    a, blocks = _problem(k)
    full = _run(a, blocks)
    for max_ctas in (1, 2, 3, 0):      # fewer CTAs than blocks still runs one CTA per block
        _assert_same_bits(_run(a, blocks, max_ctas=max_ctas), full, "max_ctas={}".format(max_ctas))


@pytest.mark.parametrize("k", DEPTH_K)
def test_row_bits_do_not_depend_on_part_layout(k):
    part_rows = 384
    a, blocks = _problem(k, m=3 * part_rows)
    for n_parts, m in ((2, 2 * part_rows - 50), (3, 3 * part_rows - 200)):
        want = _run(a[:m], blocks)
        parts = [a[i * part_rows:(i + 1) * part_rows].clone() for i in range(n_parts)]
        for first in range(n_parts):
            got = _run(parts[0], blocks, m=m, parts=parts, part_rows=part_rows, first_part=first)
            _assert_same_bits(got, want, "{} parts, first part {}".format(n_parts, first))


@pytest.mark.parametrize("k", DEPTH_K)
def test_transposed_weights_give_the_same_bits(k):
    a, blocks = _problem(k)
    want = _run(a, blocks)
    wide = [torch.zeros((w.shape[1], k + 4), device="cuda") for w, _, _ in blocks]      # ldb = K + 4 > K
    for buf, (w, _, _) in zip(wide, blocks):
        buf[:, :k] = w.t()
    for wts in ([w.t().contiguous() for w, _, _ in blocks], [buf[:, :k] for buf in wide]):
        got = proj(a, [(wt, b, act, nan_like(a.shape[0], wt.shape[0]), True) for wt, (_, b, act) in zip(wts, blocks)])
        _assert_same_bits(got, want, "transB")


@pytest.mark.parametrize("k", DEPTH_K)
def test_scalar_epilogue_gives_the_same_bits(k):
    """The epilogue stores (col, col + 1) as one float2 when ldc is even and C 8-byte aligned, else one float at a time."""
    a, blocks = _problem(k, widths=(128, 40))
    m = a.shape[0]
    want = _run(a, blocks)                                              # contiguous: float2 stores
    odd = [torch.full((m, w.shape[1] + 1), 7.0, device="cuda") for w, _, _ in blocks]      # ldc odd
    shifted = [torch.full((m, w.shape[1] + 2), 7.0, device="cuda") for w, _, _ in blocks]  # C at an odd float offset
    for bufs, c0 in ((odd, 0), (shifted, 1)):
        outs = [buf[:, c0:c0 + w.shape[1]] for buf, (w, _, _) in zip(bufs, blocks)]
        proj(a, [(w, b, act, o) for o, (w, b, act) in zip(outs, blocks)])
        _assert_same_bits(outs, want, "scalar epilogue (column offset {})".format(c0))
        for buf, (w, _, _) in zip(bufs, blocks):
            rest = torch.cat([buf[:, :c0], buf[:, c0 + w.shape[1]:]], dim=1)
            assert bool((rest == 7.0).all()), "columns outside the block were written"


# ---- d. tfgk_gemm_f32 routing --------------------------------------------------------------------------------------

def _blocks_of(w, c, bias=None, act=ops.ACT_NONE, trans_b=False):
    """The column blocks tfgk_gemm_f32 hands to the tensor-core kernel: <= 128 columns each."""
    n = w.shape[0] if trans_b else w.shape[1]
    out = []
    for c0 in range(0, n, 128):
        c1 = min(n, c0 + 128)
        out.append((w[c0:c1] if trans_b else w[:, c0:c1], None if bias is None else bias[c0:c1], act, c[:, c0:c1], trans_b))
    return out


@pytest.mark.parametrize("m,k,lda", [(16383, 1, 4), (129, 127, 128)])
def test_gemm_below_threshold_is_simt(monkeypatch, m, k, lda):
    """M K = 16383 stays on the exact-fp32 kernel, M K = 16384 goes to the tensor cores."""
    rs = np.random.RandomState(m + k)
    buf = dev(randn(rs, (m + 1, lda)))
    w = dev(randn(rs, (k + 1, 128)))
    below = ops.gemm(buf[:m, :k], w[:k])
    assert torch.equal(below, simt_gemm(monkeypatch, buf[:m, :k], w[:k]))
    m1, k1 = (m + 1, k) if k == 1 else (128, k + 1)
    above = ops.gemm(buf[:m1, :k1], w[:k1])
    assert m1 * k1 == 1 << 14
    assert torch.equal(above, proj(buf[:m1, :k1], _blocks_of(w[:k1], nan_like(m1, 128)))[0])
    if k > 1:       # the two kernels round differently: the checks above could not pass by accident
        assert not torch.equal(simt_gemm(monkeypatch, buf[:m, :k], w[:k]), proj(buf[:m, :k], _blocks_of(w[:k], nan_like(m, 128)))[0])


@pytest.mark.parametrize("n,trans_b", [(129, False), (385, False), (385, True), (512, False), (512, True)])
def test_gemm_cuts_n_into_tensor_core_blocks(n, trans_b):
    rs = np.random.RandomState(n)
    m, k = 300, 100
    a = dev(randn(rs, (m, k)))
    w_host = randn(rs, (k, n))
    bias = dev(randn(rs, (n,)))
    w = dev(w_host.T.copy()) if trans_b else dev(w_host)
    got = ops.gemm(a, w, bias=bias, act=ops.ACT_RELU, trans_b=trans_b)
    want = nan_like(m, n)
    proj(a, _blocks_of(w, want, bias, ops.ACT_RELU, trans_b))
    assert torch.equal(got, want)
    pre, scale = reference(a.cpu().numpy(), w_host, bias.cpu().numpy())
    check_bound(got, pre, scale, k, ops.ACT_RELU, what="N={}".format(n))


def test_gemm_wider_than_four_blocks_is_simt(monkeypatch):
    rs = np.random.RandomState(513)
    m, k, n = 300, 100, 513
    a, w_host = dev(randn(rs, (m, k))), randn(rs, (k, n))
    got = ops.gemm(a, dev(w_host))
    assert torch.equal(got, simt_gemm(monkeypatch, a, dev(w_host)))
    pre, scale = reference(a.cpu().numpy(), w_host)
    check_bound(got, pre, scale, k, what="N=513")


def _workspace(m, n, k):
    need = ctypes.c_size_t()
    _ffi.call("tfgk_gemm_workspace_bytes", m, n, k, ctypes.byref(need))
    return need.value


@pytest.mark.parametrize("k", [4095, 4096])
def test_split_k_weight_gradient(k):
    """dW = X^T dY (transposed A, the SIMT kernel): split-K starts at K = 4096 when the tiles leave SMs idle."""
    m, n = 100, 64
    assert (_workspace(m, n, k) > 0) == (k >= 4096)
    rs = np.random.RandomState(k)
    x, dy, bias, c0 = randn(rs, (k, m)), randn(rs, (k, n)), randn(rs, (n,)), randn(rs, (m, n))
    xd, dyd = dev(x), dev(dy)
    got = ops.gemm(xd, dyd, trans_a=True)
    pre, scale = reference(x.T, dy)
    check_bound(got, pre, scale, k, what="X^T dY, K={}".format(k))
    for _ in range(3):
        assert torch.equal(ops.gemm(xd, dyd, trans_a=True), got), "split-K result changed between runs"
    out = dev(c0)
    ops.gemm(xd, dyd, bias=dev(bias), act=ops.ACT_RELU, trans_a=True, beta=1.0, out=out)
    pre, scale = reference(x.T, dy, bias, c0)
    check_bound(out, pre, scale, k, ops.ACT_RELU, what="relu(X^T dY + bias + C), K={}".format(k))
    again = dev(c0)
    ops.gemm(xd, dyd, bias=dev(bias), act=ops.ACT_RELU, trans_a=True, beta=1.0, out=again)
    assert torch.equal(again, out)


# ---- e. non-finite and extreme values ------------------------------------------------------------------------------

def _classes(x):
    x = x.cpu().numpy() if torch.is_tensor(x) else x
    return np.stack([np.isnan(x), np.isposinf(x), np.isneginf(x)])


@pytest.mark.parametrize("value", [np.inf, -np.inf, np.nan])
@pytest.mark.parametrize("where", ["A", "W"])
@pytest.mark.parametrize("k", [8, 100, MAX_K])
def test_non_finite_entries_match_ieee(monkeypatch, k, where, value):
    """One inf / -inf / NaN in A (or W) reaches its own row (or column) only, with IEEE fp32's NaN / +inf / -inf
    pattern: inf times a zero partner is NaN, inf times anything else is inf of the product's sign."""
    rs = np.random.RandomState(k)
    m, n, i0, k0, j0 = 300, 96, 137, k // 2, 41
    a, w, bias = randn(rs, (m, k)), randn(rs, (k, n)) / np.float32(np.sqrt(k)), randn(rs, (n,))
    a_fin, w_fin = a.copy(), w.copy()
    if where == "A":
        w[k0, 5] = w_fin[k0, 5] = 0.0
        a_fin[i0, k0] = 0.0
    else:
        a[200, k0] = a_fin[200, k0] = 0.0
        w_fin[k0, j0] = 0.0
    pre, scale = reference(a_fin, w_fin, bias)              # everything but the non-finite entry's products
    with np.errstate(invalid="ignore"):
        if where == "A":
            a[i0, k0] = value
            pre[i0] += np.float64(value) * w[k0].astype(np.float64)
        else:
            w[k0, j0] = value
            pre[:, j0] += a[:, k0].astype(np.float64) * np.float64(value)
    ad, wd, bd = dev(a), dev(w), dev(bias)
    tc = proj(ad, [(wd, bd, ops.ACT_NONE, nan_like(m, n))])[0]
    simt = simt_gemm(monkeypatch, ad, wd, bias=bd)
    want = _classes(pre)
    assert want.any(axis=0).sum() == (n if where == "A" else m)
    for name, got in (("SIMT", simt), ("tensor cores", tc)):
        cls = _classes(got)
        assert np.array_equal(cls, want), "{}: NaN/+inf/-inf pattern differs from IEEE at {} entries".format(
            name, int((cls != want).any(axis=0).sum()))
        check_bound(got, pre, scale, k, what=name + " finite entries", mask=np.isfinite(pre))


@pytest.mark.parametrize("where", ["A", "W"])
@pytest.mark.parametrize("k", [8, 100, MAX_K])
def test_largest_finite_inputs_stay_finite(monkeypatch, k, where):
    """|x| in [3.3e38, FLT_MAX] times small partners: the exact result is finite, so both kernels must give it within
    the bound.  rna_tf32 rounds |x| >= (2 - 2^-11) 2^127 up to inf; the split has to keep hi finite."""
    rs = np.random.RandomState(k + 7)
    m, n, i0 = 200, 64, 77
    big = rs.uniform(3.3e38, FLT_MAX, k).astype(np.float32) * rs.choice([-1, 1], k).astype(np.float32)
    edge = np.array([FLT_MAX, -FLT_MAX, np.uint32(0x7F7FF000).view(np.float32), np.uint32(0x7F7FEFFF).view(np.float32)],
                    np.float32)
    big[:min(k, 4)] = edge[:min(k, 4)]
    small = np.float32(2.0 ** -12 / k)
    if where == "A":
        a, w = randn(rs, (m, k)), randn(rs, (k, n)) * small
        a[i0] = big
    else:
        a, w = randn(rs, (m, k)) * small, randn(rs, (k, n))
        w[:, i0 % n] = big
    pre, scale = reference(a, w)
    assert np.all(np.abs(pre) < FLT_MAX / 2)
    ad, wd = dev(a), dev(w)
    tc = proj(ad, [(wd, None, ops.ACT_NONE, nan_like(m, n))])[0]
    simt = simt_gemm(monkeypatch, ad, wd)
    for name, got in (("SIMT", simt), ("tensor cores", tc)):
        assert bool(torch.isfinite(got).all()), "{}: non-finite output from finite inputs".format(name)
        check_bound(got, pre, scale, k, what=name)
