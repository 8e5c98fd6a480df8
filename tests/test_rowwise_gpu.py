"""Kernel-level parity of the row kernels that the model tests only reach through whole encoders: mer_layernorm (both
kernel forms, every width and output form), mer_segment_reduce, mer_wave_normalize, the fp32 mer_swiglu and
mer_videomae_patchify, each against a float64 restatement (tests/_kernel_refs.py) of the formula include/mer_b200.h
documents, on the same operand values.

Operands come from seeded host generators; every output is pre-filled with NaN (or a sentinel) between NaN guard rows,
so an element the kernel skips or a row it writes out of place fails.  Each test prints its worst observed error."""
import functools

import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
U = R.U32
DIMS = [512, 768, 1024, 1280, 1536]
FORMS = [None, "1"]  # MER_LN_VER unset: the prefetching kernel; 1: the first form
F16_MAX = 65504.0


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _second_row_count(cuda):
    """First row count at which a warp takes a second row: the grid is capped at 16 blocks of 8 warps per SM."""
    return torch.cuda.get_device_properties(cuda).multi_processor_count * 16 * 8 + 11


# ---------------------------------------------------------------- LayerNorm ----
@functools.lru_cache(maxsize=1)
def _ln_rows(dim, rows):
    """Rows cycling through the conditionings a model test never feeds: N(0, 1); mean 10, std 0.1; magnitude 1e4 with
    std 1e3; one 1e4 outlier among N(0, 1e-2) values; N(0, 1) shifted by -3."""
    g = _gen(100 + dim)
    x = torch.randn(rows, dim, generator=g)
    kind = torch.arange(rows) % 5
    x[kind == 1] = x[kind == 1] * 0.1 + 10.0
    x[kind == 2] = x[kind == 2] * 1e3 + 1e4
    x[kind == 3] *= 0.1
    x[kind == 3, (torch.arange(rows)[kind == 3] * 7) % dim] = 1e4
    x[kind == 4] = x[kind == 4] - 3.0
    return x


def _affine(dim, seed=5):
    g = _gen(seed)
    gamma, beta = torch.randn(dim, generator=g), torch.randn(dim, generator=g)
    gamma[::7] = 0.0          # exact zeros; about half of the rest is negative
    beta[3::11] = 0.0
    return gamma, beta


def _ln(x, gamma, beta, eps, flags=0, form=None, y="f32", ys=None, acc=None, in_place=None):
    """One mer_layernorm call over guarded, NaN-filled outputs.  y: "f32" | "f16" | None; ys: "bf16" | "f16" | None;
    acc: None | an fp32 [rows + 4, dim] buffer whose rows 2 .. -2 are the accumulator; in_place: None | "y" | "ys"
    (the output is x itself).  Returns a dict of the device outputs."""
    rows, dim = x.shape
    dev = x.device
    out, bufs = {}, []
    xbuf, xv = R.guarded(rows, dim, torch.float32, dev)
    xv.copy_(x)
    yv = ysv = None
    if in_place == "y":
        yv = xv
    elif y is not None:
        b, yv = R.guarded(rows, dim, torch.float16 if y == "f16" else torch.float32, dev)
        bufs.append(b)
    if in_place == "ys":
        ysv = xv
    elif ys == "f16":
        b, ysv = R.guarded(rows, dim, torch.float16, dev)
        bufs.append(b)
    elif ys == "bf16":
        b, ysv = R.guarded(rows, dim, torch.float32, dev)
        b.view(torch.int32).fill_(0x7FC17FC1)       # a bf16 NaN in both halves of every slot
        bufs.append(b)
    with R.env("MER_LN_VER", form):
        L.layernorm(xv, gamma, beta, yv, eps=eps, y_split=ysv, acc=None if acc is None else acc[2:-2], flags=flags)
        torch.cuda.synchronize()
    bufs.append(xbuf)
    for b in bufs:
        assert R.guards_intact(b, rows), "guard row written"
    if acc is not None:
        assert bool(torch.isnan(torch.cat([acc[:2], acc[-2:]])).all()), "accumulator guard row written"
    out["y"], out["ys"] = yv, ysv
    return out


@pytest.mark.parametrize("form", FORMS, ids=["prefetch", "first"])
@pytest.mark.parametrize("dim", DIMS)
def test_layernorm_vs_float64(cuda, dim, form):
    """fp32 y against float64 at the row counts around a block (8 warps), a full grid and the grid-stride tail, on rows
    of every conditioning, within the bound of a two-pass fp32 evaluation (_kernel_refs.layernorm_bound: on the mean-10
    / std-0.1 rows about 1e-5 of max |y|; a one-pass E[x^2] - E[x]^2 variance is ~1e-3 off there)."""
    R2 = _second_row_count(cuda)
    gamma, beta = (t.to(cuda) for t in _affine(dim))
    host = _ln_rows(dim, 3 * R2 - 5)
    worst = 0.0
    for rows, eps in ((1, 1e-5), (7, 1e-12), (8, 1e-5), (9, 1e-5), (1000, 1e-12), (R2, 1e-5), (3 * R2 - 5, 1e-5)):
        # the last `rows` rows of the tensor, so that small counts see every conditioning as well
        x = host[-rows:].to(cuda) if rows > 9 else host[5:5 + rows].to(cuda)
        y = _ln(x, gamma, beta, eps, form=form)["y"]
        assert bool(torch.isfinite(y).all()), rows
        ref = R.layernorm(x, gamma, beta, eps)
        ratio = float(((y.double() - ref).abs() / R.layernorm_bound(x, gamma, ref, eps)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (rows, ratio)
        del x, y, ref
    print(f"mer_layernorm dim {dim} form {form}: worst |y - float64| = {worst:.3f} of the two-pass fp32 bound")


def _same(a, b):
    return a.dtype == b.dtype and bool((R.bits(a) == R.bits(b)).all())


@pytest.mark.parametrize("dim", DIMS)
def test_layernorm_output_forms_and_both_kernel_forms_agree(cuda, dim):
    """Every output form, alone and combined, derives bit for bit from the plain fp32 result, and the two kernel forms
    write the same bits ("the same arithmetic, row for row") at a row count with a second, ragged round of rows."""
    rows = _second_row_count(cuda)
    x = _ln_rows(dim, 3 * rows - 5)[:rows].to(cuda)
    gamma, beta = (t.to(cuda) for t in _affine(dim))
    big = gamma.clone()
    big[1::5] *= 1e5         # |y| beyond the fp16 range on those columns
    eps = 1e-5
    split_err = 0.0
    per_form = []
    for form in FORMS:
        plain = _ln(x, gamma, beta, eps, form=form)["y"]
        got = {"plain": plain}
        # MER_LN_ROUND_TF32: ties-away tf32 rounding of the un-rounded result
        t = _ln(x, gamma, beta, eps, L.MER_LN_ROUND_TF32, form)["y"]
        assert _same(t, L.round_tf32_(plain.clone())) and _same(t, R.round_tf32_ties_away(plain))
        assert bool((R.bits(t) & 0x1FFF == 0).all())
        got["tf32"] = t
        # MER_LN_OUT_F16: round to nearest even, saturating at +-65504 where .half() would give inf
        wide = _ln(x, big, beta, eps, form=form)["y"]
        assert float(wide.abs().max()) > 2 * F16_MAX
        h = _ln(x, big, beta, eps, L.MER_LN_OUT_F16, form, y="f16")["y"]
        assert _same(h, wide.clamp(-F16_MAX, F16_MAX).half()) and float(h.float().abs().max()) == F16_MAX
        got["f16"] = h
        # y and y_split (bf16 hi | lo) together, with the tf32 flag: y rounded, the split row from the un-rounded value
        both = _ln(x, gamma, beta, eps, L.MER_LN_ROUND_TF32, form, ys="bf16")
        assert _same(both["y"], t)
        hi, lo = R.split_halves(both["ys"])
        assert _same(hi, R.round_bf16_nearest_even(plain))
        assert _same(lo, R.round_bf16_nearest_even(plain - hi))
        # hi + lo: |x - hi| <= 2^-9 |x| and lo is its bf16 rounding, 2^-9 of that: 2^-18 |x| << 2^-16 |x|
        rel = (L.unsplit_bf16(both["ys"]).double() - plain.double()).abs() / plain.double().abs().clamp_min(1e-30)
        split_err = max(split_err, float(rel.max()))
        assert split_err <= 2.0 ** -16
        got["split"] = both["ys"]
        # y = NULL with only y_split
        only = _ln(x, gamma, beta, eps, 0, form, y=None, ys="bf16")
        assert _same(only["ys"], both["ys"])
        # MER_LN_SPLIT_F16: an fp16 row next to the fp32 y
        s16 = _ln(x, big, beta, eps, L.MER_LN_SPLIT_F16, form, ys="f16")
        assert _same(s16["y"], wide) and _same(s16["ys"], h)
        # MER_LN_GELU combined with the tf32 rounding and an fp16 second output
        ge = _ln(x, gamma, beta, eps, L.MER_LN_GELU, form)["y"]
        # gelu_erf_fast: 5e-7 max(1, |x|), see test_layernorm_gelu_against_float64_erf
        assert bool(((ge.double() - R.gelu_erf(plain)).abs() <= 5e-7 * plain.double().abs().clamp_min(1.0)).all())
        gc = _ln(x, gamma, beta, eps, L.MER_LN_GELU | L.MER_LN_ROUND_TF32 | L.MER_LN_SPLIT_F16, form, ys="f16")
        assert _same(gc["y"], R.round_tf32_ties_away(ge)) and _same(gc["ys"], ge.clamp(-F16_MAX, F16_MAX).half())
        got["gelu"] = ge
        per_form.append(got)
    for key in per_form[0]:
        assert _same(per_form[0][key], per_form[1][key]), f"the two kernel forms differ on {key}"
    print(f"mer_layernorm dim {dim}: output forms exact; worst |hi + lo - y| / |y| = {split_err:.2e} (2^-16 = 1.5e-5)")


@pytest.mark.parametrize("form", FORMS, ids=["prefetch", "first"])
def test_layernorm_constant_rows(cuda, form):
    """A constant row of 0 or a power of two has an exact fp32 sum.  At 512 and 1024 columns 1 / dim is exact too: the
    variance is exactly 0 and y exactly beta for either eps.  At 768, 1280 and 1536 columns fl(1 / dim) is 2^-25 or 2^-26
    (relative) above 1 / dim and the compiler fuses x - sum * fl(1 / dim) into one FMA, which sees the unrounded product:
    every centred value is -c 2^-25 instead of 0, and with eps 1e-12 (rsqrt = 1e6) a row of 1024 comes out as
    beta - gamma.  That is inside the conditioning bound (max |x| / sqrt(eps) is enormous), so it is pinned as it is:
    zero rows exact, the others within the bound.  For an arbitrary constant (3.7) the mean's last-bit error is large
    by nature at every width: finiteness and the agreement of the two kernel forms only."""
    for dim in DIMS:
        gamma, beta = (t.to(cuda) for t in _affine(dim))
        vals = torch.tensor([0.0, 1.0, -2.0, 0.5, 1024.0, 2.0 ** -20, 0.0, 4.0, -0.25, 8.0, 16.0])
        x = vals[:, None].expand(-1, dim).contiguous().to(cuda)
        for eps in (1e-12, 1e-5):
            y = _ln(x, gamma, beta, eps, form=form)["y"]
            assert bool((y[vals == 0] == beta[None]).all()), (dim, eps)
            if dim in (512, 1024):
                assert bool((y == beta[None]).all()), (dim, eps)
            else:
                ref = R.layernorm(x, gamma, beta, eps)
                assert bool(((y.double() - ref).abs() <= R.layernorm_bound(x, gamma, ref, eps)).all()), (dim, eps)
            odd = torch.full((9, dim), 3.7, device=cuda)
            a = _ln(odd, gamma, beta, eps, form=form)["y"]
            b = _ln(odd, gamma, beta, eps, form="1" if form is None else None)["y"]
            assert bool(torch.isfinite(a).all()) and _same(a, b)


def test_layernorm_gelu_against_float64_erf(cuda):
    """gelu_erf_fast (Abramowitz-Stegun 7.1.26 with rcp.approx / ex2.approx) over 49152 points of [-8, 8], placed in the
    kernel through gamma = 0, beta = sweep.  The erf polynomial is 1.5e-7 off, the approximate instructions add about as
    much, and gelu = x / 2 * (1 + erf): bound 5e-7 * max(1, |x|).  Measured on an H100 80GB HBM3 (700 W): worst |error|
    3.7e-7, worst |error| / max(1, |x|) 1.4e-7."""
    dim, calls = 1536, 32
    sweep = torch.linspace(-8.0, 8.0, dim * calls, dtype=torch.float64).float().view(dim, calls).T.contiguous().to(cuda)
    x = torch.randn(3, dim, generator=_gen(1)).to(cuda)
    zero = torch.zeros(dim, device=cuda)
    worst, worst_rel = 0.0, 0.0
    for form in FORMS:
        for i in range(calls):
            y = _ln(x, zero, sweep[i], 1e-5, L.MER_LN_GELU, form)["y"]
            err = (y.double() - R.gelu_erf(sweep[i])[None]).abs()
            worst = max(worst, float(err.max()))
            worst_rel = max(worst_rel, float((err / sweep[i].double().abs().clamp_min(1.0)[None]).max()))
    print(f"gelu_erf_fast over [-8, 8]: worst |error| {worst:.2e}, worst |error| / max(1, |x|) {worst_rel:.2e}")
    assert worst_rel <= 5e-7


@pytest.mark.parametrize("form", FORMS, ids=["prefetch", "first"])
def test_layernorm_accumulator(cuda, form):
    """acc = y (MER_LN_ACC_INIT) and acc += y (MER_LN_ACC_ADD) take the value BEFORE the tf32 / fp16 rounding of y; four
    calls give the sum of the last four hidden states; without either flag acc is not touched."""
    dim = 768
    rows = _second_row_count(cuda)
    gamma, beta = (t.to(cuda) for t in _affine(dim))
    host = _ln_rows(dim, 3 * rows - 5)
    xs = [host[i * 7:i * 7 + rows].to(cuda) for i in range(4)]
    eps = 1e-5
    plain = [_ln(x, gamma, beta, eps, form=form)["y"] for x in xs]
    nan_acc = lambda: torch.full((rows + 4, dim), float("nan"), device=cuda)  # noqa: E731
    for extra, kw in ((0, {}), (L.MER_LN_ROUND_TF32, {}), (L.MER_LN_OUT_F16, {"y": "f16"}),
                      (0, {"y": None, "ys": "bf16"})):
        acc = nan_acc()
        _ln(xs[0], gamma, beta, eps, L.MER_LN_ACC_INIT | extra, form, acc=acc, **kw)
        assert _same(acc[2:-2], plain[0]), "ACC_INIT must store the un-rounded y"
        run = plain[0].clone()
        for i in (1, 2, 3):
            _ln(xs[i], gamma, beta, eps, L.MER_LN_ACC_ADD | extra, form, acc=acc, **kw)
            run += plain[i]       # the same fp32 additions in the same order
            assert _same(acc[2:-2], run), "ACC_ADD must add the un-rounded y"
    # against float64: four LayerNorm bounds and three fp32 additions
    ref = sum(R.layernorm(x, gamma, beta, eps) for x in xs)
    bound = sum(R.layernorm_bound(x, gamma, R.layernorm(x, gamma, beta, eps), eps) for x in xs) + 3 * U * sum(
        p.double().abs() for p in plain)
    ratio = float(((acc[2:-2].double() - ref).abs() / bound).max())
    assert ratio <= 1.0
    # INIT wins over ADD when both are set (the kernel tests INIT first): a NaN accumulator is overwritten
    acc = nan_acc()
    _ln(xs[0], gamma, beta, eps, L.MER_LN_ACC_INIT | L.MER_LN_ACC_ADD, form, acc=acc)
    assert _same(acc[2:-2], plain[0])
    # no flag: untouched
    acc = nan_acc()
    y = _ln(xs[0], gamma, beta, eps, 0, form, acc=acc)["y"]
    assert bool(torch.isnan(acc).all()) and _same(y, plain[0])
    print(f"mer_layernorm accumulator ({form}): last-four sum at {ratio:.3f} of its fp32 bound")


@pytest.mark.parametrize("form", FORMS, ids=["prefetch", "first"])
@pytest.mark.parametrize("dim", [512, 768, 1536])
def test_layernorm_in_place(cuda, dim, form):
    """y == x and y_split == x: a warp holds its row in registers before it writes, and the row it requests next is its
    own, so in-place runs give the out-of-place bits; at a row count where that next-row request overlaps the stores."""
    rows = _second_row_count(cuda)
    x = _ln_rows(dim, 3 * rows - 5)[7:7 + rows].to(cuda)
    gamma, beta = (t.to(cuda) for t in _affine(dim))
    out = _ln(x, gamma, beta, 1e-5, L.MER_LN_ROUND_TF32, form, ys="bf16")
    assert _same(_ln(x, gamma, beta, 1e-5, L.MER_LN_ROUND_TF32, form, in_place="y")["y"], out["y"])
    assert _same(_ln(x, gamma, beta, 1e-5, 0, form, y=None, in_place="ys")["ys"], out["ys"])
    two = _ln(x, gamma, beta, 1e-5, L.MER_LN_ROUND_TF32, form, in_place="y", ys="bf16")
    assert _same(two["y"], out["y"]) and _same(two["ys"], out["ys"])


def test_layernorm_refusals(cuda):
    dim = 768
    x = torch.randn(4, dim, generator=_gen(2)).to(cuda)
    gamma, beta = (t.to(cuda) for t in _affine(dim))
    y = torch.full((4, dim), float("nan"), device=cuda)
    before = L.launch_count()
    with pytest.raises(L.MerError, match="mer_layernorm: an fp16 output cannot alias the input"):
        L.layernorm(x, gamma, beta, x, eps=1e-5, flags=L.MER_LN_OUT_F16)
    with pytest.raises(L.MerError, match=r"mer_layernorm: dim 640 not supported \(512, 768, 1024, 1280, 1536\)"):
        L.layernorm(x.view(-1)[:4 * 640].view(4, 640), gamma, beta, y, eps=1e-5)
    with pytest.raises(L.MerError, match="mer_layernorm: null operand"):
        L.layernorm(x, gamma, beta, None, eps=1e-5)
    with pytest.raises(L.MerError, match="mer_layernorm: null operand"):
        L.layernorm(x, None, beta, y, eps=1e-5)
    with pytest.raises(L.MerError, match="mer_layernorm: null operand"):
        L.layernorm(x, gamma, None, y, eps=1e-5)
    for rows in (0, -3):
        rc = L.lib().mer_layernorm(L.ptr(x), L.ptr(gamma), L.ptr(beta), L.ptr(y), None, None, rows, dim, 1e-5, 0,
                                   L.stream_ptr())
        assert rc == 0
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(y).all())


# ----------------------------------------------------------- segment reduce ----
SEG_LENS = [5000, 1, 2, 31, 32, 33, 197]


@pytest.mark.parametrize("mean", [False, True], ids=["sum", "mean"])
@pytest.mark.parametrize("dim", [4, 64, 516, 768, 1024, 1540])
def test_segment_reduce_vs_float64(cuda, dim, mean):
    """Arbitrary begins / ends: every length around the four row groups and the 32-row boundary, empty and reversed
    (clamped to empty: zeros, no 0 / 0 in MEAN), overlapping and out-of-order segments; 516 and 1540 columns leave a
    partial last 512-column block.  Rows no segment owns are NaN.  Bound: each of the four row groups adds n / 4 terms
    one after another and three more additions combine them: (n / 4 + 3) u sum |x|, over n for MEAN plus one rounding."""
    begins, ends, at = [], [], 0
    for n in SEG_LENS:
        begins.append(at)
        ends.append(at + n)
        at += n + 1                      # one NaN row between neighbours
    total = at + 3
    x = torch.randn(total, dim, generator=_gen(dim)) + 1.0
    owned = torch.zeros(total, dtype=torch.bool)
    for a, b in zip(begins, ends):
        owned[a:b] = True
    x[~owned] = float("nan")
    begins += [at, 120, 10, 200, 5001]   # empty at a NaN row; reversed; two segments inside the first; a repeat
    ends += [at, 50, 300, 250, 5002]
    order = torch.randperm(len(begins), generator=_gen(3)).tolist()
    begins, ends = [begins[i] for i in order], [ends[i] for i in order]
    xd = x.to(cuda)
    bd, ed = (torch.tensor(t, dtype=torch.int32, device=cuda) for t in (begins, ends))
    buf, out = R.guarded(len(begins), dim, torch.float32, cuda)
    L.segment_reduce(xd, bd, ed, out, dim=dim, mean=mean)
    torch.cuda.synchronize()
    assert R.guards_intact(buf, len(begins)) and bool(torch.isfinite(out).all())
    ref = R.segment_reduce(xd, begins, ends, mean)
    worst = 0.0
    for s, (a, b) in enumerate(zip(begins, ends)):
        n = max(b - a, 0)
        if n == 0:
            assert bool((out[s] == 0).all()), "an empty segment gives zeros"
            continue
        mass = xd[a:b].double().abs().sum(0)
        bound = (n / 4 + 3) * U * mass / (n if mean else 1) + 3 * U * ref[s].abs()   # 1 / n, the product, the store
        ratio = float(((out[s].double() - ref[s]).abs() / bound).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (a, b, ratio)
    if not mean:                          # a single row is copied exactly
        s = begins.index(5001)
        assert bool((out[s] == xd[5001]).all())
    print(f"mer_segment_reduce dim {dim} {'mean' if mean else 'sum'}: worst error {worst:.3f} of the fp32 sum bound")


def test_segment_reduce_offsets_form_and_refusals(cuda):
    """Back-to-back segments passed as (offsets, offsets + 1), n_seg = 0, and the refusals."""
    dim = 768
    x = (torch.randn(300, dim, generator=_gen(4)) + 1.0).to(cuda)
    offs = [0, 7, 7, 40, 41, 300]
    od = torch.tensor(offs, dtype=torch.int32, device=cuda)
    buf, out = R.guarded(5, dim, torch.float32, cuda)
    L.segment_reduce(x, od, od[1:], out, dim=dim, mean=True, n_seg=5)
    torch.cuda.synchronize()
    ref = R.segment_reduce(x, offs[:-1], offs[1:], True)
    assert R.guards_intact(buf, 5) and bool((out[1] == 0).all()) and bool((out[3] == x[40]).all())
    assert float((out.double() - ref).abs().max()) <= (259 / 4 + 6) * U * float(x.abs().max())   # the longest: 259 rows
    before = L.launch_count()
    out.fill_(float("nan"))
    L.segment_reduce(x, od, od[1:], out, dim=dim, n_seg=0)
    with pytest.raises(L.MerError, match="mer_segment_reduce: dim 6 must be a multiple of 4"):
        L.segment_reduce(x, od, od[1:], out, dim=6, n_seg=5)
    with pytest.raises(L.MerError, match="mer_segment_reduce: dim 0 must be a multiple of 4"):
        L.segment_reduce(x, od, od[1:], out, dim=0, n_seg=5)
    with pytest.raises(L.MerError, match="mer_segment_reduce: null operand"):
        L.segment_reduce(x, od, None, out, dim=dim, n_seg=5)
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(out).all())


# ----------------------------------------------------------- wave normalise ----
def _waves(n, seed):
    g = _gen(seed)
    t = torch.arange(n, dtype=torch.float64)
    return {
        "dc": (0.5 + 1e-3 * torch.sin(2 * np.pi * 220.0 / 16000.0 * t) + 1e-4 * torch.randn(n, generator=g).double()).float(),
        "speech": (torch.randn(n, generator=g) * 3000.0 * (1.0 + torch.sin(t / 400.0)).float()).round().clamp(
            -32768, 32767) / 32768.0,
        "zeros": torch.zeros(n),
        "const": torch.full((n,), 0.3),
    }


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("n", [1, 2, 399, 1024, 1025, 16000, 160001])
def test_wave_normalize_vs_float64(cuda, n, batch):
    """(x - mean) / sqrt(var + 1e-7) of HF Wav2Vec2FeatureExtractor with distinct row pitches, NaN in the input padding
    and a sentinel in the output padding.  The kernel takes mean and variance in double and evaluates in fp32: the mean's
    cast (u |mean|) and the subtraction (u |x - mean|) over sigma, plus the cast of the variance, the addition of the fp32
    1e-7, the square root and the division: 6 u (|mean| / sigma + |y|).  A constant row (variance 0) gives exactly
    0 = (x - mean) / sqrt(1e-7), and so does n_samples = 1."""
    ld_in, ld_out = n + 5, n + 9
    w = _waves(n, 10 + n % 97)
    groups = [[k] for k in w] if batch == 1 else [["dc", "speech", "const"], ["zeros", "dc", "speech"]]
    worst = 0.0
    for kinds in groups:
        xin = torch.full((batch, ld_in), float("nan"))
        for r, k in enumerate(kinds):
            xin[r, :n] = w[k]
        xin = xin.to(cuda)
        out = torch.full((batch + 1, ld_out), 12345.0, device=cuda)
        L.wave_normalize(xin, out, batch=batch, n_samples=n, ld_in=ld_in, ld_out=ld_out)
        torch.cuda.synchronize()
        assert bool((out[:batch, n:] == 12345.0).all()) and bool((out[batch] == 12345.0).all()), "padding written"
        y = out[:batch, :n]
        assert bool(torch.isfinite(y).all())
        x = xin[:, :n].double()
        ref = R.wave_normalize(x)
        mu = x.mean(1, keepdim=True)
        sig = torch.sqrt(((x - mu) ** 2).mean(1, keepdim=True) + 1e-7)
        ratio = ((y.double() - ref).abs() / (6 * U * (mu.abs() / sig + ref.abs()) + 1e-30)).amax(1)
        for r, k in enumerate(kinds):
            if k in ("zeros", "const") or n == 1:
                assert bool((y[r] == 0).all()), (k, n)
            else:
                worst = max(worst, float(ratio[r]))
                assert float(ratio[r]) <= 1.0, (k, n, float(ratio[r]))
    print(f"mer_wave_normalize n {n} batch {batch}: worst error {worst:.3f} of 6 u (|mean| / sigma + |y|)")


def test_wave_normalize_refusals(cuda):
    x = torch.zeros(2, 64, device=cuda)
    y = torch.full((2, 64), float("nan"), device=cuda)
    before = L.launch_count()
    for kw in (dict(batch=0, n_samples=64), dict(batch=2, n_samples=0)):
        with pytest.raises(L.MerError, match="mer_wave_normalize: bad arguments"):
            L.wave_normalize(x, y, ld_in=64, ld_out=64, **kw)
    with pytest.raises(L.MerError, match="mer_wave_normalize: bad arguments"):
        L.wave_normalize(None, y, batch=2, n_samples=64, ld_in=64, ld_out=64)
    # a row pitch shorter than the row would make neighbouring rows overlap
    with pytest.raises(L.MerError, match="mer_wave_normalize: row pitches"):
        L.wave_normalize(x, y, batch=2, n_samples=64, ld_in=63, ld_out=64)
    with pytest.raises(L.MerError, match="mer_wave_normalize: row pitches"):
        L.wave_normalize(x, y, batch=2, n_samples=64, ld_in=64, ld_out=32)
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(y).all())


# ------------------------------------------------------------------ SwiGLU ----
@pytest.mark.parametrize("hidden", [4, 1536, 4096])
@pytest.mark.parametrize("rows", [1, 3, 1000])
def test_swiglu_vs_float64(cuda, rows, hidden):
    """silu(gate) * up in fp32: expf, one addition, a division and a product, 6 u relative.  Gates of +-100 overflow or
    flush the exponential: the result must be the finite limit, x * up or 0."""
    g = _gen(rows * 10000 + hidden)
    worst = 0.0
    for scale in (1.0, 100.0):
        x = torch.randn(rows, 2 * hidden, generator=g) * scale
        if scale == 100.0:
            x[:, 0:hidden:2] = 100.0
            x[:, 1:hidden:2] = -100.0
            x[:, 1] = -88.0                                  # exp(88) is still finite in fp32
        xd = x.to(cuda)
        buf, out = R.guarded(rows, hidden, torch.float32, cuda)
        L.swiglu(xd, out, rows=rows, hidden=hidden)
        torch.cuda.synchronize()
        assert R.guards_intact(buf, rows) and bool(torch.isfinite(out).all())
        ref = R.swiglu(xd, hidden)
        ratio = float(((out.double() - ref).abs() / (6 * U * ref.abs() + 1e-36)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0
        if scale == 100.0:
            assert bool((out[:, 0:hidden:2] == 100.0 * xd[:, hidden::2]).all())
            assert bool((out[:, 3:hidden:2] == 0).all())
        buf2, rounded = R.guarded(rows, hidden, torch.float32, cuda)
        L.swiglu(xd, rounded, rows=rows, hidden=hidden, round_out=True)
        torch.cuda.synchronize()
        assert R.guards_intact(buf2, rows) and bool((R.bits(rounded) & 0x1FFF == 0).all())
        assert bool((R.bits(rounded) == R.bits(R.round_tf32_ties_away(out))).all())
    print(f"mer_swiglu rows {rows} hidden {hidden}: worst error {worst:.3f} of 6 u |silu(gate) up|")


def test_swiglu_refusals(cuda):
    x = torch.zeros(2, 16, device=cuda)
    y = torch.full((2, 8), float("nan"), device=cuda)
    before = L.launch_count()
    for kw, a, b in ((dict(rows=2, hidden=8), x, x), (dict(rows=2, hidden=6), x, y), (dict(rows=0, hidden=8), x, y),
                     (dict(rows=2, hidden=0), x, y), (dict(rows=2, hidden=8), None, y)):
        with pytest.raises(L.MerError, match="mer_swiglu: bad arguments"):
            L.swiglu(a, b, **kw)
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(y).all())


# --------------------------------------------------------- VideoMAE patches ----
@pytest.mark.parametrize("n_clips", [1, 2])
def test_videomae_patchify_vs_float64(cuda, n_clips):
    """tf32 rounding of (pix / 255 - mean) / std in the [n_clips * 1568, 1536] layout of _kernel_refs.videomae_patches
    (the definition the CPU stand-in of the VideoMAE backend uses).  fp32 evaluation: pix * fl(1 / 255) and the
    subtraction leave 2 u absolute, divided by std, then half a tf32 ulp (2^-11 relative) of rounding."""
    frames = torch.from_numpy(np.random.default_rng(40 + n_clips).integers(0, 256, (n_clips * 16, 224, 224, 3),
                                                                          dtype=np.uint8)).to(cuda)
    # the fp32 values the kernel receives, so that the reference starts from the same operands
    mean, std = ([float(np.float32(v)) for v in t] for t in ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)))
    buf, out = R.guarded(n_clips * 1568, 1536, torch.float32, cuda)
    L.videomae_patchify(frames, mean, std, out, n_clips=n_clips)
    torch.cuda.synchronize()
    assert R.guards_intact(buf, n_clips * 1568) and bool(torch.isfinite(out).all())
    assert bool((R.bits(out) & 0x1FFF == 0).all())
    ref = R.videomae_patches(frames, mean, std)
    err = (out.double() - ref).abs()
    bound = 2.0 ** -11 * (1 + 2.0 ** -10) * ref.abs() + 3 * U / min(std)
    ratio = float((err / bound).max())
    assert ratio <= 1.0
    # the bound is below the spacing of neighbouring grey levels (1 / 255 / std), so a permuted column cannot pass
    assert float(bound.max()) < 0.25 / 255.0 / max(std)
    with pytest.raises(L.MerError, match="mer_videomae_patchify: bad arguments"):
        L.videomae_patchify(frames, mean, std, out, n_clips=0)
    print(f"mer_videomae_patchify {n_clips} clips: worst error {ratio:.3f} of half a tf32 ulp + 3 u / std")
