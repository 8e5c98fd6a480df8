"""GPU parity of the tensor-core attention kernels -- attention_short.cu, attention_f16.cu (fp16 and tf32) and
attention_causal.cu (plain, ALiBi, multi-query) -- against the float64 attention_packed of the same operand values,
element by element under attention_tc_bound (tests/_kernel_refs.py, where the bound is derived from the kernels'
arithmetic).  One table of routes (ATT_TC_CASES): each entry point, with the kernel that must run it asserted by name
under torch.profiler, so that a routing change cannot turn a short-kernel case into a tile-kernel one unnoticed.

Every case runs at operand scale 1.5 and at 4 (peaked rows), on lengths at every kernel boundary with an empty
sequence inside cu_seqlens, NaN in every column the kernel must not read (the V block of qkv, V^T past `tokens`, the
unread columns of a multi-query row) and NaN guard rows around ctx.  The non-causal routes write ctx in all four
formats: fp32 is checked against the bound, and fp16 / tf32 / split rows must be exactly the fp32 values stored in that
format.  Each case prints its worst |ctx - ref| / bound per length class."""
import time

import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
vp, i32, i64, f32 = L.C.c_void_p, L.C.c_int, L.C.c_longlong, L.C.c_float
CLASSES = ((1, 16), (17, 128), (129, 249), (250, 505), (506, 4096))
OUT_FLAGS = {"fp32": 0, "tf32": L.MER_EPI_ROUND_TF32, "split": L.MER_EPI_SPLIT_BF16, "f16": L.MER_EPI_OUT_F16}


def _device_operands(c, ops, cuda):
    """(qkv, vt, cu) on the device: qkv in the case's operand type with NaN in the columns no kernel reads, V^T
    [heads * hd (hd for multi-query), pad8(tokens) + 64] with NaN past `tokens`."""
    dt = torch.float16 if c["fmt"] == "f16" else torch.float32
    H, hd = c["heads"], c["hd"]
    qkv = ops["qkv"].to(cuda, dt)
    if c["mqa"]:
        qkv[:, (H + 1) * hd:] = float("nan")
    else:
        qkv[:, 2 * H * hd:] = float("nan")
    T = qkv.shape[0]
    v = ops["v"].to(cuda, dt)
    vt = torch.full((v.shape[1], (T + 7) // 8 * 8 + 64), float("nan"), dtype=dt, device=cuda)
    vt[:, :T] = v.T
    return qkv, vt, torch.tensor(ops["cu"], dtype=torch.int32, device=cuda)


def _launch(c, qkv, vt, cu, ctx, fmt, slopes=None):
    H, hd = c["heads"], c["hd"]
    n_seq, T = cu.numel() - 1, qkv.shape[0]
    max_len = int((cu[1:] - cu[:-1]).max())
    e = c["entry"]
    if e == "attention":
        with R.env("MER_ATT_SHORT", c["env"]):
            if c["fmt"] == "f16":
                L.attention(qkv, ctx, cu, max_len, H, vt=vt, round_out=fmt == "tf32", split_out=fmt == "split")
            else:
                L.attention(qkv, ctx, cu, max_len, H, vt=vt, round_out=fmt == "tf32", split_out=fmt == "split",
                            f16_out=fmt == "f16")
        return
    flags = OUT_FLAGS[fmt]
    if e == "hd":
        f = L.declare("mer_attention_hd", [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, f32, i32, vp])
        rc = f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), n_seq, T, max_len, H, hd, c["scale"],
               flags | (L.MER_ATT_QKV_F16 if c["fmt"] == "f16" else 0), L.stream_ptr())
    elif e == "long":
        f = L.declare("mer_attention_long", [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, vp])
        rc = f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), n_seq, T, max_len, H, flags, L.stream_ptr())
    elif e == "causal":
        f = L.declare("mer_causal_attention_hd_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, i32, vp])
        rc = f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), n_seq, T, max_len, H, hd, L.stream_ptr())
    elif e == "causal128":
        f = L.declare("mer_causal_attention_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, vp])
        rc = f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), n_seq, T, max_len, H, L.stream_ptr())
    elif e == "alibi":
        f = L.declare("mer_causal_alibi_attention_f16", [vp, vp, i64, vp, vp, i32, i64, i32, i32, vp, vp])
        rc = f(L.ptr(qkv), L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), n_seq, T, max_len, H, L.ptr(slopes),
               L.stream_ptr())
    else:
        f = L.declare("mer_causal_mqa_attention_f16", [vp, i64, vp, i64, vp, vp, i32, i64, i32, i32, vp])
        rc = f(L.ptr(qkv), qkv.shape[1], L.ptr(vt), vt.shape[1], L.ptr(ctx), L.ptr(cu), n_seq, T, max_len, H,
               L.stream_ptr())
    L.check(rc)


def _run(c, qkv, vt, cu, fmt, slopes=None):
    """ctx in `fmt` between NaN guard rows, which must stay NaN."""
    T, D = qkv.shape[0], c["heads"] * c["hd"]
    buf, ctx = R.guarded(T, D, torch.float16 if fmt == "f16" else torch.float32, qkv.device)
    _launch(c, qkv, vt, cu, ctx, fmt, slopes)
    torch.cuda.synchronize()
    assert R.guards_intact(buf, T), (c["entry"], fmt)
    return ctx


def _value(ctx, fmt):
    if fmt == "split":
        hi, lo = R.split_halves(ctx)
        return hi.double() + lo.double()
    return ctx.double()


def _worst_by_class(ratio, cu):
    """Worst ratio per length class, over the rows of the sequences in that class."""
    out = {}
    for a, b in zip(cu, cu[1:]):
        if b > a:
            cls = next(f"{lo}..{hi}" for lo, hi in CLASSES if lo <= b - a <= hi)
            out[cls] = max(out.get(cls, 0.0), float(ratio[a:b].max()))
    return out


@pytest.mark.parametrize("amp", [1.5, 4.0])
@pytest.mark.parametrize("name", list(R.ATT_TC_CASES))
def test_tc_attention_vs_float64(cuda, name, amp):
    t0 = time.perf_counter()
    c = R.att_tc_case(name)
    ops = R.att_tc_operands(c, amp)
    ref, mag, A, st = R.att_tc_reference(c, ops, cuda)
    qkv, vt, cu = _device_operands(c, ops, cuda)
    slopes = None if ops["slopes"] is None else ops["slopes"].to(cuda)
    first = "f16" if c["causal"] else "fp32"
    base, kernels = R.attention_kernels(lambda: _run(c, qkv, vt, cu, first, slopes))
    assert any(c["kernel"] in k for k in kernels), (name, kernels)
    assert len(kernels) == 1, (name, kernels)     # one attention launch, of that kernel only
    outs = {first: base}
    if not c["causal"]:
        for fmt in ("f16", "tf32", "split"):
            outs[fmt] = _run(c, qkv, vt, cu, fmt)
        x = base
        assert torch.equal(R.bits(outs["f16"]), R.bits(R.f16_satfinite(x).half())), name
        assert torch.equal(R.bits(outs["tf32"]), R.bits(R.round_tf32_ties_away(x))), name
        hi, lo = R.split_halves(outs["split"])
        want_hi, want_lo = R.split_bf16(x)
        assert torch.equal(R.bits(hi), R.bits(want_hi)) and torch.equal(R.bits(lo), R.bits(want_lo)), name
    msg = []
    for fmt, ctx in outs.items():
        got = _value(ctx, fmt)
        assert torch.isfinite(got).all(), (name, fmt)
        ratio = R.bound_ratio(got, ref, R.attention_tc_bound(mag, A, st, ref, fmt)).amax(-1).cpu()
        worst = _worst_by_class(ratio, ops["cu"])
        msg.append(f"{fmt}: " + " ".join(f"{k} {v:.2f}" for k, v in worst.items()))
        assert float(ratio.max()) <= 1.0, (name, fmt, worst)
    if c["valid"] < c["hd"]:                     # ALBERT's zero-padded head columns come out exactly 0
        pad = base.view(base.shape[0], c["heads"], c["hd"])[:, :, c["valid"]:]
        assert int(R.bits(pad).abs().max()) == 0, name
    print(f"\n{name} x{amp} [{c['kernel']}] " + "; ".join(msg) + f" ({time.perf_counter() - t0:.1f} s)")


@pytest.mark.parametrize("name", list(R.ATT_TC_CASES))
def test_tc_attention_neighbours_do_not_leak(cuda, name):
    """A sequence's ctx rows stay bit for bit when every other sequence's (finite) q, k and v change: the leading
    foreign keys of its 8-token aligned key axis and the keys after it are masked, whatever they hold."""
    c = R.att_tc_case(name)
    ops = R.att_tc_operands(c, 1.5)
    other = R.att_tc_operands(c, 1.5, seed=1)
    cu = ops["cu"]
    s = max(range(len(cu) - 1), key=lambda i: (cu[i + 1] - cu[i], cu[i] % 8))   # the longest row
    a, b = cu[s], cu[s + 1]
    for key in ("qkv", "v"):
        other[key][a:b] = ops[key][a:b]
    fmt = "f16" if c["causal"] else "fp32"
    slopes = None if ops["slopes"] is None else ops["slopes"].to(cuda)
    x = _run(c, *_device_operands(c, ops, cuda), fmt, slopes)
    y = _run(c, *_device_operands(c, other, cuda), fmt, slopes)
    assert torch.equal(R.bits(x[a:b]), R.bits(y[a:b])), name
    assert not torch.equal(R.bits(x[:a]), R.bits(y[:a])) or a == 0
