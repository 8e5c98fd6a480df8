"""GPU parity of the relative-position tensor-core attention kernels -- attention_rel.cu (DeBERTa's disentangled
attention, mer_disentangled_attention) and attention_xl.cu (XLNet's relative attention, mer_xlnet_attention) -- against
the float64 attention_packed of the same operand values with the kernel's score term (deberta_rel / xlnet_rel), element
by element under attention_tc_bound with the score coefficient derived for each kernel (tests/_kernel_refs.py).  One
table of cases (ATT_REL_CASES): entry point, operand format, heads, row map and lengths, with the kernel that must run
asserted by name under torch.profiler and by the launch counter.

Every case runs at operand scale 1.5 and at 4 (peaked rows), on lengths at every 64-token tile edge with an empty
sequence inside cu_seqlens and most starts off a multiple of 8, with NaN in everything the kernel must not read (the V
block of qkv, V^T past `tokens`, the pitch tail of the tables, every table row rel_row does not name) and NaN guard rows
around ctx; some pass max_seqlen beyond the longest sentence.  ctx is written in all four formats: fp32 is checked
against the bound, fp16 / tf32 / split rows must be exactly the fp32 values stored in that format.  Each case prints its
worst |ctx - ref| / bound per length class and format."""
import time

import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
vp, i32, i64, f32 = L.C.c_void_p, L.C.c_int, L.C.c_longlong, L.C.c_float
CLASSES = ((1, 16), (17, 128), (129, 257), (258, 1100))
OUT_FLAGS = {"fp32": 0, "tf32": L.MER_EPI_ROUND_TF32, "split": L.MER_EPI_SPLIT_BF16, "f16": L.MER_EPI_OUT_F16}
NAN = float("nan")


def _table(t, n_rows, rows, D, dt, cuda):
    """A [n_rows, D + 64] table on the device: NaN in the pitch tail and in every row `rows` does not name."""
    buf = torch.full((n_rows, D + 64), NAN, dtype=dt, device=cuda)
    named = torch.unique(torch.as_tensor(rows).long().clamp(0, n_rows - 1))
    buf[named.to(cuda), :D] = t[named].to(cuda, dt)
    return buf


def _device(c, ops, cuda):
    """The case's operands on the device in its operand type, NaN wherever the kernel must not read."""
    dt = torch.float16 if c["fmt"] == "f16" else torch.float32
    D = c["heads"] * 64
    qkv = ops["qkv"].to(cuda, dt)
    qkv[:, 2 * D:] = NAN
    T = qkv.shape[0]
    vt = torch.full((D, (T + 7) // 8 * 8 + 64), NAN, dtype=dt, device=cuda)
    vt[:, :T] = ops["v"].T.to(cuda, dt)
    d = dict(qkv=qkv, vt=vt, cu=torch.tensor(ops["cu"], dtype=torch.int32, device=cuda),
             rows=torch.as_tensor(ops["rows"]).to(cuda, torch.int32), T=T, ms=ops["max_seqlen"])
    if c["entry"] == "deberta":
        d.update(span=ops["span"], **{k: _table(ops[k], 2 * ops["span"], ops["rows"], D, dt, cuda) for k in ("pk", "pq")})
    else:
        d["r"] = _table(ops["r"], ops["r"].shape[0] + 3, ops["rows"], D, dt, cuda)
        d.update({k: ops[k].to(cuda).contiguous() for k in ("r_w", "r_r", "r_s", "seg")})
        d["types"] = None if ops["types"] is None else ops["types"].to(cuda, torch.int32)
    return d


def _launch(c, d, ctx, fmt):
    flags = OUT_FLAGS[fmt] | (L.MER_ATT_QKV_F16 if c["fmt"] == "f16" else 0)
    n_seq = d["cu"].numel() - 1
    if c["entry"] == "deberta":
        f = L.declare("mer_disentangled_attention", [vp, vp, i64, vp, vp, i64, i32, vp, f32, vp, vp, i32, i64, i32, i32,
                                                     i32, vp])
        rc = f(L.ptr(d["qkv"]), L.ptr(d["vt"]), d["vt"].shape[1], L.ptr(d["pk"]), L.ptr(d["pq"]), d["pk"].shape[1],
               d["span"], L.ptr(d["rows"]), c["scale"], L.ptr(ctx), L.ptr(d["cu"]), n_seq, d["T"], d["ms"], c["heads"],
               flags, L.stream_ptr())
    else:
        rc = L.lib().mer_xlnet_attention(
            L.ptr(d["qkv"]), L.ptr(d["vt"]), d["vt"].shape[1], L.ptr(d["r"]), d["r"].shape[1], L.ptr(d["rows"]),
            L.ptr(d["r_w"]), L.ptr(d["r_r"]), L.ptr(d["r_s"]), L.ptr(d["seg"]), L.ptr(d["types"]), c["scale"],
            L.ptr(ctx), L.ptr(d["cu"]), n_seq, d["T"], d["ms"], c["heads"], flags, L.stream_ptr())
    L.check(rc)


def _run(c, d, fmt):
    """ctx in `fmt` between NaN guard rows, which must stay NaN."""
    T, D = d["T"], c["heads"] * 64
    buf, ctx = R.guarded(T, D, torch.float16 if fmt == "f16" else torch.float32, d["qkv"].device)
    _launch(c, d, ctx, fmt)
    torch.cuda.synchronize()
    assert R.guards_intact(buf, T), (c["kernel"], fmt)
    return ctx


def _value(ctx, fmt):
    if fmt == "split":
        hi, lo = R.split_halves(ctx)
        return hi.double() + lo.double()
    return ctx.double()


def _worst_by_class(ratio, cu):
    out = {}
    for a, b in zip(cu, cu[1:]):
        if b > a:
            cls = next(f"{lo}..{hi}" for lo, hi in CLASSES if lo <= b - a <= hi)
            out[cls] = max(out.get(cls, 0.0), float(ratio[a:b].max()))
    return out


@pytest.mark.parametrize("amp", [1.5, 4.0])
@pytest.mark.parametrize("name", list(R.ATT_REL_CASES))
def test_rel_attention_vs_float64(cuda, name, amp):
    t0 = time.perf_counter()
    c = R.att_rel_case(name)
    ops = R.att_rel_operands(c, amp)
    ref, mag, A, st = R.att_rel_reference(c, ops, cuda)
    d = _device(c, ops, cuda)
    base, kernels = R.attention_kernels(lambda: _run(c, d, "fp32"))
    assert any(c["kernel"] in k for k in kernels), (name, kernels)
    assert len(kernels) == 1, (name, kernels)      # one attention launch, of that kernel only
    outs = {"fp32": base}
    for fmt in ("f16", "tf32", "split"):
        n0 = L.launch_count()
        outs[fmt] = _run(c, d, fmt)
        assert L.launch_count() - n0 == 1, (name, fmt)
    assert torch.equal(R.bits(outs["f16"]), R.bits(R.f16_satfinite(base).half())), name
    assert torch.equal(R.bits(outs["tf32"]), R.bits(R.round_tf32_ties_away(base))), name
    hi, lo = R.split_halves(outs["split"])
    want_hi, want_lo = R.split_bf16(base)
    assert torch.equal(R.bits(hi), R.bits(want_hi)) and torch.equal(R.bits(lo), R.bits(want_lo)), name
    msg = []
    for fmt, ctx in outs.items():
        got = _value(ctx, fmt)
        assert torch.isfinite(got).all(), (name, fmt)
        bound = R.attention_tc_bound(mag, A, st, ref, fmt, c["score"])
        ratio = R.bound_ratio(got, ref, bound).amax(-1).cpu()
        worst = _worst_by_class(ratio, ops["cu"])
        msg.append(f"{fmt}: " + " ".join(f"{k} {v:.2f}" for k, v in worst.items()))
        assert float(ratio.max()) <= 1.0, (name, fmt, worst)
    print(f"\n{name} x{amp} max_seqlen {ops['max_seqlen']} [{c['kernel']}] " + "; ".join(msg) +
          f" ({time.perf_counter() - t0:.1f} s)")


def _swap_every_other(c, ops, other):
    """ops with the q | k | v rows (and token types) of every odd-numbered sentence taken from `other`."""
    out = dict(ops, qkv=ops["qkv"].clone(), v=ops["v"].clone())
    if ops.get("types") is not None:
        out["types"] = ops["types"].clone()
    cu = ops["cu"]
    for s in range(1, len(cu) - 1, 2):
        a, b = cu[s], cu[s + 1]
        out["qkv"][a:b], out["v"][a:b] = other["qkv"][a:b], other["v"][a:b]
        if ops.get("types") is not None:
            out["types"][a:b] = (ops["types"][a:b] + 1) % 3
    return out


@pytest.mark.parametrize("name", ["deb_v1_h16_f16", "deb_v2_tf32", "xl_clamp20_h12_f16", "xl_tf32"])
def test_rel_attention_neighbours_do_not_leak(cuda, name):
    """New q, k, v (and token types) in every other sentence leave the remaining sentences' ctx bit for bit: the leading
    foreign keys of a sentence's 8-token aligned key axis and the keys after it are masked, whatever they hold, and the
    table rows a sentence reads depend on its own distances only."""
    c = R.att_rel_case(name)
    ops = R.att_rel_operands(c, 1.5)
    mixed = _swap_every_other(c, ops, R.att_rel_operands(c, 1.5, seed=1))
    x = _run(c, _device(c, ops, cuda), "fp32")
    y = _run(c, _device(c, mixed, cuda), "fp32")
    cu = ops["cu"]
    for s in range(len(cu) - 1):
        a, b = cu[s], cu[s + 1]
        if b > a:
            assert torch.equal(R.bits(x[a:b]), R.bits(y[a:b])) == (s % 2 == 0), (name, s)


@pytest.mark.parametrize("fmt", ["f16", "tf32"])
def test_disentangled_attention_clamps_the_row_map(cuda, fmt):
    """mer_disentangled_attention clamps rel_row's entries to [0, 2 span): a map whose entries run below 0 and past
    2 span - 1 (here d + span over distances up to +-299, span 40) gives, bit for bit, the ctx of the map clamped on
    the host, and that ctx is the float64 reference of the clamped rows under the bound."""
    span = 40
    c = dict(R.att_rel_case(f"deb_v1_{fmt}"), lens=[3, 129, 0, 300, 17], heads=2)
    ops = R.att_rel_operands(c, 1.5)
    ms = ops["max_seqlen"]
    raw = (np.arange(-(ms - 1), ms) + span).astype(np.int32)
    assert raw.min() < 0 and raw.max() >= 2 * span
    ops.update(span=span, pk=ops["pk"][:2 * span], pq=ops["pq"][:2 * span])
    got = {}
    for key, rows in (("raw", raw), ("clamped", np.clip(raw, 0, 2 * span - 1))):
        d = _device(c, dict(ops, rows=rows), cuda)
        got[key] = _run(c, d, "fp32")
    assert torch.equal(R.bits(got["raw"]), R.bits(got["clamped"])), fmt
    ref, mag, A, st = R.attention_packed(ops["qkv"].to(cuda), ops["cu"], 2, 64, c["scale"], v=ops["v"].to(cuda),
                                         stats=True, rel=R.deberta_rel(ops["pk"], ops["pq"], raw, ms, span))
    ratio = R.bound_ratio(got["raw"].double(), ref, R.attention_tc_bound(mag, A, st, ref, "fp32", c["score"]))
    print(f"\nclamped row map {fmt}: worst ratio {float(ratio.max()):.2f}")
    assert float(ratio.max()) <= 1.0, fmt
