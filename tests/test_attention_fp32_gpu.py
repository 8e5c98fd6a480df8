"""Kernel-level parity of the fp32 attention entry points that the model tests only reach through a whole encoder:
mer_attention on fp32 operands through the kernel that reads V from qkv (attention.cu: rows over 253 tokens, or no V^T),
mer_biased_attention / mer_wavlm_gate (wavlm.cu) and mer_small_attention (whisper.cu), each against the float64
formula of include/mer_b200.h (tests/_kernel_refs.py) on the same operand values.

Outputs are pre-filled with NaN between NaN guard rows; columns and rows a kernel must not read hold NaN.  Each test
prints its worst observed error as a fraction of the bound derived next to the assert."""
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
U = R.U32
HD = 64
# attention_kernel works on 64-query blocks (BQ) and 64-key tiles (BKV): each boundary -1 / 0 / +1, then the lengths of
# the models that take this route (254 .. 505: fp32 stacks without fp16 rows; 1500: Whisper; 1568: VideoMAE; 2049: past
# the 2048 of a 32-tile row), between short rows so that most sequence starts are not multiples of 8
LENS_3 = [1, 63, 17, 64, 65, 197, 127, 128, 129, 254, 1, 499, 505, 17, 506, 1500, 197, 1568, 2049]
LENS_16 = [17, 254, 1, 506, 197, 1500]


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _cu(lens):
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    return cu


def _qkv(lens, heads, scale, cuda, seed):
    x = (torch.randn(sum(lens), 3 * heads * HD, generator=_gen(seed)) * scale).to(cuda)
    return L.round_tf32_(x)          # the tf32 operands the QKV GEMM writes


def _attend(qkv, lens, heads, *, vt=None, max_seqlen=None, round_out=False, split_out=False):
    cu = torch.tensor(_cu(lens), dtype=torch.int32, device=qkv.device)
    buf, ctx = R.guarded(qkv.shape[0], heads * HD, torch.float32, qkv.device)
    L.attention(qkv, ctx, cu, max_seqlen or max(lens), heads, vt=vt, round_out=round_out, split_out=split_out)
    torch.cuda.synchronize()
    assert R.guards_intact(buf, qkv.shape[0]), "guard row written"
    return ctx


def _bound(mag, amp):
    """P is rounded to tf32 for the P V product (2^-11 relative per probability).  A score is 8 chained tensor-core
    steps with fp32 accumulation, 8 u A, and moves a probability and the normaliser by that much each; the online
    rescaling, the fp32 P V accumulation and the final division add a few u.  So (2^-11 + 16 u A + 8 u) P |V|."""
    return (2.0 ** -11 + 16 * U * amp + 8 * U) * mag + 1e-30


@pytest.mark.parametrize("heads,lens,scale", [(3, LENS_3, 1.5), (3, LENS_3, 4.0), (16, LENS_16, 1.5)],
                         ids=["3heads", "3heads-peaked", "16heads"])
def test_attention_fp32_qkv_kernel_vs_float64(cuda, heads, lens, scale):
    """vt = NULL sends every length, the short ones included, through attention_kernel: one launch."""
    qkv = _qkv(lens, heads, scale, cuda, 11)
    before = L.launch_count()
    ctx = _attend(qkv, lens, heads)
    assert L.launch_count() == before + 1
    assert bool(torch.isfinite(ctx).all()), "a row was not written"
    ref, mag, amp = R.attention_packed(qkv, _cu(lens), heads)
    ratio = (ctx.double() - ref).abs() / _bound(mag, amp)
    worst = float(ratio.max())
    cu = _cu(lens)
    per_len = {n: round(float(ratio[cu[i]:cu[i + 1]].max()), 3) for i, n in enumerate(lens)}
    print(f"mer_attention fp32 (V from qkv) {heads} heads, scale {scale}: worst {worst:.3f} of the bound; by length {per_len}")
    assert worst <= 1.0

    # MER_EPI_ROUND_TF32 / MER_EPI_SPLIT_BF16: the same result, rounded (ties away) or split (hi nearest-even, lo the rest)
    t = _attend(qkv, lens, heads, round_out=True)
    assert bool((R.bits(t) == R.bits(R.round_tf32_ties_away(ctx))).all()) and bool((R.bits(t) & 0x1FFF == 0).all())
    s = _attend(qkv, lens, heads, split_out=True)
    hi, lo = R.split_halves(s)
    assert bool((R.bits(hi) == R.bits(R.round_bf16_nearest_even(ctx))).all())
    assert bool((R.bits(lo) == R.bits(R.round_bf16_nearest_even(ctx - hi))).all())

    # a sequence's result does not depend on its neighbours: new q / k / v everywhere but in three sequences
    other = _qkv(lens, heads, scale, cuda, 12)
    keep = [i for i, n in enumerate(lens) if n in (17, 506, 1500)]
    for i in keep:
        other[cu[i]:cu[i + 1]] = qkv[cu[i]:cu[i + 1]]
    ctx2 = _attend(other, lens, heads)
    for i in keep:
        assert bool((R.bits(ctx2[cu[i]:cu[i + 1]]) == R.bits(ctx[cu[i]:cu[i + 1]])).all()), f"sequence {i} changed"
    assert not bool((R.bits(ctx2) == R.bits(ctx)).all())


def _vt_of(qkv, heads, fill=None):
    tokens, D = qkv.shape[0], heads * HD
    ld = (tokens + 3) // 4 * 4
    vt = torch.zeros(D, ld, device=qkv.device)
    vt[:, :tokens] = qkv[:, 2 * D:].T
    if fill is not None:
        vt.fill_(fill)
    return vt


def test_attention_fp32_routes(cuda):
    """With V^T and fp32 operands, 253 tokens is the last length of the tf32 V^T kernel: at max_seqlen 254 the kernel
    that reads V from qkv runs and V^T is not read (it holds NaN here).  Up to 253 both kernels accept the batch and agree
    to the order of the two rounded-P sums: twice the bound."""
    heads = 3
    lens = [254, 17, 197, 1]
    qkv = _qkv(lens, heads, 1.5, cuda, 13)
    a = _attend(qkv, lens, heads, vt=_vt_of(qkv, heads, fill=float("nan")))
    b = _attend(qkv, lens, heads)
    assert bool(torch.isfinite(a).all()) and bool((R.bits(a) == R.bits(b)).all())
    # max_seqlen decides, not the lengths: the same call with the rows declared as <= 253 would read V^T
    lens = [1, 17, 63, 64, 65, 197, 253, 128]
    qkv = _qkv(lens, heads, 1.5, cuda, 14)
    ref, mag, amp = R.attention_packed(qkv, _cu(lens), heads)
    own = _attend(qkv, lens, heads)
    poisoned = qkv.clone()
    poisoned[:, 2 * heads * HD:] = float("nan")     # the V^T kernel must not read the V columns of qkv
    tc = _attend(poisoned, lens, heads, vt=_vt_of(qkv, heads))
    assert bool(torch.isfinite(tc).all())
    r_own = float(((own.double() - ref).abs() / _bound(mag, amp)).max())
    r_tc = float(((tc.double() - ref).abs() / _bound(mag, amp)).max())
    r_two = float(((tc.double() - own.double()).abs() / (2 * _bound(mag, amp))).max())
    print(f"mer_attention <= 253 tokens: qkv kernel {r_own:.3f}, V^T kernel {r_tc:.3f} of the bound; apart {r_two:.3f}")
    assert r_own <= 1.0 and r_two <= 1.0
    assert not bool((R.bits(tc) == R.bits(own)).all()), "the V^T route was not taken"


def test_attention_fp32_refusals(cuda):
    heads, lens = 3, [300, 17]
    qkv = _qkv(lens, heads, 1.0, cuda, 15)
    cu = torch.tensor(_cu(lens), dtype=torch.int32, device=cuda)
    ctx = torch.full((sum(lens), heads * HD), float("nan"), device=cuda)
    before = L.launch_count()
    for max_seqlen in (300, 253):
        with pytest.raises(L.MerError, match=r"mer_attention: fp16 ctx needs V\^T"):
            L.attention(qkv, ctx.half(), cu, max_seqlen, heads, f16_out=True)
    with pytest.raises(L.MerError, match=r"mer_attention: fp16 ctx needs V\^T"):  # V^T given, but a row over 253 tokens
        L.attention(qkv, ctx.half(), cu, 300, heads, f16_out=True, vt=_vt_of(qkv, heads))
    q16 = qkv.half()
    vt16 = torch.zeros(heads * HD, 320, dtype=torch.float16, device=cuda)
    with pytest.raises(L.MerError, match=r"mer_attention: fp16 inputs need V\^T and sequences <= 505 tokens \(max_seqlen 506\)"):
        L.attention(q16, ctx, cu, 506, heads, vt=vt16)
    with pytest.raises(L.MerError, match="mer_attention: null operand"):
        L.check(L.lib().mer_attention(L.ptr(qkv), None, 0, None, L.ptr(cu), 2, sum(lens), 300, heads, 0, L.stream_ptr()))
    with pytest.raises(L.MerError, match=r"mer_attention: bad grid \(0 heads, 2 seqs\)"):
        L.attention(qkv, ctx, cu, 300, 0)
    with pytest.raises(L.MerError, match=r"mer_attention: bad grid \(3 heads, 65536 seqs\)"):
        L.check(L.lib().mer_attention(L.ptr(qkv), None, 0, L.ptr(ctx), L.ptr(cu), 65536, sum(lens), 300, heads, 0,
                                      L.stream_ptr()))
    # nothing to do: no sequences, or no tokens in any of them
    for n_seq, max_seqlen in ((0, 300), (2, 0)):
        L.check(L.lib().mer_attention(L.ptr(qkv), None, 0, L.ptr(ctx), L.ptr(cu), n_seq, sum(lens), max_seqlen, heads, 0,
                                      L.stream_ptr()))
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(ctx).all())


# ------------------------------------------------ WavLM: biased attention, gate ----
def _biased_bound(mag, units, T):
    """Plain fp32: a score is 64 chained FMAs and one more for the bias (`units` u, _kernel_refs.biased_attention), which
    moves a probability and the normaliser by that much each; the row sum adds T / 32 + 5 terms one after another and
    the P V column T; expf, the division and the stores a few u more."""
    return (2 * units + T + T / 32 + 16) * U * mag + 1e-30


@pytest.mark.parametrize("heads,batch", [(1, 3), (12, 1), (16, 3)])
@pytest.mark.parametrize("T", [1, 7, 8, 9, 33, 197, 499, 1024])
def test_biased_attention_vs_float64(cuda, T, heads, batch):
    """softmax_j((q_i / 8) . k_j + rowscale * bias_ij) v_j with masked keys (-1e4: probability exactly 0, whatever their
    1e30 values), one row whose every bias is -1e4 (a constant shift: the unbiased softmax, to the fp32 spacing at 1e4),
    rowscale absent and given with zeros and negative entries (a negative one turns the mask into the only visible keys)."""
    D = heads * HD
    g = _gen(1000 * T + heads)
    qkv = (torch.randn(batch * T, 3 * D, generator=g) * 1.5)
    bias = torch.randn(heads, T, T, generator=g) * 2.0
    masked = sorted({T - 1, 3}) if T > 4 else []
    for j in masked:
        bias[:, :, j] = -1e4
        qkv.view(batch, T, 3, D)[:, j, 2] = 1e30
    if T > 4:
        bias[:, T // 2, :] = -1e4
    rs = torch.rand(batch * T, heads, generator=g) * 2.0 + 0.25
    rs[1::5] = 0.0
    rs[2::7] *= -1.0
    qkv, bias, rs = qkv.to(cuda), bias.to(cuda), rs.to(cuda)
    worst = 0.0
    for rowscale in (None, rs):
        buf, ctx = R.guarded(batch * T, D, torch.float32, cuda)
        L.biased_attention(qkv, bias, rowscale, ctx, batch=batch, T=T, heads=heads)
        torch.cuda.synchronize()
        assert R.guards_intact(buf, batch * T) and bool(torch.isfinite(ctx).all())
        ref, mag, units = R.biased_attention(qkv, bias, rowscale, batch, T, heads)
        ratio = float(((ctx.double() - ref).abs() / _biased_bound(mag, units, T)).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (rowscale is None, ratio)
        if rowscale is None and masked:        # no masked key leaks: every row but the all-masked one stays far below 1e30
            rows = torch.ones(T, dtype=torch.bool)
            rows[T // 2] = False
            assert float(ctx.view(batch, T, D)[:, rows.to(cuda)].abs().max()) < 1e3
        buf2, rounded = R.guarded(batch * T, D, torch.float32, cuda)
        L.biased_attention(qkv, bias, rowscale, rounded, batch=batch, T=T, heads=heads, round_out=True)
        torch.cuda.synchronize()
        assert R.guards_intact(buf2, batch * T)
        assert bool((R.bits(rounded) == R.bits(R.round_tf32_ties_away(ctx))).all())
        assert bool((R.bits(rounded) & 0x1FFF == 0).all())
    print(f"mer_biased_attention T {T} heads {heads} batch {batch}: worst {worst:.3f} of the fp32 bound")


def test_biased_attention_refusals(cuda):
    heads, T = 2, 8
    qkv = torch.zeros(T + 1, 3 * heads * HD, device=cuda)
    bias = torch.zeros(heads, T, T, device=cuda)
    ctx = torch.full((T, heads * HD), float("nan"), device=cuda)
    before = L.launch_count()
    for kw, text in ((dict(batch=1, T=1025, heads=heads), r"batch 1, heads 2, T 1025 \(<= 1024\)"),
                     (dict(batch=1, T=0, heads=heads), r"batch 1, heads 2, T 0 \(<= 1024\)"),
                     (dict(batch=65536, T=T, heads=heads), r"batch 65536, heads 2, T 8 \(<= 1024\)"),
                     (dict(batch=0, T=T, heads=heads), r"batch 0, heads 2, T 8"),
                     (dict(batch=1, T=T, heads=0), r"batch 1, heads 0, T 8"),
                     (dict(batch=1, T=T, heads=65536), r"batch 1, heads 65536, T 8")):
        with pytest.raises(L.MerError, match="mer_biased_attention: " + text):
            L.biased_attention(qkv, bias, None, ctx, **kw)
    with pytest.raises(L.MerError, match="mer_biased_attention: qkv must be 16-byte aligned"):
        L.biased_attention(qkv.view(-1)[1:], bias, None, ctx, batch=1, T=T, heads=heads)
    with pytest.raises(L.MerError, match="mer_biased_attention: batch 1, heads 2, T 8"):
        L.biased_attention(qkv, None, None, ctx, batch=1, T=T, heads=heads)
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(ctx).all())


@pytest.mark.parametrize("heads", [12, 16])
@pytest.mark.parametrize("tokens", [1, 9, 4001])
def test_wavlm_gate_vs_float64(cuda, tokens, heads):
    """gate = ga (gb c - 1) + 2 with (ga, gb) the sigmoids of two sums of four 64-long dot products.  Each sum s carries
    (64 + 8) u M with M = sum |w x| + |b| over its four rows; a sigmoid's slope is at most 1 / 4, and the gate's slope in
    (ga, gb) at most 1 + |c|: (18 u M + 4 u)(1 + |c|) + 8 u.  Inputs of scale 20 saturate the sigmoids: no NaN."""
    g = _gen(tokens * 100 + heads)
    w, b, c = torch.randn(8, 64, generator=g), torch.randn(8, generator=g), torch.randn(heads, generator=g) * 2.0
    worst = 0.0
    for scale in (1.0, 20.0):
        x = torch.randn(tokens, heads * HD, generator=g) * scale
        xd, wd, bd, cd = (t.to(cuda) for t in (x, w, b, c))
        buf, gate = R.guarded(tokens, heads, torch.float32, cuda)
        L.wavlm_gate(xd, wd, bd, cd, gate, tokens=tokens, heads=heads)
        torch.cuda.synchronize()
        assert R.guards_intact(buf, tokens) and bool(torch.isfinite(gate).all())
        ref = R.wavlm_gate(xd, wd, bd, cd, heads)
        m = (xd.double().abs().view(tokens, heads, 64) @ wd.double().abs().T + bd.double().abs())      # [tokens, heads, 8]
        m = torch.maximum(m[..., :4].sum(-1), m[..., 4:].sum(-1))
        bound = (18 * U * m + 4 * U) * (1 + cd.double().abs()[None]) + 8 * U
        ratio = float(((gate.double() - ref).abs() / bound).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (scale, ratio)
        if scale == 20.0:   # saturated sigmoids reach their limits: gate in {2, 1, c + 1} up to rounding
            assert float(gate.min()) >= float(min(1.0, 1.0 + cd.min())) - 1e-6
    with pytest.raises(L.MerError, match="mer_wavlm_gate: bad arguments"):
        L.wavlm_gate(xd, wd, bd, cd, gate, tokens=0, heads=heads)
    with pytest.raises(L.MerError, match="mer_wavlm_gate: bad arguments"):
        L.wavlm_gate(xd, wd, bd, None, gate, tokens=tokens, heads=heads)
    print(f"mer_wavlm_gate tokens {tokens} heads {heads}: worst {worst:.3f} of the fp32 bound")


# ------------------------------------------------ Whisper decoder: small attention ----
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
@pytest.mark.parametrize("nk", [1, 3, 63, 64, 65, 127, 128, 129, 1500, 1536])
def test_small_attention_vs_float64(cuda, nk, causal):
    """nq 1 / 4 / 8 query rows against nk keys (below, at and above nq), with k and v as column blocks of one fused buffer
    (the decoder's cross-attention) or as buffers of their own, every pitch distinct and wider than heads * 64, NaN in the
    columns no head owns and, under `causal`, in the keys no query may see.  Bound as for the biased kernel, without the
    bias: a score is 64 chained FMAs (65 u A with the 1 / 8), the row sum nk / 128 + 8 terms, a P V column nk / 2 + 2."""
    worst = 0.0
    for (batch, heads, fused), nq in zip([(1, 1, True), (3, 6, False), (1, 20, True), (3, 6, True), (1, 1, False)],
                                         [1, 4, 8, 8, 4]):
        D = heads * HD
        g = _gen(nk * 100 + heads + nq)
        q, k, v = (torch.randn(batch, n, heads, HD, generator=g) * 1.5 for n in (nq, nk, nk))
        if causal:
            k[:, nq:], v[:, nq:] = float("nan"), float("nan")
        ld_q, ld_out = D + 8, D + 20
        qb = torch.full((batch * nq, ld_q), float("nan"))
        qb[:, 4:4 + D] = q.reshape(batch * nq, D)
        if fused:       # [4 NaN | k | 3 NaN | v | NaN ...]: k 16-byte aligned, v not
            ld_k = ld_v = 2 * D + 12
            kv = torch.full((batch * nk, ld_k), float("nan"))
            kv[:, 4:4 + D] = k.reshape(batch * nk, D)
            kv[:, 7 + D:7 + 2 * D] = v.reshape(batch * nk, D)
            kv = kv.to(cuda)
            kview, vview = kv[:, 4:], kv[:, 7 + D:]
        else:
            ld_k, ld_v = D + 4, D + 7
            kb, vb = torch.full((batch * nk, ld_k), float("nan")), torch.full((batch * nk, ld_v), float("nan"))
            kb[:, :D], vb[:, 5:5 + D] = k.reshape(batch * nk, D), v.reshape(batch * nk, D)
            kb, vb = kb.to(cuda), vb.to(cuda)
            kview, vview = kb, vb[:, 5:]
        qb = qb.to(cuda)
        buf, out = R.guarded(batch * nq, ld_out, torch.float32, cuda)
        L.small_attention(qb[:, 4:], kview, vview, out[:, 2:], ld_q=ld_q, ld_k=ld_k, ld_v=ld_v, ld_out=ld_out, batch=batch,
                          heads=heads, nq=nq, nk=nk, causal=causal)
        torch.cuda.synchronize()
        assert R.guards_intact(buf, batch * nq)
        assert bool(torch.isnan(out[:, :2]).all()) and bool(torch.isnan(out[:, 2 + D:]).all()), "padding column written"
        got = out[:, 2:2 + D]
        assert bool(torch.isfinite(got).all())
        ref, mag, amp = R.small_attention(q.to(cuda), k.to(cuda), v.to(cuda), causal)
        bound = (2 * 65 * amp + nk / 2 + nk / 128 + 16) * U * mag + 1e-30
        ratio = float(((got.double().view(batch, nq, heads, HD) - ref).abs() / bound).max())
        worst = max(worst, ratio)
        assert ratio <= 1.0, (batch, heads, nq, ratio)
    print(f"mer_small_attention nk {nk} causal {causal}: worst {worst:.3f} of the fp32 bound")


def test_small_attention_refusals(cuda):
    heads = 2
    D = heads * HD
    q = torch.zeros(9, D, device=cuda)
    kv = torch.zeros(1540, 2 * D + 4, device=cuda)
    out = torch.full((9, D), float("nan"), device=cuda)
    kw = dict(ld_q=D, ld_k=2 * D + 4, ld_v=2 * D + 4, ld_out=D, batch=1, heads=heads, nq=4, nk=16)
    before = L.launch_count()
    for change, text in ((dict(nq=9), r"9 queries \(<= 8\), 16 keys \(<= 1536\)"),
                         (dict(nk=1537), r"4 queries \(<= 8\), 1537 keys \(<= 1536\)"),
                         (dict(nq=0), r"0 queries"), (dict(nk=0), r"4 queries \(<= 8\), 0 keys"), (dict(batch=0), r"4 queries"),
                         (dict(heads=0), r"4 queries"),
                         (dict(ld_k=770), "k rows must be 16-byte aligned")):
        with pytest.raises(L.MerError, match="mer_small_attention: " + text):
            L.small_attention(q, kv, kv[:, D:], out, **{**kw, **change})
    with pytest.raises(L.MerError, match="mer_small_attention: k rows must be 16-byte aligned"):
        L.small_attention(q, kv.view(-1)[1:], kv[:, D:], out, **kw)
    torch.cuda.synchronize()
    assert L.launch_count() == before and bool(torch.isnan(out).all())
