"""Kernel-level parity of the HuBERT front end against float64 (tests/_kernel_refs.py): conv0 through mer_hubert_conv0
in both GroupNorm kernel forms and both output formats, the LayerNorm form, per-clip statistics of ragged batches, the
refusals of mer_hubert_conv0, and hidden_states[0] of mer_hubert_frontend for every front-end form (GroupNorm / LayerNorm
feature encoder, fp16 / split conv1 and conv2, the positional conv as the windowed GEMM, the mma.sync kernel, or the
data2vec chain).

Outputs sit between NaN guard rows, with NaN in the padded rows of every batch stride; every test prints its worst
|kernel - float64| / bound."""
import ctypes as C

import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L
from mertools_b200.encoders import HubertEncoder, MerHubertModel

pytestmark = pytest.mark.gpu
PAD = 3           # rows past T0 inside each clip's batch stride; they must stay NaN
SPLIT_NAN = 0x7FC17FC1


def _t0(n):
    return (n - 10) // 5 + 1


def _model(w0, gamma, beta, bias=None, family="group"):
    m = MerHubertModel()
    m.conv0_w = w0.data_ptr()
    if family == "group":
        m.gn_g, m.gn_b = gamma.data_ptr(), beta.data_ptr()
    else:
        m.feat_norm_layer = 1
        m.conv_ln_g[0], m.conv_ln_b[0] = gamma.data_ptr(), beta.data_ptr()
        m.conv_b[0] = bias.data_ptr() if bias is not None else None
    return m


def _conv0(m, wave, n, f16, frames=None, ld=None):
    """mer_hubert_conv0 into a guarded NaN buffer of batch stride (T0 + PAD) rows.  Returns [B, T0, 512] float64 after
    checking the guards and the padded rows."""
    B, T0 = wave.shape[0], _t0(n)
    rows = B * (T0 + PAD)
    buf, out = R.guarded(rows, 512, torch.float16 if f16 else torch.float32, wave.device)
    if not f16:
        buf.view(torch.int32).fill_(SPLIT_NAN)
    L.hubert_conv0(m, wave, out, batch=B, n_samples=n, ld_wave=ld or wave.shape[1], out_bstride=(T0 + PAD) * 512,
                   frames=frames, f16_out=f16)
    torch.cuda.synchronize()
    v = out.view(B, T0 + PAD, 512)
    pad = v[:, T0:]
    if f16:
        assert bool(torch.isnan(buf[:2]).all() and torch.isnan(buf[-2:]).all()), "guard row written"
        assert bool(torch.isnan(pad).all()), "row past T0 written"
        return v[:, :T0].double()
    assert bool((buf[:2].view(torch.int32) == SPLIT_NAN).all() and (buf[-2:].view(torch.int32) == SPLIT_NAN).all())
    assert bool((pad.view(torch.int32) == SPLIT_NAN).all()), "row past T0 written"
    hi, lo = R.split_halves(v[:, :T0])
    return hi.double() + lo.double()


def _weights(cuda, seed):
    return [t.to(cuda) for t in R.conv0_weights(seed)]


def _clips(n, B, cuda, seed):
    """Row 0, 3, ...: speech-like, normalised on the device (mer_wave_normalize); the others raw (normalize=0): a DC
    offset 100x the noise, silence, a constant."""
    raw = torch.stack([R.speech_like(n, seed + b) for b in range(B)]).to(cuda)
    x = torch.empty_like(raw)
    L.wave_normalize(raw, x, batch=B, n_samples=n, ld_in=n, ld_out=n)
    for b in range(B):
        k = b % 4
        if k == 1:
            x[b] = R.speech_like(n, seed + 50 + b, dc=30.0).to(cuda)
        elif k == 2:
            x[b] = 0.0
        elif k == 3:
            x[b] = 0.25
    torch.cuda.synchronize()
    return x


LENGTHS = [10, 15, 400, 645, 650, 655, 5125, 5130, 80000, 160000]


@pytest.mark.parametrize("f16", [False, True], ids=["split", "f16"])
@pytest.mark.parametrize("n", LENGTHS)
def test_conv0_group_norm_vs_float64(cuda, n, f16):
    """Both kernel forms (packed: four frames per window with a tail loop; MER_CONV0_PACKED=0: one channel per thread)
    against float64 within the derived bound, at T0 = 1, 2, the nt % 4 tails at the 128-frame chunk edge, the
    1024-frame moments chunk edge, 5 s and 10 s; and against each other within the sum of their bounds."""
    w0, gamma, beta, _ = _weights(cuda, 11)
    m = _model(w0, gamma, beta)
    worst = 0.0
    for B in ((1, 3, 16) if n <= 5130 else (1, 3) if n <= 80000 else (1,)):
        x = _clips(n, B, cuda, seed=n % 97 + B)
        ref, bound = R.hubert_conv0(x, w0, gamma, beta, f16=f16)
        outs = []
        for form in (None, "0"):
            with R.env("MER_CONV0_PACKED", form):
                y = _conv0(m, x, n, f16)
            r = float(((y - ref).abs() / bound).max())
            assert r <= 1.0, (B, form, r)
            worst = max(worst, r)
            outs.append(y)
        assert bool(((outs[0] - outs[1]).abs() <= 2 * bound).all()), B
        del ref, bound, outs, y
    print(f"conv0 GroupNorm n={n} {'fp16' if f16 else 'split'}: worst |y - float64| / bound = {worst:.3f}")


@pytest.mark.parametrize("bias", [True, False], ids=["bias", "no_bias"])
@pytest.mark.parametrize("T0", [1, 31, 32, 33, 15999])
def test_conv0_layer_norm_vs_float64(cuda, T0, bias):
    """conv0_ln_kernel (32 frames per block, 4 per warp) with and without the conv bias (hubert-large / data2vec), on a
    normalised clip, a quiet one (amplitude 1e-3: the LayerNorm's variance near eps) and silence."""
    n = 5 * (T0 - 1) + 10
    w0, gamma, beta, b0 = _weights(cuda, 12)
    m = _model(w0, gamma, beta, b0 if bias else None, family="layer")
    x = _clips(n, 3, cuda, seed=T0)
    x[1] = x[0] * 1e-3
    x[2] = 0.0
    ref, bound = R.hubert_conv0(x, w0, gamma, beta, family="layer", bias=b0 if bias else None)
    y = _conv0(m, x, n, False)
    worst = float(((y - ref).abs() / bound).max())
    assert worst <= 1.0
    print(f"conv0 LayerNorm T0={T0} bias={bias}: worst |y - float64| / bound = {worst:.3f}")


def test_conv0_ragged_clips_equal_their_solo_runs(cuda):
    """Clips of different lengths in one call with per-clip frame counts: each normalised over its own samples, a 1e3
    tail past its last sample.  A clip's valid frames equal the clip run alone -- bit for bit up to 1024 frames (one
    atomicAdd of the moments onto zero), within the bound beyond (the chunk order of the moments is not fixed) -- and
    frames past its count are finite."""
    w0, gamma, beta, _ = _weights(cuda, 13)
    m = _model(w0, gamma, beta)
    lens = [80000, 5125, 650, 15, 5130, 10]
    ld = max(lens) + 64
    raw = torch.stack([torch.nn.functional.pad(R.speech_like(k, 70 + i), (0, ld - k)) for i, k in enumerate(lens)])
    raw = raw.to(cuda)
    x = torch.full_like(raw, 1e3)
    for b, k in enumerate(lens):
        L.wave_normalize(raw[b:b + 1], x[b:b + 1], batch=1, n_samples=k, ld_in=ld, ld_out=ld)
    torch.cuda.synchronize()
    n = max(lens)
    frames = torch.tensor([_t0(k) for k in lens], dtype=torch.int32, device=cuda)
    worst = 0.0
    for f16 in (False, True):
        y = _conv0(m, x, n, f16, frames=frames, ld=ld)
        for b, k in enumerate(lens):
            t = _t0(k)
            assert bool(torch.isfinite(y[b]).all()), b
            solo = _conv0(m, x[b:b + 1], k, f16, ld=ld)[0]
            ref, bound = R.hubert_conv0(x[b:b + 1, :k], w0, gamma, beta, f16=f16)
            r = float(((y[b, :t] - ref[0]).abs() / bound[0]).max())
            assert r <= 1.0, (b, r)
            worst = max(worst, r)
            if t <= 1024:
                assert bool((y[b, :t] == solo).all()), (b, k)
            else:
                assert bool(((y[b, :t] - solo).abs() <= 2 * bound[0]).all()), (b, k)
    print(f"ragged conv0: worst |y - float64| / bound = {worst:.3f}")


def test_conv0_refusals(cuda):
    """Each bad call is refused before any launch, with its error text."""
    w0, gamma, beta, b0 = _weights(cuda, 14)
    gm, lm = _model(w0, gamma, beta), _model(w0, gamma, beta, b0, family="layer")
    n, B = 4005, 2
    T0 = _t0(n)
    x = torch.zeros(B, n, device=cuda)
    out = torch.empty(B * T0 * 512, device=cuda)
    need = L.hubert_conv0_workspace_bytes(B)
    assert need == 5120 * B
    ws = torch.empty(need + 16, dtype=torch.uint8, device=cuda)
    f = L.declare("mer_hubert_conv0", [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_int,
                                       C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p])

    def call(m=gm, n=n, ld=n, fmt=L.MER_EPI_SPLIT_BF16, stride=T0 * 512, wsp=ws.data_ptr(), wsb=need):
        return f(C.byref(m), x.data_ptr(), B, n, ld, None, fmt, out.data_ptr(), stride, wsp, wsb, L.stream_ptr())

    assert call() == 0
    torch.cuda.synchronize()
    cases = [
        (dict(wsb=need - 1), "workspace"),
        (dict(wsp=ws.data_ptr() + 8), "aligned"),
        (dict(wsp=None, wsb=0), "workspace"),
        (dict(ld=n - 1), "row pitch"),
        (dict(stride=T0 * 512 - 1), "batch stride"),
        (dict(fmt=0), "output format"),
        (dict(fmt=L.MER_EPI_OUT_F16, stride=T0 * 512 + 1), "output format"),
        (dict(m=lm, fmt=L.MER_EPI_OUT_F16), "split-bf16 rows only"),
        (dict(n=9, ld=9), "too short"),
    ]
    for kw, text in cases:
        before = L.launch_count()
        assert call(**kw) != 0, kw
        assert text in L.last_error(), (kw, L.last_error())
        assert L.launch_count() == before, kw
    print(f"mer_hubert_conv0: {len(cases)} refusals, none launched")


FRONT = {  # form: (state-dict options, HubertEncoder options, MER_POSCONV_LEGACY)
    "base_f16conv": (dict(), dict(conv_precision="f16", stack_precision="f16"), None),
    "base_bf16x3conv": (dict(), dict(conv_precision="bf16x3"), None),
    "base_mma_posconv": (dict(), dict(conv_precision="bf16x3"), "1"),
    "large": (dict(large=True), dict(), None),
    "w2v2_large_960h": (dict(large=True, group_norm=True), dict(), None),
    "data2vec": (dict(data2vec=True), dict(), None),
}
FRAMES = [1, 2, 63, 64, 65, 128, 129, 249, 499]


@pytest.mark.parametrize("form", list(FRONT))
def test_frontend_hidden0_vs_float64(cuda, form):
    """mer_hubert_frontend -> hidden_states[0] (after encoder.layer_norm for the post-LN families, the positional-conv
    sum for the stable one) against the float64 oracle, restated with its error bound (hubert_hidden0), at 1 .. 499
    frames (the 64-frame tile of posconv_kernel and the 128-row GEMM tiles), batch 1 and 3.  The first clip of a batch
    equals the clip run alone: bit for bit while conv0 has <= 1024 frames, within the bound beyond (moments order)."""
    from mertools_b200.synthetic import hubert_state_dict
    sd_kw, enc_kw, legacy = FRONT[form]
    sd = R.fp16_exact_front_end(hubert_state_dict(seed=31, layers=4, **sd_kw))
    with R.env("MER_POSCONV_LEGACY", legacy):
        enc = HubertEncoder(sd, device=cuda, **enc_kw)
    if legacy:
        assert enc.model.pos_w_bd is None       # mer_hubert_frontend runs posconv_kernel
    conv_f16 = bool(enc.model.conv_w_f16[0])
    assert conv_f16 == (form == "base_f16conv")
    fe = L.declare("mer_hubert_frontend", [C.POINTER(MerHubertModel), C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p])
    lib = L.lib()

    def run(x):
        B, n = x.shape
        T, D = enc.num_frames(n), enc.hidden
        ws = torch.empty(lib.mer_hubert_model_workspace_bytes(C.byref(enc.model), B, n), dtype=torch.uint8,
                         device=cuda)
        buf, h0 = R.guarded(B * T, D, torch.float32, cuda)
        L.check(fe(C.byref(enc.model), L.ptr(x), B, n, 0, L.ptr(ws), ws.numel(), L.ptr(h0), L.stream_ptr()))
        torch.cuda.synchronize()
        assert R.guards_intact(buf, B * T)
        return h0.view(B, T, D).double()

    worst = 0.0
    for T in FRAMES:
        n = 400 + 320 * (T - 1) + 7
        assert enc.num_frames(n) == T
        raw = torch.stack([R.speech_like(n, 90 + T + b) for b in range(3)]).to(cuda)
        x = torch.empty_like(raw)
        L.wave_normalize(raw, x, batch=3, n_samples=n, ld_in=n, ld_out=n)
        ref, bound = R.hubert_hidden0(sd, x, conv_f16=conv_f16)
        solo = run(x[:1].contiguous())
        both = run(x)
        for y, r, b in ((solo, ref[:1], bound[:1]), (both, ref, bound)):
            ratio = float(((y - r).abs() / b).max())
            assert ratio <= 1.0, (T, y.shape[0], ratio)
            worst = max(worst, ratio)
        if _t0(n) <= 1024:
            assert bool((solo[0] == both[0]).all()), T
        else:
            assert bool(((solo[0] - both[0]).abs() <= 2 * bound[0]).all()), T
    print(f"hidden_states[0] {form}: worst |h0 - float64| / bound = {worst:.3f}")
