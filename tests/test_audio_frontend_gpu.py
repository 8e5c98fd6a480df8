"""Kernel-level parity of the two log-mel front ends against float64: mer_logmel (the VGGish front end, logmel.cu)
against oracle.pipeline.log_mel_spectrogram and mer_whisper_logmel (the Whisper front end, whisper.cu) against
oracle.pipeline.whisper_log_mel, both fed the fp32 samples the kernel reads, widened to float64.

mer_logmel: 1, 2, 8 and 9 frames (the partial last block of 8 frames), 1 s, 1.5 s, 10 s and 60 s; batch 1 and 3 at
row pitch n and n + 37 with NaN in the pitch tail; rows of a batch bit-identical to the row run alone.
mer_whisper_logmel: every signal kind at 30 s, short clips zero-padded to 30 s, bursts at the two reflect-padded ends,
clip maxima of log10 on both sides of zero (the two branches of the order-preserving integer image the per-clip maximum
is found on), batches mixing loud, quiet and silent clips, reuse of the scratch buffer, ld_out 80 / 96 / 97 and the
TF32-rounded form.  Both: refusals, and the launch counter moves by exactly the kernels launched (1 and 2).

Outputs sit between NaN guard rows; every parity test prints its worst |kernel - float64|.

Bars, absolute in the log domain, from a CPU emulation of each kernel's fp32 arithmetic (fp32 twiddles, window and mel
weights, sequential fp32 accumulation of the 400-term DFT and of the mel sums).  GPU sincospif / log10f / logf are not
emulated bit for bit, so the emulated worst cases are a guide, not a bound.

mer_logmel: 1.2e-4 emulated, on the quiet bands of full-scale tones, which carry the DFT's rounding error of the loud
bins; noise and quiet input stay below 1e-6.  Bar LOGMEL_TOL = 5e-4.

mer_whisper_logmel: the DFT's rounding error is a fixed fraction (~u sqrt(400)) of the frame's amplitude, so the
relative error of a band's power, and the error of its log10, grows by up to sqrt(10) for every decade the band lies
below the frame's loudest band.  The clamp at (clip maximum - 8) stops that growth: no unclamped value lies more than 8
decades below its frame's maximum, and a value more than 2 decades above the clamp lies less than 6 below it.  Signals
whose spectra fall smoothly through those 8 decades (a chirp, a tone between two bins: Hann side lobes) put values
right at the clamp; a tone on a bin centre or a DC offset does not (its other bins are exactly zero in float64 and
clamped).  Emulated on the chirp: 1.0e-5 more than 2 decades above the clamp, 4.6e-5 within them.  Bars: WHISPER_TOL
= 5e-5 above, WHISPER_EDGE_TOL = 2e-4 within the last 2 decades (0.5 in (x + 4) / 4 units) above the clamp level.

Worst errors seen on an H100 80GB HBM3 (700 W power limit): mer_logmel 1.3e-4 (1020 Hz tone); mer_whisper_logmel
9.5e-5 within the last 2 decades above the clamp (chirp), 9.1e-6 elsewhere (chirp).  Each bar stays far below what a
wrong window, reflection or clamp level moves."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import _kernel_refs as R
from mertools_b200 import _lib as L
from oracle import pipeline as P

pytestmark = pytest.mark.gpu

SR = 16000
LOGMEL_TOL = 5e-4
WHISPER_TOL, WHISPER_EDGE_TOL = 5e-5, 2e-4
WH_SAMPLES, WH_FRAMES, WH_MELS = 480000, 3000, 80

KINDS = ("speech", "silence", "dc", "tone_on_bin", "tone_off_bin", "square", "chirp", "int16", "quiet")


def signal(kind, n, seed=0):
    """fp32 [n] test signal of one kind: speech-like at 0.1, silence, a DC offset of 0.5, a full-scale sine on a DFT bin
    centre (1 kHz: bin 32 of 512, bin 25 of 400) or between bins (1020 Hz), a +-1 square wave (clipping), a linear chirp
    100 Hz -> 7.9 kHz at 0.5, int16-quantised noise at 0.1, or speech-like at 1e-3."""
    t = torch.arange(n, dtype=torch.float64) / SR
    if kind == "speech":
        x = 0.1 * R.speech_like(n, seed).double()
    elif kind == "silence":
        x = torch.zeros(n, dtype=torch.float64)
    elif kind == "dc":
        x = torch.full((n,), 0.5, dtype=torch.float64)
    elif kind == "tone_on_bin":
        x = torch.sin(2 * math.pi * 1000.0 * t)
    elif kind == "tone_off_bin":
        x = torch.sin(2 * math.pi * 1020.0 * t + 0.3)
    elif kind == "square":
        x = torch.where(torch.sin(2 * math.pi * 440.0 * t + 0.1) >= 0, 1.0, -1.0).double()
    elif kind == "chirp":
        x = 0.5 * torch.sin(2 * math.pi * (100.0 * t + 7800.0 / (2 * n / SR) * t * t))
    elif kind == "int16":
        g = torch.Generator().manual_seed(seed)
        x = torch.clamp(torch.round(0.1 * 32768 * torch.randn(n, generator=g, dtype=torch.float64)), -32768, 32767)
        x = x / 32768
    else:
        assert kind == "quiet"
        x = 1e-3 * R.speech_like(n, seed).double()
    return x.float()


def _rows(sigs, ld, device):
    """[B, ld] fp32 rows holding the signals, NaN past each one's end."""
    x = torch.full((len(sigs), ld), float("nan"), dtype=torch.float32)
    for b, s in enumerate(sigs):
        x[b, :len(s)] = s
    return x.to(device)


# ---- mer_logmel ------------------------------------------------------------------------------------------------------
def _nf(n):
    return 1 + (n - 400) // 160


def _logmel_fn():
    return L.declare("mer_logmel", [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p])


def _logmel(x, n):
    """mer_logmel on the rows of x [B, ld] (n samples each) into a guarded NaN buffer: [B, frames, 64] on the host."""
    B, ld = x.shape
    nf = _nf(n)
    buf, out = R.guarded(B * nf, 64, torch.float32, x.device)
    before = L.launch_count()
    L.check(_logmel_fn()(L.ptr(x), B, n, ld, L.ptr(out), L.stream_ptr()))
    assert L.launch_count() == before + 1
    torch.cuda.synchronize()
    assert R.guards_intact(buf, B * nf)
    return out.view(B, nf, 64).cpu()


LENGTHS = [400, 559, 560, 400 + 160 * 7, 400 + 160 * 8, 15999, 16000, 16001, 24000, 160000, 960000]


@pytest.mark.parametrize("n", LENGTHS)
def test_logmel_vs_float64(cuda, n):
    """Batch 3 (three different signal kinds, rotating with the length) and each row alone, at row pitch n and n + 37:
    every value within LOGMEL_TOL of float64, and each row of the batch bit-identical to its solo run."""
    i = LENGTHS.index(n)
    kinds = [KINDS[(i + 3 * j) % len(KINDS)] for j in range(3)]
    sigs = [signal(k, n, seed=n % 1000 + j) for j, k in enumerate(kinds)]
    refs = [torch.from_numpy(P.log_mel_spectrogram(s.double().numpy())) for s in sigs]
    assert L.lib().mer_logmel_num_frames(n) == _nf(n) == refs[0].shape[0]
    worst, where = 0.0, None
    for ld in (n, n + 37):
        x = _rows(sigs, ld, cuda)
        both = _logmel(x, n)
        for b, k in enumerate(kinds):
            solo = _logmel(x[b:b + 1].contiguous(), n)[0]
            assert bool((R.bits(solo) == R.bits(both[b])).all()), (k, ld)
            err = float((solo.double() - refs[b]).abs().max())
            assert err <= LOGMEL_TOL, (k, ld, err)
            if err >= worst:
                worst, where = err, k
    print(f"mer_logmel n={n} ({_nf(n)} frames) {kinds}: worst |y - float64| = {worst:.2e} ({where})")


def test_logmel_silence(cuda):
    """Silence is logf(0 + 0.01f) everywhere: within 2 ulp of float32(log(0.01))."""
    n = 16000 + 160 * 9
    y = _logmel(torch.zeros(2, n, device=cuda), n)
    target = np.float32(np.log(0.01))
    ulp = float(np.spacing(np.abs(target)))
    worst = float((y.double() - float(target)).abs().max())
    assert worst <= 2 * ulp
    print(f"mer_logmel silence: worst |y - float32(log 0.01)| = {worst / ulp:.1f} ulp")


def test_logmel_refusals(cuda):
    """Each bad call is refused with a mer_logmel: message before any launch."""
    n, B = 1600, 2
    x = torch.zeros(B, n, device=cuda)
    out = torch.empty(B * _nf(n) * 64, device=cuda)
    f = _logmel_fn()

    def call(wave=x.data_ptr(), batch=B, n=n, ld=n, o=out.data_ptr()):
        return f(wave, batch, n, ld, o, L.stream_ptr())

    before = L.launch_count()
    assert call() == 0
    torch.cuda.synchronize()
    assert L.launch_count() == before + 1
    cases = [dict(n=399, ld=399), dict(n=0, ld=0), dict(ld=n - 1), dict(batch=0), dict(batch=-1), dict(wave=None),
             dict(o=None)]
    for kw in cases:
        before = L.launch_count()
        assert call(**kw) != 0, kw
        assert "mer_logmel:" in L.last_error(), (kw, L.last_error())
        assert L.launch_count() == before, kw
    print(f"mer_logmel: {len(cases)} refusals, none launched")


# ---- mer_whisper_logmel ----------------------------------------------------------------------------------------------
_MEL = {}


def _mel(device):
    """The fp32 [201, 80] Slaney filter bank the Whisper extractor passes to the kernel."""
    if device not in _MEL:
        from mertools_b200.extract.whisper import whisper_mel_filters
        _MEL[device] = torch.from_numpy(np.ascontiguousarray(whisper_mel_filters(), np.float32)).to(device)
    return _MEL[device]


def _whisper_fn():
    return L.declare("mer_whisper_logmel", [C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                            C.c_void_p, C.c_void_p])


def _whisper(x, ld_out=WH_MELS, tf32=0, scratch=None):
    """mer_whisper_logmel on the rows of x [B, ld_wave] into a guarded NaN buffer [B * 3000, ld_out]: checks the guards
    and that pad columns 80 .. ld_out - 1 are +0.0, and returns columns 0..79 as [B, 3000, 80] on the host."""
    B, ldw = x.shape
    buf, out = R.guarded(B * WH_FRAMES, ld_out, torch.float32, x.device)
    if scratch is None:
        scratch = torch.full((B,), 0x7F7F7F7F, dtype=torch.int32, device=x.device)
    before = L.launch_count()
    L.check(_whisper_fn()(L.ptr(x), B, ldw, L.ptr(_mel(x.device)), L.ptr(out), ld_out, tf32, L.ptr(scratch),
                          L.stream_ptr()))
    assert L.launch_count() == before + 2
    torch.cuda.synchronize()
    assert R.guards_intact(buf, B * WH_FRAMES)
    v = out.view(B, WH_FRAMES, ld_out).cpu()
    assert bool((R.bits(v[..., WH_MELS:]) == 0).all()), "pad column not +0.0"
    return v[..., :WH_MELS].contiguous()


def _whisper_ref(s):
    """(whisper_log_mel of the fp32 samples [3000, 80] as float64, the clip's maximum of log10 before the clamp).  The
    largest value is never clamped, so the maximum is 4 * max - 4 of the output."""
    ref = torch.from_numpy(P.whisper_log_mel(s.double().numpy()).T.astype(np.float64))
    return ref, 4.0 * float(ref.max()) - 4.0


def _whisper_check(y, ref, mx, what):
    """Assert y [3000, 80] within the bars of float64 `ref` for a clip of maximum `mx`: WHISPER_EDGE_TOL for values
    within 2 decades above the clamp level (mx - 8 + 4) / 4, WHISPER_TOL elsewhere.  Returns the worst error of each."""
    err = (y.double() - ref).abs()
    edge = ref <= (mx - 4.0) / 4.0 + 0.5
    far = float(err[~edge].max()) if bool((~edge).any()) else 0.0
    near = float(err[edge].max()) if bool(edge.any()) else 0.0
    assert far <= WHISPER_TOL and near <= WHISPER_EDGE_TOL, (what, far, near)
    return far, near


def _padded(s):
    x = torch.zeros(WH_SAMPLES)
    x[:min(len(s), WH_SAMPLES)] = s[:WH_SAMPLES]
    return x


def _burst(where, seed):
    """Silence with full-scale noise in the first 2000 samples (reflect padding of frames 0 and 1) or in the last 60:
    inside frame 2999 near its window's tail (clip maximum -0.45), and at the centre of frame 3000 (+0.90), which is
    dropped and must not set the clip maximum: every other frame of this clip is clamped relative to it."""
    g = torch.Generator().manual_seed(seed)
    x = torch.zeros(WH_SAMPLES)
    k = 2000 if where == "start" else 60
    noise = torch.clamp(torch.randn(k, generator=g), -1.0, 1.0)
    if where == "start":
        x[:k] = noise
    else:
        x[-k:] = noise
    return x


# case: (clip builder, sign of the clip's maximum of log10)
WHISPER_CASES = {
    **{k: (lambda k=k: signal(k, WH_SAMPLES, seed=21), s) for k, s in (
        ("speech", +1), ("silence", -1), ("dc", +1), ("tone_on_bin", +1), ("tone_off_bin", +1), ("square", +1),
        ("chirp", +1), ("int16", -1), ("quiet", -1))},
    "int16_2s_padded": (lambda: _padded(signal("int16", 2 * SR, seed=22)), -1),
    "speech_10s_padded": (lambda: _padded(signal("speech", 10 * SR, seed=23)), +1),
    "tone_2s_padded": (lambda: _padded(signal("tone_on_bin", 2 * SR, seed=24)), +1),
    "burst_start": (lambda: _burst("start", 25), +1),
    "burst_end": (lambda: _burst("end", 26), -1),
}


@pytest.mark.parametrize("case", list(WHISPER_CASES))
def test_whisper_logmel_vs_float64(cuda, case):
    """One 30 s clip (ld_wave = 480000, ld_out = 80, no TF32 rounding) within the bars of float64 (_whisper_check).  The
    sign of the reference's clip maximum is asserted so that each case keeps exercising its branch of the integer
    image (bits >= 0 for a positive maximum, bits ^ 0x7fffffff for a negative one)."""
    make, sign = WHISPER_CASES[case]
    s = make()
    assert s.dtype == torch.float32 and s.numel() == WH_SAMPLES
    ref, mx = _whisper_ref(s)
    assert (mx > 0) == (sign > 0), (case, mx)
    y = _whisper(s[None].to(cuda))[0]
    far, near = _whisper_check(y, ref, mx, case)
    clamped = float((ref == ref.min()).all(1).double().mean())
    print(f"mer_whisper_logmel {case}: max log10 {mx:+.3f}, {100 * clamped:.0f}% of frames clamped, "
          f"worst |y - float64| = {far:.2e}, {near:.2e} within 2 decades of the clamp")


def test_whisper_logmel_batch_rows_are_independent(cuda):
    """Loud, quiet and silent clips in one batch at ld_wave = 480000 + 64 with a NaN tail: each clip bit-identical to
    its solo run and within the bars of float64; the silent clip is (log10f(1e-10f) + 4) / 4 = -1.5 everywhere."""
    sigs = [signal("square", WH_SAMPLES, 31), signal("quiet", WH_SAMPLES, 32), signal("silence", WH_SAMPLES)]
    x = _rows(sigs, WH_SAMPLES + 64, cuda)
    both = _whisper(x)
    worst = [0.0, 0.0]
    for b, s in enumerate(sigs):
        solo = _whisper(x[b:b + 1].contiguous())[0]
        assert bool((R.bits(solo) == R.bits(both[b])).all()), b
        ref, mx = _whisper_ref(s)
        assert (mx > 0) == (b == 0), (b, mx)
        worst = [max(w, e) for w, e in zip(worst, _whisper_check(both[b], ref, mx, b))]
    assert float((both[2].double() + 1.5).abs().max()) <= 1e-6
    print(f"mer_whisper_logmel batch (loud, quiet, silent): worst |y - float64| = {worst[0]:.2e}, {worst[1]:.2e} "
          f"within 2 decades of the clamp")


def test_whisper_logmel_scratch_reuse(cuda):
    """A loud batch, then a quiet one through the same scratch buffer: the second call equals a fresh run of the quiet
    batch (the per-clip maxima start over on every call)."""
    loud = _rows([signal("tone_on_bin", WH_SAMPLES), signal("square", WH_SAMPLES)], WH_SAMPLES, cuda)
    quiet = _rows([signal("quiet", WH_SAMPLES, 41), signal("int16", WH_SAMPLES, 42)], WH_SAMPLES, cuda)
    scratch = torch.empty(2, dtype=torch.int32, device=cuda)
    _whisper(loud, scratch=scratch)
    again = _whisper(quiet, scratch=scratch)
    fresh = _whisper(quiet)
    assert bool((R.bits(again) == R.bits(fresh)).all())
    for b in range(2):
        ref, mx = _whisper_ref(quiet[b].cpu())
        assert mx < 0
        _whisper_check(again[b], ref, mx, b)


@pytest.mark.parametrize("ld_out", [80, 96, 97])
def test_whisper_logmel_output_forms(cuda, ld_out):
    """ld_out 80, 96 (the K-padded operand of the first convolution) and 97: columns 0..79 bit-identical across them,
    pad columns +0.0 (in _whisper); round_tf32_out = 1 gives the ties-away TF32 rounding of the unrounded values, bit
    for bit."""
    x = _rows([signal("chirp", WH_SAMPLES), signal("int16", WH_SAMPLES, 51)], WH_SAMPLES, cuda)
    base = _whisper(x, ld_out=WH_MELS)
    plain = _whisper(x, ld_out=ld_out)
    rounded = _whisper(x, ld_out=ld_out, tf32=1)
    assert bool((R.bits(plain) == R.bits(base)).all())
    assert bool((R.bits(rounded) == R.bits(R.round_tf32_ties_away(plain))).all())
    assert bool((rounded != plain).any())


def test_whisper_logmel_refusals(cuda):
    """Each bad call is refused with a mer_whisper_logmel: message before any launch (and before the scratch memset)."""
    B = 2
    x = torch.zeros(B, WH_SAMPLES, device=cuda)
    out = torch.empty(B * WH_FRAMES * 96, device=cuda)
    scratch = torch.empty(B, dtype=torch.int32, device=cuda)
    f = _whisper_fn()
    mel = _mel(cuda)

    def call(wave=x.data_ptr(), batch=B, ld=WH_SAMPLES, m=mel.data_ptr(), o=out.data_ptr(), ld_out=96,
             sc=scratch.data_ptr()):
        return f(wave, batch, ld, m, o, ld_out, 1, sc, L.stream_ptr())

    before = L.launch_count()
    assert call() == 0
    torch.cuda.synchronize()
    assert L.launch_count() == before + 2
    cases = [dict(ld=WH_SAMPLES - 1), dict(ld_out=79), dict(ld_out=0), dict(sc=None), dict(m=None), dict(wave=None),
             dict(o=None), dict(batch=0), dict(batch=-1)]
    for kw in cases:
        scratch.fill_(12345)
        torch.cuda.synchronize()
        before = L.launch_count()
        assert call(**kw) != 0, kw
        assert "mer_whisper_logmel:" in L.last_error(), (kw, L.last_error())
        assert L.launch_count() == before, kw
        torch.cuda.synchronize()
        assert bool((scratch == 12345).all()), kw
    print(f"mer_whisper_logmel: {len(cases)} refusals, none launched")
