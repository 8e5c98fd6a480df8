"""GPU tests of the MER2024 VideoMAE face-clip extractor: videomae_clips_kernel against the reference's transformed
tensors bit for bit, mer_videomae_forward against the float64 restatement per element and against the golden of the
unmodified reference driver, packing invariance, and the refusals of the C ABI."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import _sun_videomae_ref as R
from mertools_b200 import _lib as L
from mertools_b200.extract import sun_videomae as SV

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "sun_videomae_golden.npz")
NONSQUARE = {40: (120, 100)}
CASES = {"base160": ("vit_base_patch16_160", 2, 11), "base224": ("vit_base_patch16_224", 2, 12),
         "large224": ("vit_large_patch16_224", 1, 13)}
CLIPS = {"sq160": (160, 65, "UTTERANCE", 3), "ns224": (224, 40, "FRAME", 37), "wrap160": (160, 12, "FRAME", 10)}


def video(n):
    h, w = NONSQUARE.get(n, (112, 112))
    return R.synth_video(n, h, w, seed=100 + n)


_GOLDEN = dict(np.load(GOLDEN))
_EXT = {}


def extractor(case, dev, **kw):
    if (case, tuple(kw.items())) not in _EXT:
        model, blocks, seed = CASES[case]
        sd = SV.model_state_dict(R.synth_checkpoint(R.SHAPES[model][1], blocks, seed), model, n_layers=blocks)
        _EXT[(case, tuple(kw.items()))] = (SV.SunVideoMae(sd, model, device=dev, **kw), R.model_params(
            R.synth_checkpoint(R.SHAPES[model][1], blocks, seed)))
    return _EXT[(case, tuple(kw.items()))]


def _as_clip(out, S):
    """Kernel rows of one view [8 g^2, 1536] -> the [3, 16, S, S] clip tensor layout."""
    g = S // 16
    x = out.reshape(8, g, g, 3, 2, 16, 16)                   # t, py, px, c, dt, dy, dx
    return x.permute(3, 0, 4, 1, 5, 2, 6).reshape(3, 16, S, S)


def test_clips_kernel_is_the_reference_tensor(cuda):
    for name, (S, n, level, item) in CLIPS.items():
        rows = SV.plan_views(n, level)[item][1]
        frames = SV.resize_frames(video(n), S, cuda)
        table = torch.tensor([rows], dtype=torch.int32, device=cuda)
        f32 = _as_clip(SV.videomae_clips(frames, table, S, out_f32=True).cpu(), S)
        f16 = _as_clip(SV.videomae_clips(frames, table, S).cpu(), S)
        gold = torch.from_numpy(_GOLDEN[f"clip/{name}"])
        assert torch.equal(f32[:, :2, :32, :], gold), name
        assert torch.equal(f16[:, :2, :32, :], gold.half()), name
        # every token, against the restatement (the device resize is bit-exact Pillow)
        full = R.clip_tensor(R.resize(video(n), S), rows)
        assert torch.equal(f32, full) and torch.equal(f16, full.half()), name


def test_clips_kernel_many_views_and_bad_rows(cuda):
    frames = SV.resize_frames(video(19), 160, cuda)
    items = SV.plan_views(19, "FRAME")
    rows = [r for _, r in items[:19]]
    got = SV.videomae_clips(frames, torch.tensor(rows, dtype=torch.int32, device=cuda), 160, out_f32=True).cpu()
    rs = R.resize(video(19), 160)
    for v in (0, 9, 18):
        assert torch.equal(_as_clip(got[v * 800:(v + 1) * 800], 160), R.clip_tensor(rs, rows[v]))
    # frame 15 of the view (tubelet 7, dt = 1) is out of range: exactly the entries it feeds are NaN
    bad = torch.tensor([[0] * 15 + [19]], dtype=torch.int32, device=cuda)
    nan = torch.isnan(SV.videomae_clips(frames, bad, 160, out_f32=True).cpu()).reshape(8, 100, 3, 2, 256)
    assert nan[7, :, :, 1].all() and not nan[:7].any() and not nan[7, :, :, 0].any()


GOLD_KEYS = sorted(k for k in _GOLDEN if k.startswith("feat/"))


@pytest.mark.parametrize("key", GOLD_KEYS)
def test_forward_matches_golden(cuda, key):
    _, case, level, n = key.split("/")
    ext, _ = extractor(case, cuda)
    got = ext.extract_videos([video(int(n))], level)[0]
    ref = _GOLDEN[key].astype(np.float64)
    assert got.dtype == np.float64 and got.shape == ref.shape
    err = np.abs(got - ref).max() / np.abs(ref).max()
    print(f"{key}: max-abs / max-ref {err:.2e}")
    assert err <= 1e-3


@pytest.mark.parametrize("case,level,n", [("base160", "UTTERANCE", 150), ("base160", "FRAME", 12),
                                          ("base224", "FRAME", 19), ("base224", "UTTERANCE", 1),
                                          ("large224", "UTTERANCE", 65)])
def test_forward_matches_float64_per_element(cuda, case, level, n):
    """|got - ref| <= 1e-3 (max |ref| + |ref|) element by element against the float64 restatement: the fp16 operands
    round every GEMM input to 11 significant bits, fp32 accumulation and statistics elsewhere."""
    ext, params = extractor(case, cuda)
    got = ext.extract_videos([video(n)], level)[0]
    ref = R.video_features(params, video(n), CASES[case][0], level, dtype=torch.float64)
    bound = 1e-3 * (np.abs(ref).max() + np.abs(ref))
    r = float((np.abs(got - ref) / bound).max())
    print(f"{case} {level} n={n}: worst |err| / bound {r:.3f}")
    assert r <= 1.0


def test_packing_invariance(cuda):
    vids = [video(n) for n in (17, 40, 150, 1)]
    alone = [extractor("base160", cuda)[0].extract_videos([v], "FRAME")[0] for v in vids]
    packed = extractor("base160", cuda, views_per_launch=7)[0].extract_videos(vids, "FRAME")
    for a, p in zip(alone, packed):
        assert a.shape == p.shape
        assert np.abs(a - p).max() <= 1e-4 * np.abs(a).max()


def _call(ext, frames, rows, ws_bytes=None, model=None):
    rows = np.ascontiguousarray(np.asarray(rows, np.int32))
    nv = rows.shape[0]
    need = max(ext.workspace_bytes(nv), 1)
    ws = torch.empty(need if ws_bytes is None else 16, dtype=torch.uint8, device=ext.device)   # refused before use
    out = torch.empty(nv, ext.dim, device=ext.device)
    rc = ext._fwd(C.byref(model or ext.m), L.ptr(frames), frames.shape[0], rows.ctypes.data_as(C.c_void_p), nv,
                  L.ptr(ws), ws.numel() if ws_bytes is None else ws_bytes, L.ptr(out), L.stream_ptr())
    return rc, L.last_error() if rc else ""


def test_forward_refusals(cuda):
    ext, _ = extractor("base160", cuda)
    frames = SV.resize_frames(video(5), 160, cuda)
    rows = [list(SV.plan_views(5, "FRAME")[0][1])]
    assert _call(ext, frames, rows)[0] == 0
    rc, msg = _call(ext, frames, rows, ws_bytes=ext.workspace_bytes(1) - 1)
    assert rc and "workspace" in msg
    rc, msg = _call(ext, frames, [[0] * 15 + [5]])
    assert rc and "row" in msg
    rc, msg = _call(ext, frames, [[-1] + [0] * 15])
    assert rc and "row" in msg
    for field, value, text in [("heads", 11, "heads"), ("img", 192, "img"), ("img", 96, "img"),
                               ("patch_w", None, "null"), ("norm_b", None, "null")]:
        m = SV.MerVideoMaeModel.from_buffer_copy(ext.m)
        setattr(m, field, value)
        rc, msg = _call(ext, frames, rows, ws_bytes=1 << 40, model=m)
        assert rc and text in msg, (field, msg)
        assert L.lib().mer_videomae_workspace_bytes(C.byref(m), 1) == -1
    rc = ext._fwd(C.byref(ext.m), None, 5, np.zeros(16, np.int32).ctypes.data_as(C.c_void_p), 1, None, 0, None,
                  L.stream_ptr())
    assert rc and "null" in L.last_error()


def test_empty_video_is_refused(cuda):
    ext, _ = extractor("base160", cuda)
    with pytest.raises(ValueError, match="0 frames"):
        ext.extract_videos([np.zeros((0, 112, 112, 3), np.uint8)], "UTTERANCE")
