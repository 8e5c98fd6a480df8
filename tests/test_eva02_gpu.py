"""GPU tests of the EVA02 tower (MER_VISION_EVA02): mer_rope2d_f16 and mer_swiglu_ln against float64 per element, the
tower against the golden of the unmodified reference (through the stand-in) and against the float64 restatement layer
by layer, batching invariance, the CLI end to end, and the refusals of malformed variant-3 models."""
import ctypes as C
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import _eva02_ref as R  # noqa: E402
import make_golden_eva02 as G  # noqa: E402
import timm_eva_shim as T  # noqa: E402
from mertools_b200 import _lib as L  # noqa: E402
from mertools_b200 import encoders as E  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402
from mertools_b200.extract import visual as V  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = dict(np.load(os.path.join(HERE, "golden", "eva02_golden.npz")))
TABLE = json.load(open(os.path.join(HERE, "..", "profiles", "eva02_precision_table.json")))
vp, i32, i64 = C.c_void_p, C.c_int, C.c_longlong


def _bar(case, scheme="f16"):
    """1e-3 on the default checkpoint; on the x5 one twice the 12-block emulated error of the precision table."""
    if case == "default":
        return 1e-3
    err = next(r["readout_max_rel"] for r in TABLE["rows"] if r["weights"] == "x5" and r["scheme"] == scheme)
    return max(1e-3, 2 * err)


def _ulp16(a):
    """spacing of fp16 at |a| (subnormal spacing 2^-24 near zero)"""
    return np.spacing(np.abs(a).astype(np.float16)).astype(np.float64)


@pytest.mark.parametrize("frames", [1, 7])
def test_rope2d_is_one_rounding_of_the_float64_rotation(cuda, frames):
    tpf, heads, ld, guard = 257, 12, 2304, 3
    rope = L.declare("mer_rope2d_f16", [vp, i64, i64, i32, i32, i32, i32, vp, vp, i32, vp])
    cos, sin = E.eva02_rope_tables(16)
    ct, st = torch.from_numpy(cos).to(cuda), torch.from_numpy(sin).to(cuda)
    M = frames * tpf
    g = torch.Generator().manual_seed(frames)
    buf = (torch.randn(M + 2 * guard, ld, generator=g) * 3).half().to(cuda)
    before = buf.clone()
    qkv = buf[guard:guard + M]
    L.check(rope(L.ptr(qkv), ld, M, tpf, 1, heads, 64, L.ptr(ct), L.ptr(st), 256, L.stream_ptr()))
    torch.cuda.synchronize()
    got, x = buf.cpu(), before.cpu()
    assert torch.equal(got[:guard], x[:guard]) and torch.equal(got[guard + M:], x[guard + M:])   # guard rows
    assert torch.equal(got[:, 2 * heads * 64:], x[:, 2 * heads * 64:])                           # V columns
    rows = np.arange(M)
    assert torch.equal(got[guard + rows[rows % tpf == 0]], x[guard + rows[rows % tpf == 0]])      # class rows
    patch = rows[rows % tpf != 0]
    xin = x[guard + patch, :2 * heads * 64].double().numpy().reshape(len(patch), 2 * heads, 32, 2)
    p = (patch % tpf) - 1
    c, s = cos[p].astype(np.float64)[:, None, :], sin[p].astype(np.float64)[:, None, :]
    a, b = xin[..., 0], xin[..., 1]
    ref = np.stack([a * c - b * s, b * c + a * s], -1)
    out = got[guard + patch, :2 * heads * 64].double().numpy().reshape(ref.shape)
    # one fp16 rounding of the fp32 result, plus the fp32 products and sum (3 units of 2^-24 of the terms)
    mag = np.stack([np.abs(a * c) + np.abs(b * s), np.abs(b * c) + np.abs(a * s)], -1)
    bound = 0.5 * np.maximum(_ulp16(ref), _ulp16(out)) + 3 * 2.0 ** -24 * mag
    ratio = float((np.abs(out - ref) / bound).max())
    print(f"mer_rope2d_f16 {frames} frames: worst |err| / bound {ratio:.3f}")
    assert ratio <= 1.0


def test_rope2d_refusals(cuda):
    rope = L.declare("mer_rope2d_f16", [vp, i64, i64, i32, i32, i32, i32, vp, vp, i32, vp])
    cos = torch.zeros(256, 32, device=cuda)
    q = torch.zeros(257, 2304, dtype=torch.float16, device=cuda)
    n0 = _launches()
    for args, text in [((2304, 257, 257, 1, 12, 128, 256), "head_dim"), ((2304, 257, 257, 1, 12, 64, 255), "table"),
                       ((2304, 256, 257, 1, 12, 64, 256), "whole frames"), ((1000, 257, 257, 1, 12, 64, 256), "layout")]:
        ld, M, tpf, pre, h, hd, rows = args
        rc = rope(L.ptr(q), ld, M, tpf, pre, h, hd, L.ptr(cos), L.ptr(cos), rows, L.stream_ptr())
        assert rc and text in L.last_error(), (args, L.last_error())
    assert _launches() == n0


def _launches():
    L.lib().mer_launch_count.restype = C.c_longlong
    return L.lib().mer_launch_count()


@pytest.mark.parametrize("out_f16", [1, 0])
def test_swiglu_ln_against_float64(cuda, out_f16):
    fn = L.declare("mer_swiglu_ln", [vp, vp, vp, C.c_float, vp, i64, i32, i32, vp])
    rows, H, eps = 300, 2048, 1e-6
    g = torch.Generator().manual_seed(out_f16)
    inp = torch.randn(rows, 2 * H, generator=g) * 2
    inp[:, :H] += torch.linspace(-6, 6, H)          # gate values over silu's whole shape
    gamma, beta = 1 + 0.3 * torch.randn(H, generator=g), 0.2 * torch.randn(H, generator=g)
    out = torch.empty(rows, H, dtype=torch.float16 if out_f16 else torch.float32, device=cuda)
    d_in, d_g, d_b = inp.to(cuda), gamma.to(cuda), beta.to(cuda)
    L.check(fn(L.ptr(d_in), L.ptr(d_g), L.ptr(d_b), eps, L.ptr(out), rows, H, out_f16, L.stream_ptr()))
    got = out.double().cpu().numpy()
    x = inp.double()
    prod = torch.nn.functional.silu(x[:, :H]) * x[:, H:]
    z = ((prod - prod.mean(1, keepdim=True)) / torch.sqrt(prod.var(1, unbiased=False, keepdim=True) + eps)).numpy()
    ref = z * gamma.double().numpy() + beta.double().numpy()
    half_ulp = 0.5 * (np.maximum(_ulp16(ref), _ulp16(got)) if out_f16 else np.abs(ref) * 2.0 ** -10)
    # fp32 silu / product / statistics: 2^-16 of |gamma| (|z| + 1) covers the error of the normalised value
    bound = half_ulp + 2.0 ** -16 * np.abs(gamma.double().numpy()) * (np.abs(z) + 1) + 2.0 ** -24
    if not out_f16:
        assert np.all((out.cpu().view(torch.int32).numpy() & 0x1fff) == 0)   # tf32-rounded
    ratio = float((np.abs(got - ref) / bound).max())
    print(f"mer_swiglu_ln out_f16={out_f16}: worst |err| / bound {ratio:.3f}")
    assert ratio <= 1.0


def test_swiglu_ln_refuses_widths(cuda):
    fn = L.declare("mer_swiglu_ln", [vp, vp, vp, C.c_float, vp, i64, i32, i32, vp])
    a = torch.zeros(4, 2 * 4224, device=cuda)
    o = torch.zeros(4, 4224, device=cuda)
    n0 = _launches()
    for H in (2730, 0, 4224, 2048 + 64):
        rc = fn(L.ptr(a), L.ptr(a), L.ptr(a), 1e-6, L.ptr(o), 4, H, 1, L.stream_ptr())
        assert rc and "width" in L.last_error(), H
    assert fn(L.ptr(a), L.ptr(a), L.ptr(a), 1e-6, L.ptr(a), 4, 2048, 1, L.stream_ptr()) and "alias" in L.last_error()
    assert _launches() == n0


_ENC = {}


def encoder(case, dev, precision="f16", layers=G.BLOCKS):
    key = (case, precision, layers)
    if key not in _ENC:
        seed, scale = G.CASES[case]
        _ENC[key] = E.Eva02Encoder(S.eva02_state_dict(seed, layers=layers, scale=scale), device=dev,
                                   precision=precision)
    return _ENC[key]


@pytest.mark.parametrize("precision", ["f16", "tf32"])
@pytest.mark.parametrize("case", list(G.CASES))
def test_tower_matches_the_golden(cuda, case, precision):
    seed, scale = G.CASES[case]
    ext = V.VisualExtractor(S.eva02_state_dict(seed, layers=G.BLOCKS, scale=scale), device=cuda)
    ext.enc = encoder(case, cuda, precision)
    assert isinstance(ext.enc, E.Eva02Encoder) and ext.feature_dim == 768
    vids = list(G.CLIPS)
    for level in ("FRAME", "UTTERANCE"):
        outs = ext.extract_clips([G.faces(v) for v in vids], level)
        for vid, got in zip(vids, outs):
            ref = GOLDEN[f"feat/{case}/{level}/{vid}"]
            assert got.shape == ref.shape, (vid, got.shape, ref.shape)
            err = float(np.abs(got - ref).max() / np.abs(ref).max())
            print(f"{case} {precision} {level} {vid}: max-abs / max-ref {err:.2e}")
            assert err <= _bar(case, precision), (case, level, vid, err)


def test_dispatch_picks_eva02(cuda):
    ext = V.VisualExtractor(S.eva02_state_dict(27, layers=1), device=cuda)
    assert isinstance(ext.enc, E.Eva02Encoder) and ext.enc.precision == "f16"


def test_hidden_states_against_float64(cuda):
    enc = encoder("default", cuda)
    frames = G.faces("r03")
    emb, hid = enc.frame_features(torch.from_numpy(frames).to(cuda), return_hidden=True)
    seed, scale = G.CASES["default"]
    lay = E.eva02_to_clip_layout(S.eva02_state_dict(seed, layers=G.BLOCKS, scale=scale))
    tf = T.create_transform(**T.resolve_model_data_config(T.Eva(depth=0)))
    ref_emb, ref_hid = R.forward(lay, R.pixels_from_frames(frames, tf), return_hidden=True)
    hid = hid.double().cpu()
    for i in range(G.BLOCKS + 1):
        err = float((hid[i] - ref_hid[i]).abs().max() / ref_hid[i].abs().max())
        print(f"hidden state {i}: max-abs / max-ref {err:.2e}")
        assert err <= 1e-3, (i, err)   # state 0 carries the TF32 patch embedding (K = 588)
    err = float((emb.double().cpu() - ref_emb).abs().max() / ref_emb.abs().max())
    assert err <= 1e-3, err


def test_features_do_not_depend_on_the_batch(cuda):
    enc = encoder("default", cuda)
    a = torch.from_numpy(G.faces("v05")).to(cuda)
    b = torch.from_numpy(G.faces("v33")).to(cuda)
    alone = enc.frame_features(a).cpu()
    both = enc.frame_features(torch.cat([b[:20], a, b[20:]])).cpu()
    # the same rows to within a few fp16 operand roundings (the GEMM tiling follows the row count)
    err = float((alone - both[20:25]).abs().max() / alone.abs().max())
    print(f"batched vs alone: max-abs / max-ref {err:.2e}")
    assert err <= 1e-4


def test_cli_writes_the_golden(cuda, tmp_path):
    from safetensors.numpy import save_file
    face = tmp_path / "face"
    for vid in G.CLIPS:
        (face / vid).mkdir(parents=True)
        np.save(face / vid / f"{vid}.npy", G.faces(vid))
    ck = tmp_path / "models" / "timm" / V.EVACLIP_VIT
    ck.mkdir(parents=True)
    seed, scale = G.CASES["default"]
    save_file(S.eva02_state_dict(seed, layers=G.BLOCKS, scale=scale), str(ck / "model.safetensors"))
    cfg = types.SimpleNamespace(PATH_TO_RAW_FACE={"D": str(face)}, PATH_TO_FEATURES={"D": str(tmp_path / "feat")},
                                PATH_TO_PRETRAINED_MODELS=str(tmp_path / "models"))
    for level in ("UTTERANCE", "FRAME"):
        params = V.build_parser().parse_args(["--dataset", "D", "--model_name", V.EVACLIP_VIT, "--feature_level",
                                              level, "--gpu", "0"])
        V.main(params, config=cfg)
        out = tmp_path / "feat" / f"eva02_base_patch14_224-{level[:3]}"
        assert sorted(os.listdir(out)) == sorted(f"{v}.npy" for v in G.CLIPS)
        for vid in G.CLIPS:
            got, ref = np.load(out / f"{vid}.npy"), GOLDEN[f"feat/default/{level}/{vid}"]
            assert got.shape == ref.shape and np.abs(got - ref).max() <= 1e-3 * np.abs(ref).max(), (level, vid)


def _forward(enc, m, frames, ws_bytes=None):
    n, h, w, _ = frames.shape
    ws = torch.empty(16, dtype=torch.uint8, device=enc.device)
    out = torch.empty(n, 768, device=enc.device)
    rc = enc._fwd(C.byref(m), L.ptr(frames), n, h, w, 0, 0, L.ptr(ws), ws_bytes or (1 << 40), L.ptr(out), None,
                  L.stream_ptr())
    return rc, L.last_error() if rc else ""


def test_malformed_eva02_models_are_refused_before_any_launch(cuda):
    enc = encoder("default", cuda)
    frames = torch.zeros(2, 224, 224, 3, dtype=torch.uint8, device=cuda)
    norms0 = (E.MerNormWeights * enc.n_layers)(*[E.MerNormWeights(enc.ffn_norms[i].g, None)
                                                 for i in range(enc.n_layers)])
    cases = [("rope_cos", None, "rope"), ("rope_sin", None, "rope"), ("ffn_norms", None, "FFN norms"),
             ("post_ln_g", None, "fc_norm"), ("rope_rows", 255, "rope table"), ("heads", 11, "unsupported dims"),
             ("gemm_mode", L.MER_GEMM_BF16X3, "gemm_mode"), ("ffn", 2730, "unsupported dims"),
             ("ffn", 2432, "FFN width"), ("ffn_norms", C.cast(norms0, C.POINTER(E.MerNormWeights)), "FFN norm 0"),
             ("pre_ln_g", enc.model.post_ln_g, "operands")]
    for field, value, text in cases:
        m = E.MerClipVisionModel.from_buffer_copy(enc.model)
        setattr(m, field, value)
        n0 = _launches()
        rc, msg = _forward(enc, m, frames)
        assert rc and text in msg, (field, msg)
        assert _launches() == n0, field
