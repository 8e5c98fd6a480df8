"""VideoMAE face-clip features of MER2024 / MER2026 (``feature_extraction/visual/extract_sun_videomae.py``: the vendored
``videomae`` package's tubelet ViT, e.g. the ``videomae-base-VoxCeleb2-99`` features of the MER2024 baselines).

Per video (``<face_dir>/<vid>/<vid>.npy``, uint8 [n, H, W, 3] read as RGB) the reference runs four views of 16 frames
(``videomae/kinetics.py:VideoClsDatasetFrame``, 2 temporal segments x 2 spatial crops) through the model and averages
them in float64 (``engine_for_finetuning.py:final_test``).  UTTERANCE runs one set of four views per video, FRAME one
per frame.  Most of those views are the same 16 frames: both crops are the whole square image, the two UTTERANCE
segments coincide for clips of up to 64 frames (sampling rate 4), and every FRAME view of a frame is one window, shared
by the first 10 frames and by the last 9.  This extractor runs each distinct view once per video, packs the views of
many videos into one ``mer_videomae_forward`` launch, and puts the duplicates back before the reference's ``np.mean``,
so that the float64 result is what four separate forwards of the same values give.
"""
from __future__ import annotations

import argparse
import ctypes as C
import glob
import os

import numpy as np
import torch

from .. import _lib as L
from .. import weights as W
from .videomae import sinusoid_table

CLIP_LEN = 16
TEST_NUM_SEGMENT = TEST_NUM_CROP = 2
KPATCH = 3 * 2 * 16 * 16
EPS = 1e-6
# modeling_finetune.py:1585 / 1649 / 1666 (qkv_bias=True, LayerNorm eps 1e-6, mlp_ratio 4)
MODELS = {
    "vit_base_patch16_160": dict(img=160, dim=768, depth=12, heads=12),
    "vit_base_patch16_224": dict(img=224, dim=768, depth=12, heads=12),
    "vit_large_patch16_224": dict(img=224, dim=1024, depth=24, heads=16),
}


# ---- view planning (kinetics.py:VideoClsDatasetFrame, mode 'test') ----
def _row(idx, n):
    """``frames[min(idx, n - 1)]`` as numpy resolves it: a negative index counts from the end."""
    i = min(idx, n - 1)
    return i + n if i < 0 else i


def _pad(idxs):
    while len(idxs) < CLIP_LEN:
        idxs.append(idxs[-1])
    return idxs


def frame_window(f, n):
    """Source indices of the FRAME-level clip of frame f (kinetics.py:77-86)."""
    if f < 10:
        start, end = 0, 16
    elif f > n - 10:
        start, end = n - 17, n - 1
    else:
        start, end = f - 8, f + 8
    return _pad(list(range(start, end)))


def plan_views(n, feature_level, sampling_rate=4):
    """The dataset's items in order: a list of (frame id, 16 resolved frame rows), four per frame id (segment-major,
    crop-minor).  UTTERANCE: frame id 0; FRAME: ids 0 .. n - 1."""
    if n <= 0:
        raise ValueError("a video of 0 frames has no clip (the reference fails on it)")
    if feature_level == "UTTERANCE":
        idxs = _pad(list(range(0, n, sampling_rate)))
        groups = [(0, idxs)]
    elif feature_level == "FRAME":
        groups = [(f, frame_window(f, n)) for f in range(n)]
    else:
        raise ValueError(f"feature_level {feature_level!r} (UTTERANCE or FRAME)")
    # test_seg order: segment ck, crop cp, then frame id.  The buffer is square after the resize, so spatial_step = 0
    # and both crops are the whole image; the segment starts at int(ck * temporal_step).
    out = []
    for ck in range(TEST_NUM_SEGMENT):
        for _cp in range(TEST_NUM_CROP):
            for fid, idxs in groups:
                s = int(ck * max(1.0 * (len(idxs) - CLIP_LEN) / (TEST_NUM_SEGMENT - 1), 0))
                out.append((fid, tuple(_row(i, n) for i in idxs[s:s + CLIP_LEN])))
    return out


def readout(items, feats, feature_level):
    """``final_test`` (engine_for_finetuning.py:6-46) over the dataset's items: ``items`` [(frame id, rows)] in
    order, ``feats`` {rows: fp32 [D] feature}.  Returns the float64 array the reference saves."""
    saved = {}
    for fid, rows in items:
        saved.setdefault("%010d" % fid, []).append(np.asarray(feats[rows], np.float32).tolist())
    emb = []
    for key in sorted(saved):
        block = saved[key]
        assert len(block) == 4
        emb.append(np.mean(block, axis=0))
    emb = np.array(emb).squeeze()
    if feature_level == "FRAME":
        return emb[np.newaxis, :] if emb.ndim == 1 else emb
    return np.mean(emb, axis=0) if emb.ndim == 2 else emb


# ---- checkpoint (extract_sun_videomae.py:296-323, utils.load_state_dict) ----
def _expected(model, n_layers):
    """Every parameter the model's forward reads: name -> (shape, default or None when the init is random)."""
    cfg = MODELS[model]
    D, F = cfg["dim"], 4 * cfg["dim"]
    one, zero = (lambda s: np.ones(s, np.float32)), (lambda s: np.zeros(s, np.float32))
    exp = {"patch_embed.proj.weight": ((D, 3, 2, 16, 16), None), "patch_embed.proj.bias": ((D,), None)}
    for i in range(n_layers):
        p = f"blocks.{i}."
        exp.update({
            p + "norm1.weight": ((D,), one), p + "norm1.bias": ((D,), zero),
            p + "attn.qkv.weight": ((3 * D, D), None),
            p + "attn.q_bias": ((D,), zero), p + "attn.v_bias": ((D,), zero),
            p + "attn.proj.weight": ((D, D), None), p + "attn.proj.bias": ((D,), zero),
            p + "norm2.weight": ((D,), one), p + "norm2.bias": ((D,), zero),
            p + "mlp.fc1.weight": ((F, D), None), p + "mlp.fc1.bias": ((F,), zero),
            p + "mlp.fc2.weight": ((D, F), None), p + "mlp.fc2.bias": ((D,), zero),
        })
    exp.update({"norm.weight": ((D,), one), "norm.bias": ((D,), zero)})
    return exp


def model_state_dict(checkpoint, model="vit_base_patch16_224", model_key="model|module", n_layers=None):
    """The parameters the reference's ``VisionTransformer`` ends up with after its non-strict load, as float32 numpy
    arrays: ``checkpoint[model_key]`` (first key present, else the checkpoint itself), ``backbone.`` / ``encoder.``
    prefixes stripped, keys the forward does not read ignored (decoder, mask_token, gamma_*, head, ...), LayerNorm 1 / 0
    and zero biases where the checkpoint has none.  Refused (ValueError): a missing weight whose init is random (the
    patch Conv3d, any Linear weight) and any shape that does not fit ``model``, which the reference would run with
    random weights."""
    if model not in MODELS:
        raise ValueError(f"model {model!r}: one of {sorted(MODELS)}")
    n_layers = MODELS[model]["depth"] if n_layers is None else n_layers
    cm = None
    for k in model_key.split("|"):
        if k in checkpoint:
            cm = checkpoint[k]
            break
    if cm is None:
        cm = checkpoint
    sd = {}
    for k, v in cm.items():
        if k.startswith("backbone."):
            k = k[9:]
        elif k.startswith("encoder."):
            k = k[8:]
        sd[k] = v
    out, missing, bad = {}, [], []
    for k, (shape, default) in _expected(model, n_layers).items():
        if k not in sd:
            if default is None:
                missing.append(k)
            else:
                out[k] = default(shape)
            continue
        v = sd[k]
        v = v.detach().cpu().float().numpy() if isinstance(v, torch.Tensor) else np.asarray(v, np.float32)
        if tuple(v.shape) != shape:
            bad.append(f"{k} {tuple(v.shape)} != {shape}")
        out[k] = np.ascontiguousarray(v, np.float32)
    if missing or bad:
        raise ValueError(f"checkpoint does not fit {model} ({n_layers} layers): "
                         + "; ".join(([f"missing {missing}"] if missing else []) + bad))
    return out


def load_checkpoint(path, model="vit_base_patch16_224", model_key="model|module", n_layers=None):
    """``torch.load`` with ``weights_only=True`` (tensors and plain containers; ``argparse.Namespace`` for the
    ``args`` entry of training checkpoints), then ``model_state_dict``."""
    with torch.serialization.safe_globals([argparse.Namespace]):
        ckpt = torch.load(path, map_location="cpu", weights_only=True)
    return model_state_dict(ckpt, model, model_key, n_layers)


_NAMES = dict(
    ln1_g="blocks.{i}.norm1.weight", ln1_b="blocks.{i}.norm1.bias",
    q_w="blocks.{i}.q_w", k_w="blocks.{i}.k_w", v_w="blocks.{i}.v_w",
    q_b="blocks.{i}.attn.q_bias", k_b="blocks.{i}.k_b", v_b="blocks.{i}.attn.v_bias",
    o_w="blocks.{i}.attn.proj.weight", o_b="blocks.{i}.attn.proj.bias",
    ln2_g="blocks.{i}.norm2.weight", ln2_b="blocks.{i}.norm2.bias",
    fc1_w="blocks.{i}.mlp.fc1.weight", fc1_b="blocks.{i}.mlp.fc1.bias",
    fc2_w="blocks.{i}.mlp.fc2.weight", fc2_b="blocks.{i}.mlp.fc2.bias",
)


class MerVideoMaeModel(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("dim", C.c_int), ("heads", C.c_int), ("ffn", C.c_int), ("img", C.c_int),
                ("ln_eps", C.c_float), ("patch_w", C.c_void_p), ("patch_b", C.c_void_p), ("pos", C.c_void_p),
                ("layers", C.POINTER(W.MerLayerWeights)), ("norm_g", C.c_void_p), ("norm_b", C.c_void_p)]


def _declare():
    lib = L.lib()
    lib.mer_videomae_workspace_bytes.restype = C.c_longlong
    lib.mer_videomae_workspace_bytes.argtypes = [C.POINTER(MerVideoMaeModel), C.c_int]
    lib.mer_resize_workspace_bytes.restype = C.c_longlong
    lib.mer_resize_workspace_bytes.argtypes = [C.c_int] * 5
    fwd = L.declare("mer_videomae_forward", [C.POINTER(MerVideoMaeModel), C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                             C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p])
    resize = L.declare("mer_resize_bilinear_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                  C.c_void_p, C.c_void_p])
    return fwd, resize


def resize_frames(frames, S, device, _fn=None):
    """uint8 [n, H, W, 3] (host or device) -> [n, S, S, 3] on the device: PIL bilinear to S x S, aspect ignored
    (video_transforms.Resize((S, S), 'bilinear'))."""
    f = torch.as_tensor(np.ascontiguousarray(frames) if isinstance(frames, np.ndarray) else frames)
    if f.dim() != 4 or f.shape[-1] != 3 or f.dtype != torch.uint8:
        raise ValueError(f"frames must be uint8 [n, H, W, 3], got {tuple(f.shape)} {f.dtype}")
    f = f.to(device).contiguous()
    n, h, w, _ = f.shape
    if (h, w) == (S, S):
        return f
    fn = _fn if _fn is not None else _declare()[1]
    out = torch.empty(n, S, S, 3, dtype=torch.uint8, device=device)
    ws = torch.empty(max(int(L.lib().mer_resize_workspace_bytes(n, h, w, S, S)), 1), dtype=torch.uint8, device=device)
    L.check(fn(L.ptr(f), n, h, w, L.ptr(out), S, S, L.ptr(ws), L.stream_ptr()))
    return out


def videomae_clips(frames, view_rows, S, out_f32=False):
    """``mer_videomae_clips`` on CUDA tensors: frames uint8 [n, S, S, 3], view_rows int32 [n_views, 16] -> the patch
    operand [n_views * 8 (S / 16)^2, 1536] (fp16, or fp32 with ``out_f32``)."""
    f = L.declare("mer_videomae_clips", [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                         C.c_void_p])
    nv = view_rows.shape[0]
    out = torch.empty(nv * 8 * (S // 16) ** 2, KPATCH, dtype=torch.float32 if out_f32 else torch.float16,
                      device=frames.device)
    L.check(f(L.ptr(frames), frames.shape[0], S, L.ptr(view_rows), nv, L.ptr(out), 1 if out_f32 else 0, L.stream_ptr()))
    return out


class SunVideoMae:
    """The reference model on the device: ``forward_views`` runs views, ``extract_videos`` whole videos."""

    def __init__(self, state_dict, model="vit_base_patch16_224", device="cuda", views_per_launch=64):
        cfg = MODELS[model]
        self.model, self.img, self.dim = model, cfg["img"], cfg["dim"]
        self.device = torch.device(device)
        if self.device.index is not None:
            torch.cuda.set_device(self.device)
        self.views_per_launch = int(views_per_launch)
        if self.views_per_launch < 1:
            raise ValueError(f"views per launch {views_per_launch}")
        sd = state_dict
        D = self.dim
        n_layers = W.count_layers(sd, "blocks.{i}.attn.qkv.weight")
        zeros = np.zeros(D, np.float32)
        pack_sd = dict(sd)
        for i in range(n_layers):
            qkv = sd[f"blocks.{i}.attn.qkv.weight"]
            pack_sd[f"blocks.{i}.q_w"], pack_sd[f"blocks.{i}.k_w"], pack_sd[f"blocks.{i}.v_w"] = qkv[:D], qkv[D:2 * D], qkv[2 * D:]
            pack_sd[f"blocks.{i}.k_b"] = zeros
        pk = self.pk = W.Packed(self.device)
        self._layers = W.pack_layers(pack_sd, _NAMES, n_layers, pk, f16=True)
        g = self.img // 16
        self.tokens = 8 * g * g
        m = self.m = MerVideoMaeModel()
        m.n_layers, m.dim, m.heads, m.ffn, m.img, m.ln_eps = n_layers, D, cfg["heads"], 4 * D, self.img, EPS
        m.patch_w = pk.keep(sd["patch_embed.proj.weight"].reshape(D, -1), f16=True).data_ptr()
        m.patch_b = pk.keep(sd["patch_embed.proj.bias"]).data_ptr()
        m.pos = pk.keep(sinusoid_table(self.tokens, D)).data_ptr()
        m.layers = C.cast(self._layers, C.POINTER(W.MerLayerWeights))
        m.norm_g, m.norm_b = pk.keep(sd["norm.weight"]).data_ptr(), pk.keep(sd["norm.bias"]).data_ptr()
        self._fwd, self._resize = _declare()
        self._ws = None

    def workspace_bytes(self, n_views):
        b = int(L.lib().mer_videomae_workspace_bytes(C.byref(self.m), n_views))
        if b < 0:
            raise L.MerError(L.last_error())
        return b

    def resize(self, frames):
        return resize_frames(frames, self.img, self.device, self._resize)

    def forward_views(self, frames, view_rows):
        """frames: uint8 CUDA [n, S, S, 3]; view_rows: int [n_views, 16] (host) -> fp32 CUDA [n_views, D]."""
        rows = np.ascontiguousarray(np.asarray(view_rows, np.int32).reshape(-1, CLIP_LEN))
        nv = rows.shape[0]
        need = self.workspace_bytes(nv)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        out = torch.empty(nv, self.dim, dtype=torch.float32, device=self.device)
        L.check(self._fwd(C.byref(self.m), L.ptr(frames), frames.shape[0], rows.ctypes.data_as(C.c_void_p), nv,
                          L.ptr(self._ws), self._ws.numel(), L.ptr(out), L.stream_ptr()))
        return out

    def extract_videos(self, videos, feature_level="UTTERANCE", sampling_rate=4, save_files=None):
        """videos: uint8 [n, H, W, 3] arrays (the face .npy files).  Returns the arrays the reference saves (float64;
        FRAME [n, D], UTTERANCE [D]), and writes them to ``save_files`` when given."""
        plans = [plan_views(len(v), feature_level, sampling_rate) for v in videos]
        distinct = [list(dict.fromkeys(rows for _, rows in p)) for p in plans]
        results = [None] * len(videos)
        b = 0
        while b < len(videos):
            # videos whose distinct views fill a launch: their frames go up once, their views run in launches of
            # views_per_launch
            e, nv = b, 0
            while e < len(videos) and (e == b or nv + len(distinct[e]) <= self.views_per_launch):
                nv += len(distinct[e])
                e += 1
            frames = [self.resize(videos[i]) for i in range(b, e)]
            base = np.cumsum([0] + [f.shape[0] for f in frames])
            allf = torch.cat(frames) if len(frames) > 1 else frames[0]
            keys = [(i, rows) for i in range(b, e) for rows in distinct[i]]
            table = np.array([[base[i - b] + r for r in rows] for i, rows in keys], np.int32)
            feats = torch.cat([self.forward_views(allf, table[s:s + self.views_per_launch])
                               for s in range(0, len(keys), self.views_per_launch)]).cpu().numpy()
            for i in range(b, e):
                got = {rows: feats[k] for k, (j, rows) in enumerate(keys) if j == i}
                results[i] = readout(plans[i], got, feature_level)
            b = e
        if save_files is not None:
            for path, r in zip(save_files, results):
                np.save(path, r)
        return results


# ---- CLI (extract_sun_videomae.py:22-221, 224-359) ----
def build_parser():
    """The reference's flags that change what is computed.  Every other flag of the reference (optimiser, mixup,
    dropout, ...) is accepted and has no effect on evaluation."""
    p = argparse.ArgumentParser("VideoMAE face-clip features (MER2024 extract_sun_videomae.py)")
    p.add_argument("--batch_size", default=64, type=int, help="distinct views per device launch")
    p.add_argument("--dataset", default="MER2023", type=str)
    p.add_argument("--feature_level", default="UTTERANCE", type=str)
    p.add_argument("--debug", action="store_true", default=False)
    p.add_argument("--model", default="vit_base_patch16_224", type=str)
    p.add_argument("--tubelet_size", type=int, default=2)
    p.add_argument("--input_size", default=224, type=int)
    p.add_argument("--attn_type", default="joint", type=str)
    p.add_argument("--short_side_size", type=int, default=224)
    p.add_argument("--test_num_segment", type=int, default=2)
    p.add_argument("--test_num_crop", type=int, default=2)
    p.add_argument("--finetune", default="")
    p.add_argument("--model_key", default="model|module", type=str)
    p.add_argument("--use_mean_pooling", action="store_true")
    p.set_defaults(use_mean_pooling=False)
    p.add_argument("--num_segments", type=int, default=1)
    p.add_argument("--num_frames", type=int, default=16)
    p.add_argument("--sampling_rate", type=int, default=4)
    p.add_argument("--device", default="cuda")
    return p


def parse_args(argv=None):
    args, _ = build_parser().parse_known_args(argv)
    return args


def check_args(args):
    """ValueError for a configuration this extractor does not run (before any file is read)."""
    if args.model not in MODELS:
        raise ValueError(f"--model {args.model}: one of {sorted(MODELS)}")
    fixed = [("--attn_type", args.attn_type, "joint"), ("--num_frames", args.num_frames, 16),
             ("--tubelet_size", args.tubelet_size, 2), ("--num_segments", args.num_segments, 1),
             ("--test_num_segment", args.test_num_segment, TEST_NUM_SEGMENT),
             ("--test_num_crop", args.test_num_crop, TEST_NUM_CROP)]
    for flag, got, want in fixed:
        if got != want:
            raise ValueError(f"{flag} {got}: only {want} is supported")
    if args.use_mean_pooling:
        raise ValueError("--use_mean_pooling: only the final-norm + token-mean feature (the default) is supported")
    img = MODELS[args.model]["img"]
    if args.short_side_size != args.input_size or args.input_size != img:
        raise ValueError(f"--input_size {args.input_size} / --short_side_size {args.short_side_size}: {args.model} "
                         f"takes {img} x {img} clips (the reference fails PatchEmbed's size assert otherwise)")
    if args.feature_level not in ("UTTERANCE", "FRAME"):
        raise ValueError(f"--feature_level {args.feature_level}: UTTERANCE or FRAME")
    if args.batch_size < 1 or args.sampling_rate < 1:
        raise ValueError(f"--batch_size {args.batch_size} / --sampling_rate {args.sampling_rate} must be positive")
    if not args.finetune:
        raise ValueError("--finetune: a checkpoint is required (the reference would run randomly initialised weights)")
    if not str(args.device).startswith("cuda"):
        raise ValueError(f"--device {args.device}: mertools_b200 runs on a CUDA device")


def save_dir_name(finetune, feature_level):
    """``.../videomae-base-VoxCeleb2/checkpoint-99.pth`` -> ``videomae-base-VoxCeleb2-99-UTT`` (:232-235)."""
    model_name, epoch_name = finetune.split("/")[-2:]
    epoch_name = epoch_name[:-4].split("-")[1]
    return f"{model_name}-{epoch_name}-{feature_level[:3]}"


def main(args, config=None):
    if config is None:
        from .. import config as config  # noqa: PLW0127
    from .. import shard
    check_args(args)
    face_dir = config.PATH_TO_RAW_FACE[args.dataset]
    save_dir = os.path.join(config.PATH_TO_FEATURES[args.dataset], save_dir_name(args.finetune, args.feature_level))
    os.makedirs(save_dir, exist_ok=True)
    sd = load_checkpoint(args.finetune, args.model, args.model_key)
    out_path = lambda f: os.path.join(save_dir, os.path.basename(f).rsplit(".", 1)[0] + ".npy")  # noqa: E731
    face_npys = glob.glob(face_dir + "/*/*.npy")
    if args.debug:
        face_npys = sorted(face_npys)[:10]
    todo, rank, world = shard.my_work(face_npys, out_path)
    print(f"process sample number: {len(todo)}" + (f" (rank {rank}/{world})" if world > 1 else ""))
    ext = SunVideoMae(sd, args.model, device=args.device, views_per_launch=args.batch_size)
    chunk = max(1, args.batch_size)
    for s in range(0, len(todo), chunk):
        files = todo[s:s + chunk]
        ext.extract_videos([np.load(f) for f in files], args.feature_level, args.sampling_rate,
                           save_files=[out_path(f) for f in files])


if __name__ == "__main__":
    main(parse_args())
