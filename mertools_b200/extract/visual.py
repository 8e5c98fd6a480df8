"""Frame-level visual feature extraction — H100 mirror of
MERBench/feature_extraction/visual/extract_vision_huggingface.py.

Same CLI flags (:67-72), same ``config.py`` keys, same output naming
``PATH_TO_FEATURES[dataset]/<model>-<UTT|FRA>/<vid>.npy`` (:79-80,175-189) and the same helper
names.  The per-clip python loop of the reference (:104-171, one clip per forward, CPU
preprocessing) becomes: stage uint8 BGR frames of MANY clips in pinned memory, one H2D copy, one
fused device forward (preprocess + ViT + token-sum) through libmer_b200.so, one D2H copy.
"""
from __future__ import annotations

import argparse
import math
import os

import numpy as np
import torch

from ..encoders import VitEncoder
from . import common

DINO2_LARGE = "dinov2-large"
DINO2_GIANT = "dinov2-giant"
DATA2VEC_VISUAL = "data2vec-vision-base-ft1k"
VIDEOMAE_BASE = "videomae-base"
VIDEOMAE_LARGE = "videomae-large"
EVACLIP_VIT = "eva02_base_patch14_224.mim_in22k"


def func_read_frames(face_dir, vid):
    npy_path = os.path.join(face_dir, vid, f"{vid}.npy")
    assert os.path.exists(npy_path), f"Error: {vid} does not have frames.npy!"
    return np.load(npy_path)


def resample_frames_uniform(frames, nframe=16):
    """Uniformly sample ``nframe`` frames (reference :44-56).  Indices are floor(i * vlen / m)
    for i < m = min(nframe, vlen), padded with the last index — computed with the same float64
    product the reference's ``np.arange(0, vlen, vlen/m).astype(int)`` evaluates."""
    vlen = len(frames)
    m = min(nframe, vlen)
    step = vlen / m
    indices = [int(0 + i * step) for i in range(m)]
    indices += [indices[-1]] * (nframe - len(indices))
    return frames[indices[:nframe]]


def select_frame_indices(vlen, n_frms=8, readtype="uniform", rng=np.random):
    """The frame indices ``load_video_from_npy`` reads (MERBench/toolkit/utils/functions.py:81-104), bit for bit:
    ``all``, ``uniform`` (the rule of resample_frames_uniform), ``continuous`` and ``continuous_polish`` (one
    ``rng.randint`` call each, so a seeded ``np.random`` gives the reference's draw), then padding with the last index /
    truncation to ``n_frms`` (skipped when n_frms == 0)."""
    start, end = 0, vlen
    if readtype == "all":
        indices = np.arange(start, end, 1).astype(int).tolist()
    elif readtype == "uniform":
        m = min(n_frms, vlen)
        indices = np.arange(start, end, vlen / m).astype(int).tolist()
    elif readtype == "continuous":
        ii = rng.randint(start, max(start + 1, end - n_frms))
        indices = np.arange(ii, min(end, ii + n_frms)).astype(int).tolist()
    elif readtype == "continuous_polish":
        start += 25
        end -= 25
        ii = rng.randint(start, max(start + 1, end - n_frms * 4))
        indices = np.linspace(ii, min(end, ii + n_frms * 4), n_frms).astype(int).tolist()
    else:
        raise ValueError(f"readtype {readtype!r}")
    if n_frms != 0:
        while len(indices) < n_frms:
            indices.append(indices[-1])
        indices = indices[:n_frms]
    return indices


def load_video_from_npy(frames, n_frms=8, height=224, width=224, readtype="uniform", return_raw=False, device="cuda",
                        rng=np.random):
    """Mirror of ``load_video_from_npy`` (functions.py:79-118) for a clip already in memory (uint8 [vlen, H, W, 3] BGR,
    what ``func_video_to_face`` returns): index selection on the host, then on the device the selected frames through
    the bit-exact ``cv2.resize`` kernel (mer_resize_cv2_linear_u8) and BGR -> RGB.  Returns float [3, T, H, W] (CUDA)
    or, with ``return_raw``, uint8 [T, H, W, 3] RGB."""
    import ctypes as C

    from .. import _lib as L
    frames = np.asarray(frames)
    idx = select_frame_indices(len(frames), n_frms, readtype, rng)
    sel = torch.from_numpy(np.ascontiguousarray(frames[idx])).to(device)
    n, h, w, _ = sel.shape
    if (h, w) != (height, width):
        out = torch.empty(n, height, width, 3, dtype=torch.uint8, device=sel.device)
        fn = L.declare("mer_resize_cv2_linear_u8", [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                    C.c_void_p])
        L.check(fn(L.ptr(sel), n, h, w, L.ptr(out), height, width, L.stream_ptr()))
        sel = out
    rgb = sel.flip(-1)                       # func_opencv_to_decord
    return rgb if return_raw else rgb.permute(3, 0, 1, 2).float()


def split_into_batch(inputs, bsize=32):
    return [inputs[i * bsize:(i + 1) * bsize] for i in range(math.ceil(len(inputs) / bsize))]


class VisualExtractor:
    """ViT frame encoder + readout over batches of clips."""

    def __init__(self, state_dict, device="cuda", max_frames_per_launch=2048):
        # the CLIP checkpoints of the reference's model list carry a `vision_model.` tower + projection
        if "layer1.0.conv1.weight" in state_dict:  # torchvision resnet18 (the ImageNet CNN extractor)
            from ..encoders import ResNet18Encoder
            self.enc = ResNet18Encoder(state_dict, device=device)
            self.feature_dim = 512
        elif any(k.startswith("vision_model.") for k in state_dict):
            from ..encoders import ClipVisionEncoder
            self.enc = ClipVisionEncoder(state_dict, device=device)
            self.feature_dim = self.enc.proj_dim
        elif "encoder.layer.0.lambda_1" in state_dict:  # HF Data2VecVisionModel (data2vec-vision-base-ft1k; :124-133)
            from .data2vec_vision import Data2VecVisionEncoder
            self.enc = Data2VecVisionEncoder(state_dict, device=device)
            self.feature_dim = self.enc.hidden
        elif "encoder.layer.0.mlp.weights_in.weight" in state_dict:  # Dinov2Model with the SwiGLU MLP (dinov2-giant)
            from .dinov2_giant import Dinov2GiantEncoder
            self.enc = Dinov2GiantEncoder(state_dict, device=device)
            self.feature_dim = self.enc.hidden
        elif "blocks.0.mlp.fc1_g.weight" in state_dict:  # timm Eva (eva02_base_patch14_224; :127-131, 202-210)
            from ..encoders import Eva02Encoder
            self.enc = Eva02Encoder(state_dict, device=device)
            self.feature_dim = self.enc.hidden
        elif "encoder.layer.0.layer_scale1.lambda1" in state_dict:  # HF Dinov2Model (dinov2-large; :135-145)
            from ..encoders import Dinov2Encoder
            self.enc = Dinov2Encoder(state_dict, device=device)
            self.feature_dim = self.enc.hidden
        else:
            self.enc = VitEncoder(state_dict, device=device)
            self.feature_dim = 768
        self.device = self.enc.device
        self.max_frames = max_frames_per_launch
        self._pinned = None

    def _stage(self, frame_list, hw):
        n = sum(len(f) for f in frame_list)
        numel = n * hw[0] * hw[1] * 3
        if self._pinned is None or self._pinned.numel() < numel:
            self._pinned = torch.empty(numel, dtype=torch.uint8, pin_memory=True)
        host = self._pinned[:numel].view(n, hw[0], hw[1], 3)
        o = 0
        for f in frame_list:
            host[o:o + len(f)] = torch.from_numpy(np.ascontiguousarray(f))
            o += len(f)
        return host

    def _frame_features_same_size(self, frame_list, hw):
        host = self._stage(frame_list, hw)
        # frames smaller than 224x224 cost less to move: size the launches by their resized footprint
        outs = []
        for s in range(0, len(host), self.max_frames):
            dev = host[s:s + self.max_frames].to(self.device, non_blocking=True)
            outs.append(self.enc.frame_features(dev))  # resizes to 224x224 on the device when needed
        return torch.cat(outs).cpu().numpy()

    def frame_features(self, frame_list):
        """list of [n_i,H_i,W_i,3] uint8 (BGR) -> list of [n_i,768] float32 numpy.  Clips of the same frame
        size share one H2D copy and one launch sequence; any size other than 224x224 is resized on the
        device exactly as the HF processor does (PIL bilinear on uint8)."""
        frame_list = [np.asarray(f) for f in frame_list]
        for f in frame_list:
            assert f.dtype == np.uint8 and f.ndim == 4 and f.shape[-1] == 3, \
                f"frames must be uint8 [n,H,W,3] BGR, got {f.dtype} {f.shape}"
        res = [None] * len(frame_list)
        by_size = {}
        for i, f in enumerate(frame_list):
            if len(f) == 0:
                res[i] = np.zeros((0, self.feature_dim), np.float32)
            else:
                by_size.setdefault(f.shape[1:3], []).append(i)
        for hw, idxs in by_size.items():
            feats = self._frame_features_same_size([frame_list[i] for i in idxs], hw)
            o = 0
            for i in idxs:
                n = len(frame_list[i])
                res[i] = feats[o:o + n]
                o += n
        return res

    def extract_clips(self, clips, feature_level="UTTERANCE", nframe=None, save_files=None):
        """clips: list of uint8 [vlen,H,W,3] BGR arrays (any H, W; the reference's OpenFace crops).  ``nframe`` resamples every clip
        first (64 in the reference's DINOv2 branch :136, None in the data2vec branch)."""
        if nframe is not None:
            clips = [resample_frames_uniform(np.asarray(c), nframe) for c in clips]
        feats = self.frame_features(clips)
        out = []
        for i, f in enumerate(feats):
            sf = save_files[i] if save_files is not None else None
            out.append(common.save_feature(sf, f.squeeze(), feature_level, self.feature_dim))
        return out


def main(params, config=None, clips_per_launch=32):
    """Reproduces the script body (:74-189) for the HF ViT branches."""
    if config is None:
        from .. import config as config  # noqa: PLW0127
    print(f"==> Extracting {params.model_name} embeddings...")
    model_name = params.model_name.split(".")[0]
    face_dir = config.PATH_TO_RAW_FACE[params.dataset]
    save_dir = os.path.join(config.PATH_TO_FEATURES[params.dataset],
                            f"{model_name}-{params.feature_level[:3]}")
    os.makedirs(save_dir, exist_ok=True)
    model_dir = os.path.join(config.PATH_TO_PRETRAINED_MODELS, f"transformers/{params.model_name}")
    assert params.gpu != -1, "mertools_b200 has no CPU path (reference: --gpu=-1 means CPU)"
    from .. import shard
    params.gpu = shard.device_index(params.gpu)
    torch.cuda.set_device(params.gpu)
    if params.model_name in (VIDEOMAE_BASE, VIDEOMAE_LARGE):                    # :147-159: 16 frames -> 8 tubelet rows
        from .videomae import VideoMaeExtractor
        ext = VideoMaeExtractor.from_pretrained(model_dir, device=f"cuda:{params.gpu}")
    elif params.model_name == EVACLIP_VIT:
        ext = VisualExtractor(load_timm_state_dict(timm_checkpoint_path(config, params.model_name)),
                              device=f"cuda:{params.gpu}")
    else:
        ext = VisualExtractor(common.load_hf_state_dict(model_dir), device=f"cuda:{params.gpu}")
        if params.model_name == DATA2VEC_VISUAL:   # processor settings from the checkpoint's preprocessor_config.json
            from .data2vec_vision import Data2VecVisionEncoder
            ext.enc = Data2VecVisionEncoder.from_pretrained(model_dir, device=f"cuda:{params.gpu}")
    nframe = 64 if params.model_name in (DINO2_LARGE, DINO2_GIANT) else None
    vids = os.listdir(face_dir)
    print(f'Find total "{len(vids)}" videos.')
    # one process per GPU under torchrun: this rank's share of the videos that do not have their .npy yet
    vids, rank, world = shard.my_work(vids, lambda vid: os.path.join(save_dir, f"{vid}.npy"))
    if world > 1:
        print(f"rank {rank}/{world}: {len(vids)} videos on cuda:{params.gpu}")
    for s in range(0, len(vids), clips_per_launch):
        chunk = vids[s:s + clips_per_launch]
        clips = [func_read_frames(face_dir, vid) for vid in chunk]
        files = [os.path.join(save_dir, f"{vid}.npy") for vid in chunk]
        ext.extract_clips(clips, params.feature_level, nframe=nframe, save_files=files)
        print(f"Processed {min(s + clips_per_launch, len(vids))}/{len(vids)} videos")


def timm_checkpoint_path(config, model_name):
    """The reference's timm weights file (:128): PATH_TO_PRETRAINED_MODELS/timm/<model_name>/model.safetensors."""
    return os.path.join(config.PATH_TO_PRETRAINED_MODELS, f"timm/{model_name}/model.safetensors")


def load_timm_state_dict(path):
    from safetensors.torch import load_file
    return load_file(path)


def build_parser():
    parser = argparse.ArgumentParser(description="Run.")
    parser.add_argument("--dataset", type=str, default="MER2023", help="input dataset")
    parser.add_argument("--model_name", type=str, default=None, help="name of pretrained model")
    parser.add_argument("--feature_level", type=str, default="UTTERANCE", help="feature level [FRAME or UTTERANCE]")
    parser.add_argument("--gpu", type=int, default=0, help="gpu id")
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
