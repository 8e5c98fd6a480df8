"""FER+ CNN extractor: mirror of MERBench/feature_extraction/visual/extract_ferplus_embedding.py.

Same flags (``--dataset --feature_level --model_name --layer_name --gpu``, :130-136), input layout
(``<face_dir>/<vid>/<vid>.npy`` through FaceDataset, dataset.py:12-47), output directory
``<model prefix>face_<UTT|FRA>`` (:143-145) and save rules (:175-194).  Supported here: both models of the script
(``resnet50_ferplus_dag``, ``senet50_ferplus_dag``) with the default ``--layer_name conv5_3_3x3_relu`` (512-d); the preprocessing of
``compose_transforms`` (Resize(256), CenterCrop(224), ToTensor, x 255, Normalize) and the network run in
libmer_b200.so.  The checkpoint is the reference's ``<PRETRAINED>/ferplus/<model_name>.pth``.
"""
from __future__ import annotations

import argparse
import os

import numpy as np
import torch

from ..encoders import FerplusResnet50Encoder
from . import common
from .visual import func_read_frames

SUPPORTED = {"resnet50_ferplus_dag": "conv5_3_3x3_relu", "senet50_ferplus_dag": "conv5_3_3x3_relu"}


def extract_video(enc, frames_bgr, feature_level, save_file=None, frames_per_launch=64):
    """One video: uint8 [T, H, W, 3] BGR -> the array the reference saves (:170-194).  The reference sorts by the
    zero-padded frame index, which is the stored order."""
    frames = np.asarray(frames_bgr)
    if len(frames) == 0:
        print("Warning: number of frames of video should not be zero.")
        emb = np.zeros((0, enc.feature_dim), np.float32)
    else:
        dev = torch.from_numpy(np.ascontiguousarray(frames)).to(enc.device)
        emb = enc.frame_features(dev, max_frames=frames_per_launch).cpu().numpy()
    return common.save_feature(save_file, emb, feature_level, enc.feature_dim)


def main(params, config=None, state_dict=None):
    if config is None:
        from .. import config as config  # noqa: PLW0127
    assert params.model_name in SUPPORTED and params.layer_name == SUPPORTED[params.model_name], \
        f"the H100 path covers {SUPPORTED} (other hook layers: use the reference script)"
    print("==> Extracting ferplus embedding...")
    face_dir = config.PATH_TO_RAW_FACE[params.dataset]
    save_name = f"{params.model_name.split('_')[0]}face_{params.feature_level[:3]}"
    save_dir = os.path.join(config.PATH_TO_FEATURES[params.dataset], save_name)
    if not os.path.exists(save_dir):
        os.makedirs(save_dir)
    if state_dict is None:
        path = os.path.join(config.PATH_TO_PRETRAINED_MODELS, "ferplus", params.model_name + ".pth")
        state_dict = {k: v.float().numpy() if v.is_floating_point() else v.numpy()
                      for k, v in torch.load(path, map_location="cpu").items()}
    gpu = int(str(params.gpu).split(",")[0])
    enc = FerplusResnet50Encoder(state_dict, device=f"cuda:{gpu}")
    vids = os.listdir(face_dir)
    print(f'Find total "{len(vids)}" videos.')
    for i, vid in enumerate(vids, 1):
        print(f"Processing video '{vid}' ({i}/{len(vids)})...")
        extract_video(enc, func_read_frames(face_dir, vid), params.feature_level, os.path.join(save_dir, f"{vid}.npy"))


def build_parser():
    parser = argparse.ArgumentParser(description="Run.")
    parser.add_argument("--dataset", type=str, default=None, help="input dataset")
    parser.add_argument("--feature_level", type=str, default="UTTERANCE", help="feature level [FRAME or UTTERANCE]")
    parser.add_argument("--model_name", type=str, default=None, choices=["resnet50_ferplus_dag", "senet50_ferplus_dag"])
    parser.add_argument("--layer_name", type=str, default="conv5_3_3x3_relu", help="which layer used to extract feature")
    parser.add_argument("--gpu", type=str, default="0", help="gpu id")
    return parser


if __name__ == "__main__":
    main(build_parser().parse_args())
