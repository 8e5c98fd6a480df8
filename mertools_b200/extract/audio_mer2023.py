"""MER2023 audio features -- H100 mirror of MER2023/feature_extraction/audio/extract_transformers_embedding.py.

Keeps ``extract(model_name, audio_files, save_dir, feature_level, layer_ids=None, gpu=None)`` (:27) and the CLI
(:67-100).  Three things set it apart from MERBench's extract_audio_huggingface.py, which extract/audio.py mirrors:

* every clip goes through the model whole, as one row (:54-59): no 10 s split, so a 25 s clip is one row of 1,249
  frames.  Rows of more than 505 frames run attention on the fp16 V^T kernel (mer_b200.h, MER_ATT_LONG_MAX);
* the readout is ``torch.stack(hidden_states)[layer_ids].sum(0)`` (:60) with the CLI's ``layer_ids = [-1]`` (:88):
  ``hidden_states[-1]`` alone (MerHubertModel.readout), and ``feature[0].squeeze()`` is saved (:62);
* the model class comes from the name (:34-39): ``HubertModel`` for names containing "hubert", else
  ``Wav2Vec2Model`` for names containing "wav2vec".  Both run on the same encoder here (HubertEncoder).

Clips of any length share launches: the ragged pipelined path of ``AudioExtractor`` (pinned staging, clips sorted by
length, launches of at most ``max_samples_per_launch`` padded samples), so long clips do not pad short ones.
"""
from __future__ import annotations

import argparse
import glob
import os
import time

import numpy as np
import torch

from . import common
from .audio import MAXLEN, AudioExtractor

LAST = [-1]                   # the CLI's layer_ids (:88)
LAST_FOUR = [-4, -3, -2, -1]  # the MERBench readout, also accepted
SAMPLE_RATE = 16000


def model_class(model_name):
    """The HF class the reference loads for ``model_name`` (:34-39)."""
    if model_name.find("hubert") != -1:
        return "HubertModel"
    if model_name.find("wav2vec") != -1:
        return "Wav2Vec2Model"
    raise ValueError(f"model_name {model_name!r}: the MER2023 audio extractor loads HubertModel for names containing "
                     "'hubert' and Wav2Vec2Model for names containing 'wav2vec'; any other name leaves its model "
                     "unbound")


def last_layer_only(layer_ids):
    """True for ``[-1]`` (hidden_states[-1]), False for ``[-4, -3, -2, -1]``; anything else is refused."""
    if layer_ids is None:
        raise ValueError("layer_ids=None: the reference indexes torch.stack(hidden_states)[None], which keeps every "
                         "hidden state, and its `assert feature.shape[0] == 1` fails; pass [-1] (the CLI's value) or "
                         "[-4, -3, -2, -1]")
    ids = [int(i) for i in layer_ids]
    if ids == LAST:
        return True
    if ids == LAST_FOUR:
        return False
    raise ValueError(f"layer_ids {ids}: the device readouts are hidden_states[-1] ([-1]) and the sum of the last four "
                     "hidden states ([-4, -3, -2, -1])")


def save_dir_name(model_name, feature_level, layer_ids=LAST):
    """``{model}-{UTT|FRA}``, or ``{model}-{len(layer_ids)}-{UTT|FRA}`` for more than one layer (:96-98)."""
    name = model_name if len(layer_ids) == 1 else f"{model_name}-{len(layer_ids)}"
    return f"{name}-{feature_level[:3]}"


def prepare_save_dir(save_dir, overwrite):
    """Create ``save_dir``; an existing one is reused when ``overwrite`` is set or it is empty, else refused (:99-105)."""
    if not os.path.exists(save_dir):
        os.makedirs(save_dir)
    elif overwrite or len(os.listdir(save_dir)) == 0:
        print(f'==> Warning: overwrite save_dir "{save_dir}"!')
    else:
        raise FileExistsError(f'==> Error: save_dir "{save_dir}" already exists, set overwrite=TRUE if needed!')


class Mer2023AudioExtractor(AudioExtractor):
    """Whole clips of any length through HubertEncoder with the readout ``layer_ids`` selects."""

    def __init__(self, state_dict, layer_ids=LAST, device="cuda", do_normalize=True, max_rows_per_launch=128,
                 max_samples_per_launch=128 * MAXLEN // 2):
        super().__init__(state_dict, device=device, max_rows_per_launch=max_rows_per_launch, ragged=True,
                         max_samples_per_launch=max_samples_per_launch, do_normalize=do_normalize,
                         last_layer_only=last_layer_only(layer_ids))

    def extract_waves(self, waves, feature_level="UTTERANCE", save_files=None):
        """waves: list of 1-D float arrays (16 kHz mono).  Returns what the reference would ``np.save`` (:61-71):
        FRAME [T, D] (``[D]`` for a one-frame clip: ``feature[0].squeeze()``), UTTERANCE the mean over frames [D]."""
        for i, w in enumerate(waves):
            if np.ndim(w) != 1:
                raise ValueError(f"clip {i}: mono audio only (shape {np.shape(w)}); the reference's "
                                 "`assert feature.shape[0] == 1` fails on several channels")
        res = [None] * len(waves)
        self._extract_ragged(waves, list(range(len(waves))), feature_level, res)
        for i, r in enumerate(res):
            if r.ndim == 2 and r.shape[0] == 1:
                res[i] = r[0]
        if save_files is not None:
            for f, r in zip(save_files, res):
                np.save(f, r)
        return res


def extract(model_name, audio_files, save_dir, feature_level, layer_ids=None, gpu=None, config=None,
            clips_per_launch=128):
    """Same signature and on-disk result as the reference ``extract`` (:27-74)."""
    if config is None:
        from .. import config as config  # noqa: PLW0127
    from .. import shard
    start_time = time.time()
    model_class(model_name)
    last_layer_only(layer_ids)
    if gpu is None or gpu == -1:
        raise ValueError(f"gpu={gpu}: mertools_b200 runs on a CUDA device (the reference's gpu=-1 is its CPU path)")
    import soundfile as sf
    gpu = shard.device_index(gpu)
    torch.cuda.set_device(gpu)
    # one process per GPU under torchrun: this rank's share of the files that do not have their .npy yet
    audio_files, rank, world = shard.my_work(audio_files, lambda f: os.path.join(save_dir, os.path.basename(f)[:-4] + ".npy"))
    if world > 1:
        print(f"rank {rank}/{world}: {len(audio_files)} audio files on cuda:{gpu}")
    model_file = os.path.join(config.PATH_TO_PRETRAINED_MODELS, f"transformers/{model_name}")
    ext = Mer2023AudioExtractor(common.load_hf_state_dict(model_file), layer_ids=layer_ids, device=f"cuda:{gpu}",
                                do_normalize=common.read_do_normalize(model_file))
    for s in range(0, len(audio_files), clips_per_launch):
        chunk = audio_files[s:s + clips_per_launch]
        waves = []
        for audio_file in chunk:
            samples, sr = sf.read(audio_file)
            if sr != SAMPLE_RATE:   # Wav2Vec2FeatureExtractor refuses other rates in the reference
                raise ValueError(f"{audio_file}: sampling rate {sr}; the feature extractor expects {SAMPLE_RATE}")
            waves.append(samples)
        files = [os.path.join(save_dir, os.path.basename(f)[:-4] + ".npy") for f in chunk]
        ext.extract_waves(waves, feature_level, save_files=files)
    print(f"Total time used: {time.time() - start_time:.1f}s.")


def build_parser():
    parser = argparse.ArgumentParser(description="Run.")
    parser.add_argument("--gpu", type=int, default=0, help="index of gpu")
    parser.add_argument("--model_name", type=str, default="opensmile", help="name of feature extractor")
    parser.add_argument("--feature_level", type=str, default="FRAME", help="name of feature level, FRAME or UTTERANCE")
    parser.add_argument("--overwrite", action="store_true", default=True, help="whether overwrite existed feature folder.")
    parser.add_argument("--dataset", type=str, default="BoxOfLies", help="input dataset")
    return parser


def main(args, config=None):
    if config is None:
        from .. import config as config  # noqa: PLW0127
    layer_ids = LAST
    model_class(args.model_name)   # refused before any directory is made
    audio_dir = config.PATH_TO_RAW_AUDIO[args.dataset]
    save_dir = config.PATH_TO_FEATURES[args.dataset]
    audio_files = glob.glob(os.path.join(audio_dir, "*.wav"))
    print(f'Find total "{len(audio_files)}" audio files.')
    save_dir = os.path.join(save_dir, save_dir_name(args.model_name, args.feature_level, layer_ids))
    prepare_save_dir(save_dir, args.overwrite)
    extract(args.model_name, audio_files, save_dir, args.feature_level, layer_ids=layer_ids, gpu=args.gpu,
            config=config)


if __name__ == "__main__":
    main(build_parser().parse_args())
