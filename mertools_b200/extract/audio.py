"""Acoustic feature extraction — H100 mirror of
MERBench/feature_extraction/audio/extract_audio_huggingface.py (HuBERT / wav2vec2-base branch).

Keeps ``extract(model_name, audio_files, save_dir, feature_level, gpu)`` (:52) and
``split_into_batch`` (:40-50).  The per-file loop of the reference (batch = 1 clip, numpy
normalisation on the host) becomes: raw float32 samples of many clips staged in pinned memory,
grouped by length, one fused device pass per group (normalise + conv stack + 12 layers + readout).
"""
from __future__ import annotations

import argparse
import glob
import math
import os
import time

import numpy as np
import torch

import ctypes as C

from .. import _lib as L
from ..encoders import HubertEncoder
from . import common

HUBERT_BASE_CHINESE = "chinese-hubert-base"
WAV2VEC2_BASE_CHINESE = "chinese-wav2vec2-base"
DATA2VEC_AUDIO_BASE = "data2vec-audio-base-960h"   # Data2VecAudioModel: recognised from its positional conv chain
WAVLM_BASE = "wavlm-base"                          # WavLMModel: extract/wavlm.py (gated relative position bias)
WAVLM_LARGE = "wavlm-large"
WHISPER_BASE = "whisper-base"                      # encoder-decoder branch (:83-91): extract/whisper.py
WHISPER_LARGE = "whisper-large-v2"
MAXLEN = 16000 * 10


def split_into_batch(input_values, maxlen=MAXLEN):
    """[1, wavlen] -> [ceil(wavlen/maxlen), maxlen], zero padded (reference :40-50)."""
    if input_values.shape[1] <= maxlen:
        return input_values
    assert input_values.shape[0] == 1
    wavlen = input_values.shape[1]
    tgt = math.ceil(wavlen / maxlen) * maxlen
    out = torch.zeros((1, tgt), dtype=input_values.dtype, device=input_values.device)
    out[:, :wavlen] = input_values
    return out.view(-1, maxlen)


class AudioExtractor:
    def __init__(self, state_dict, device="cuda", max_rows_per_launch=128, ragged=None, max_samples_per_launch=128 * MAXLEN // 2,
                 do_normalize=True, last_layer_only=False):
        """ragged (default on; env MER_AUDIO_RAGGED=0 switches it off): clips of different lengths share one device pass
        (``HubertEncoder.forward_ragged``: every clip computed as if alone) instead of one pass per distinct
        length; sorted by length and cut into launches of at most ``max_samples_per_launch`` padded samples.
        last_layer_only: read out ``hidden_states[-1]`` instead of the sum of the last four (HuBERT / wav2vec2 only)."""
        if "encoder.layers.0.attention.gru_rel_pos_linear.weight" in state_dict:   # WavLMModel (wavlm-base / -large)
            from .wavlm import WavLmEncoder
            self.enc = WavLmEncoder(state_dict, device=device)
            assert not ragged, "ragged batches are implemented for the HuBERT / wav2vec2 families only"  # None: default
            assert not last_layer_only, "the last-layer readout is implemented for the HuBERT / wav2vec2 families only"
            ragged = False
        else:
            self.enc = HubertEncoder(state_dict, device=device, last_layer_only=last_layer_only)
        self.device = self.enc.device
        self.max_rows = max_rows_per_launch
        # ragged batches: one launch chain for clips of any length instead of one pass per distinct length; results
        # agree with the per-length passes to float rounding
        self.ragged = (os.environ.get("MER_AUDIO_RAGGED", "1") != "0") if ragged is None else bool(ragged)
        self.max_samples = max_samples_per_launch
        # Wav2Vec2FeatureExtractor.do_normalize of the checkpoint (common.read_do_normalize): zero-mean / unit-variance or not
        self.do_normalize = bool(do_normalize)
        self._norm = L.declare("mer_wave_normalize", [C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                      C.c_longlong, C.c_longlong, C.c_void_p])

    def _staging(self, slot, rows, cols):
        """View [rows, cols] of one of the two persistent pinned staging buffers (grown on demand)."""
        if not hasattr(self, "_pinned"):
            self._pinned = [None, None]
        need = rows * cols
        buf = self._pinned[slot]
        if buf is None or buf.numel() < need:
            buf = self._pinned[slot] = torch.zeros(max(need, self.max_samples, MAXLEN), dtype=torch.float32,
                                                   pin_memory=self.device.type == "cuda")  # (host-logic tests stub the encoder)
        return buf[:need].view(rows, cols)

    def _run_rows(self, rows, normalize):
        """rows: CUDA fp32 [R, L] -> frames [R, T, D] (sum of the last four hidden states; D = 768 or 1024)."""
        outs = []
        for s in range(0, rows.shape[0], self.max_rows):
            _, fr = self.enc.forward(rows[s:s + self.max_rows], normalize=normalize, want_frames=True)
            outs.append(fr.clone())
        return torch.cat(outs)

    def _extract_ragged(self, waves, clips, feature_level, res):
        """Clips ``clips`` (indices into waves) through ``forward_ragged``: sorted by length, cut into launches of at most
        ``max_rows`` clips and ``max_samples`` padded samples; res[i] receives clip i's frames [T, D] or mean [D]."""
        order = sorted(clips, key=lambda i: len(waves[i]))
        launches, s0 = [], 0
        while s0 < len(order):   # launches of consecutive (sorted) clips: rows * longest <= max_samples
            e = s0 + 1
            while (e < len(order) and e - s0 < self.max_rows
                   and (e - s0 + 1) * len(waves[order[e]]) <= self.max_samples):
                e += 1
            launches.append(order[s0:e])
            s0 = e
        # Two persistent pinned staging buffers (a fresh pinned allocation per launch cost as much as the launch's
        # device time) and a one-launch-deep pipeline: launch k is enqueued, the host fills the buffer of launch
        # k + 1 while the GPU works, and only then are the results of launch k read back -- in ONE device-to-host
        # copy per launch (round 2's first build synchronised once per clip).
        want_frames = feature_level != "UTTERANCE"

        def finish(p):
            idxs, utt, frames = p
            if want_frames:
                for r, i in enumerate(idxs):
                    res[i] = frames[r].cpu().numpy()
            else:
                u = utt.cpu().numpy()
                for r, i in enumerate(idxs):
                    res[i] = u[r].copy()

        pending = None
        for k, idxs in enumerate(launches):
            lens = [len(waves[i]) for i in idxs]
            host = self._staging(k & 1, len(idxs), max(lens))
            hn = host.numpy()            # shares the pinned memory; the assignment converts float64 -> float32 in place
            for r, i in enumerate(idxs):
                hn[r, :lens[r]] = waves[i]
                hn[r, lens[r]:] = 0.0
            utt, frames = self.enc.forward_ragged(host.to(self.device, non_blocking=True), lens,
                                                  normalize=self.do_normalize, want_frames=want_frames)
            if pending is not None:
                finish(pending)          # (synchronises: buffer k & 1 is free again two launches later)
            pending = (idxs, utt, frames)
        if pending is not None:
            finish(pending)

    def extract_waves(self, waves, feature_level="UTTERANCE", save_files=None):
        """waves: list of 1-D float arrays (what ``sf.read`` returns, 16 kHz mono).  Returns the
        arrays the reference would ``np.save`` (:103-110)."""
        res = [None] * len(waves)
        short = {}
        for i, w in enumerate(waves):
            w = np.asarray(w)
            assert w.ndim == 1, "mono audio only"
            if len(w) <= MAXLEN:
                short.setdefault(len(w), []).append(i)
        if self.ragged and len(short) > 1:
            self._extract_ragged(waves, [i for idxs in short.values() for i in idxs], feature_level, res)
            short = {}
        # clips <= 10 s: batch by identical length; normalisation fused on the device
        for n, idxs in short.items():
            host = torch.empty((len(idxs), n), dtype=torch.float32, pin_memory=True)
            for r, i in enumerate(idxs):
                host[r] = torch.from_numpy(np.asarray(waves[i]).astype(np.float32))
            fr = self._run_rows(host.to(self.device, non_blocking=True), normalize=self.do_normalize)
            feats = fr.mean(dim=1).cpu().numpy() if feature_level == "UTTERANCE" else fr.cpu().numpy()
            for r, i in enumerate(idxs):
                res[i] = feats[r]
        # clips > 10 s: normalise the whole waveform first, then 10 s rows (reference order :94-95)
        for i, w in enumerate(waves):
            if res[i] is not None:
                continue
            x = torch.from_numpy(np.asarray(w).astype(np.float32))[None].to(self.device)
            xn = x
            if self.do_normalize:
                xn = torch.empty_like(x)
                L.check(self._norm(L.ptr(x), L.ptr(xn), 1, x.shape[1], x.shape[1], x.shape[1],
                                   L.stream_ptr()))
            rows = split_into_batch(xn)
            fr = self._run_rows(rows.contiguous(), normalize=False).reshape(-1, self.enc.hidden)
            res[i] = (fr.mean(dim=0) if feature_level == "UTTERANCE" else fr).cpu().numpy()
        if save_files is not None:
            for f, r in zip(save_files, res):
                np.save(f, r)
        return res


def extract(model_name, audio_files, save_dir, feature_level, gpu, config=None, clips_per_launch=128):
    """Same signature and on-disk result as the reference ``extract`` (:52-113)."""
    import soundfile as sf
    if config is None:
        from .. import config as config  # noqa: PLW0127
    from .. import shard
    start_time = time.time()
    assert gpu != -1, "mertools_b200 has no CPU path (reference: gpu=-1 means CPU)"
    gpu = shard.device_index(gpu)
    torch.cuda.set_device(gpu)
    # one process per GPU under torchrun: this rank's share of the files that do not have their .npy yet
    audio_files, rank, world = shard.my_work(audio_files, lambda f: os.path.join(save_dir, os.path.basename(f)[:-4] + ".npy"))
    if world > 1:
        print(f"rank {rank}/{world}: {len(audio_files)} audio files on cuda:{gpu}")
    model_file = os.path.join(config.PATH_TO_PRETRAINED_MODELS, f"transformers/{model_name}")
    if model_name in (WHISPER_BASE, WHISPER_LARGE):
        import json

        from .whisper import WhisperExtractor
        with open(os.path.join(model_file, "config.json")) as f:
            cfg = json.load(f)
        sd = {k[len("model."):] if k.startswith("model.") else k: v for k, v in common.load_hf_state_dict(model_file).items()}
        ext = WhisperExtractor(sd, cfg["decoder_start_token_id"], device=f"cuda:{gpu}", heads=cfg["encoder_attention_heads"])
    else:
        ext = AudioExtractor(common.load_hf_state_dict(model_file), device=f"cuda:{gpu}",
                             do_normalize=common.read_do_normalize(model_file))
    for s in range(0, len(audio_files), clips_per_launch):
        chunk = audio_files[s:s + clips_per_launch]
        waves = []
        for audio_file in chunk:
            samples, sr = sf.read(audio_file)
            assert sr == 16000, "currently, we only test on 16k audio"
            waves.append(samples)
        files = [os.path.join(save_dir, os.path.basename(f)[:-4] + ".npy") for f in chunk]
        ext.extract_waves(waves, feature_level, save_files=files)
    print(f"Total time used: {time.time() - start_time:.1f}s.")


def build_parser():
    parser = argparse.ArgumentParser(description="Run.")
    parser.add_argument("--gpu", type=int, default=0, help="index of gpu")
    parser.add_argument("--model_name", type=str, default="chinese-hubert-large", help="feature extractor")  # :120
    parser.add_argument("--feature_level", type=str, default="FRAME", help="FRAME or UTTERANCE")
    parser.add_argument("--dataset", type=str, default="MER2023", help="input dataset")
    parser.add_argument("--noise_case", type=str, default=None)
    parser.add_argument("--tts_lang", type=str, default=None)
    return parser


def main(args, config=None):
    if config is None:
        from .. import config as config  # noqa: PLW0127
    audio_dir = config.PATH_TO_RAW_AUDIO[args.dataset]
    save_dir = config.PATH_TO_FEATURES[args.dataset]
    if args.noise_case is not None:
        audio_dir += "_" + args.noise_case
    if args.tts_lang is not None:
        audio_dir += "-" + f"tts{args.tts_lang[:3]}16k"
    audio_files = glob.glob(os.path.join(audio_dir, "*.wav"))
    print(f'Find total "{len(audio_files)}" audio files.')
    if args.noise_case is not None:
        dir_name = f"{args.model_name}-noise{args.noise_case}-{args.feature_level[:3]}"
    elif args.tts_lang is not None:
        dir_name = f"{args.model_name}-tts{args.tts_lang[:3]}-{args.feature_level[:3]}"
    else:
        dir_name = f"{args.model_name}-{args.feature_level[:3]}"
    save_dir = os.path.join(save_dir, dir_name)
    os.makedirs(save_dir, exist_ok=True)
    extract(args.model_name, audio_files, save_dir, args.feature_level, gpu=args.gpu, config=config)


if __name__ == "__main__":
    main(build_parser().parse_args())
