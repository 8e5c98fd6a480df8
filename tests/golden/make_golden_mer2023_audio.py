"""Golden fixture for MER2023's own audio extractor: the UNMODIFIED reference function
MER2023/feature_extraction/audio/extract_transformers_embedding.py:extract (whole clips, no 10 s split, readout
``torch.stack(hidden_states)[layer_ids].sum(0)``) run on the CPU over three seeded checkpoints:

  chinese-hubert-base    HubertModel, base configuration (12 post-LN layers)
  chinese-wav2vec2-base  Wav2Vec2Model, base configuration (12 post-LN layers)
  chinese-hubert-large   HubertModel, large stable-layer-norm configuration, 4 layers (kept shallow for the CPU run)

and clips of 1 s, 9.9 s, 10.5 s, 25 s and 40 s, at FRAME and UTTERANCE level, with the CLI's layer_ids = [-1]; the
HuBERT base model also with layer_ids = [-4, -3, -2, -1] at UTTERANCE level.

Run once in the build container (needs the reference checkout + transformers; NOT on the GPU box):
    python tests/golden/make_golden_mer2023_audio.py
Writes tests/golden/mer2023_audio_golden.npz.  Same stubs as make_golden.py (`soundfile.read` via scipy, patched
`config`).  The archive is written with fixed zip timestamps, so a second run writes the same bytes.
"""
import importlib.util
import io
import os
import sys
import tempfile
import types
import zipfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference/MER2023"
OUT = os.path.dirname(os.path.abspath(__file__))

from mertools_b200 import synthetic as S  # noqa: E402

LENS = (16000, 158400, 168000, 400000, 640000)   # 1 s, 9.9 s, 10.5 s, 25 s, 40 s
SEED0 = 700
FRAME_STEP = 64                                  # FRAME fixtures keep every 64th row ...
FRAME_COLS = 256                                 # ... and its first 256 features (fixture size)
# name -> (HF model class, state-dict kwargs of synthetic.hubert_state_dict, config kwargs, layers)
MODELS = {
    "chinese-hubert-base": ("HubertModel", dict(seed=21), dict(), 12),
    "chinese-wav2vec2-base": ("Wav2Vec2Model", dict(seed=22), dict(), 12),
    "chinese-hubert-large": ("HubertModel", dict(seed=23, large=True),
                             dict(hidden_size=1024, num_attention_heads=16, intermediate_size=4096,
                                  feat_extract_norm="layer", do_stable_layer_norm=True, conv_bias=True), 4),
}


def savez_deterministic(path, arrays):
    """np.savez with fixed member timestamps (np.savez stamps the current time)."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(),
                       compress_type=zipfile.ZIP_DEFLATED)


def main():
    import scipy.io.wavfile as wavfile
    import transformers
    from transformers import Wav2Vec2FeatureExtractor
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    work = tempfile.mkdtemp(prefix="mer_golden_m23a_")
    tools = os.path.join(work, "tools", "transformers")
    feats = os.path.join(work, "features")
    os.makedirs(tools)
    os.makedirs(feats)
    cfg = types.ModuleType("config")
    cfg.PATH_TO_RAW_AUDIO = {"MER2023": os.path.join(work, "audio")}
    cfg.PATH_TO_FEATURES = {"MER2023": feats}
    cfg.PATH_TO_PRETRAINED_MODELS = os.path.join(work, "tools")
    sys.modules["config"] = cfg
    sf = types.ModuleType("soundfile")

    def sf_read(path):
        sr, x = wavfile.read(path)
        return x.astype(np.float64) / 32768.0, sr
    sf.read = sf_read
    sys.modules["soundfile"] = sf
    os.makedirs(cfg.PATH_TO_RAW_AUDIO["MER2023"])
    files = []
    for i, n in enumerate(LENS):
        f = os.path.join(cfg.PATH_TO_RAW_AUDIO["MER2023"], f"wav{i}.wav")
        wavfile.write(f, 16000, S.synth_waves(1, n, seed=SEED0 + i)[0])
        files.append(f)
    spec = importlib.util.spec_from_file_location(
        "ref_m23_audio", os.path.join(REF, "feature_extraction", "audio", "extract_transformers_embedding.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)

    out = dict(lens=np.array(LENS), seed0=SEED0, frame_step=FRAME_STEP, frame_cols=FRAME_COLS)
    for name, (cls, sd_kw, cfg_kw, layers) in MODELS.items():
        mdir = os.path.join(tools, name)
        config_cls = getattr(transformers, cls.replace("Model", "Config"))
        m = getattr(transformers, cls)(config_cls(num_hidden_layers=layers, **cfg_kw))
        sd = {k: torch.from_numpy(v) for k, v in S.hubert_state_dict(layers=layers, **sd_kw).items()}
        missing, unexpected = m.load_state_dict(sd, strict=False)
        assert not unexpected and set(missing) <= {"masked_spec_embed"}, (missing, unexpected)
        m.save_pretrained(mdir)
        Wav2Vec2FeatureExtractor(do_normalize=True).save_pretrained(mdir)
        key = name.replace("chinese-", "").replace("-", "_")
        out[f"{key}_layers"] = layers
        out[f"{key}_seed"] = sd_kw["seed"]
        runs = [("UTTERANCE", [-1]), ("FRAME", [-1])]
        if name == "chinese-hubert-base":
            runs.append(("UTTERANCE", [-4, -3, -2, -1]))
        for level, layer_ids in runs:
            d = os.path.join(feats, f"{name}-{len(layer_ids)}-{level[:3]}")
            os.makedirs(d)
            ref.extract(name, files, d, level, layer_ids=layer_ids, gpu=-1)
            for i in range(len(LENS)):
                x = np.load(os.path.join(d, f"wav{i}.npy"))
                tag = f"{key}_{'last' if len(layer_ids) == 1 else 'last4'}_{level[:3].lower()}{i}"
                out[tag] = x if level == "UTTERANCE" else x[::FRAME_STEP, :FRAME_COLS]
                if level == "FRAME":
                    out[tag + "_frames"] = x.shape[0]
            print(name, level, layer_ids, flush=True)
    savez_deterministic(os.path.join(OUT, "mer2023_audio_golden.npz"), out)
    print({k: np.shape(v) for k, v in out.items()})


if __name__ == "__main__":
    main()
