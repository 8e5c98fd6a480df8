"""CPU tests of MER2023's audio extractor (extract/audio_mer2023.py): refusals and their messages, the directory
naming and overwrite rules of extract_transformers_embedding.py:96-105, name-to-class dispatch, the extractor's CLI,
and the C ABI (MerHubertModel.readout, mer_attention_long, the ABI version)."""
import ctypes as C
import os
import shutil
import subprocess
import types

import numpy as np
import pytest

from mertools_b200.extract import audio_mer2023 as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name,cls", [("chinese-hubert-base", "HubertModel"), ("chinese-hubert-large", "HubertModel"),
                                      ("chinese-wav2vec2-base", "Wav2Vec2Model"), ("wav2vec2-large-960h", "Wav2Vec2Model"),
                                      ("hubert-wav2vec-mix", "HubertModel")])
def test_name_to_class_dispatch(name, cls):
    assert M.model_class(name) == cls


@pytest.mark.parametrize("name", ["wavlm-base", "data2vec-audio-base-960h", "whisper-base", "opensmile", "HuBERT-base"])
def test_other_names_are_refused(name):
    with pytest.raises(ValueError, match=r"containing 'hubert'.*'wav2vec'.*unbound"):
        M.model_class(name)


def test_layer_ids():
    assert M.last_layer_only([-1]) is True
    assert M.last_layer_only((-4, -3, -2, -1)) is False
    with pytest.raises(ValueError, match=r"layer_ids=None: .*assert feature.shape\[0\] == 1"):
        M.last_layer_only(None)
    for bad in ([-2], [-1, -2], [-3, -2, -1], [12], []):
        with pytest.raises(ValueError, match=r"layer_ids .*: the device readouts are hidden_states\[-1\]"):
            M.last_layer_only(bad)


def test_extract_refuses_before_loading_anything(tmp_path):
    cfg = types.SimpleNamespace(PATH_TO_PRETRAINED_MODELS=str(tmp_path / "missing"))
    with pytest.raises(ValueError, match="unbound"):
        M.extract("wavlm-base", [], str(tmp_path), "UTTERANCE", layer_ids=[-1], gpu=0, config=cfg)
    with pytest.raises(ValueError, match="layer_ids=None"):
        M.extract("chinese-hubert-base", [], str(tmp_path), "UTTERANCE", gpu=0, config=cfg)
    for gpu in (None, -1):
        with pytest.raises(ValueError, match=r"runs on a CUDA device"):
            M.extract("chinese-hubert-base", [], str(tmp_path), "UTTERANCE", layer_ids=[-1], gpu=gpu, config=cfg)


def test_save_dir_names():
    assert M.save_dir_name("chinese-hubert-large", "UTTERANCE") == "chinese-hubert-large-UTT"
    assert M.save_dir_name("chinese-wav2vec2-base", "FRAME", [-1]) == "chinese-wav2vec2-base-FRA"
    assert M.save_dir_name("chinese-hubert-base", "FRAME", [-4, -3, -2, -1]) == "chinese-hubert-base-4-FRA"


def test_overwrite_rules(tmp_path, capsys):
    d = tmp_path / "feats" / "chinese-hubert-base-UTT"
    M.prepare_save_dir(str(d), overwrite=False)          # created
    assert d.is_dir()
    M.prepare_save_dir(str(d), overwrite=False)          # exists but empty: reused with a warning
    assert "Warning: overwrite" in capsys.readouterr().out
    (d / "a.npy").write_bytes(b"x")
    M.prepare_save_dir(str(d), overwrite=True)           # not empty, overwrite: reused, file kept
    assert (d / "a.npy").exists()
    with pytest.raises(FileExistsError, match="already exists, set overwrite=TRUE if needed"):
        M.prepare_save_dir(str(d), overwrite=False)


def test_cli_flags_mirror_the_reference():
    a = M.build_parser().parse_args([])
    assert (a.gpu, a.model_name, a.feature_level, a.overwrite, a.dataset) == (0, "opensmile", "FRAME", True, "BoxOfLies")
    a = M.build_parser().parse_args(["--gpu=1", "--model_name=chinese-hubert-base", "--feature_level=UTTERANCE",
                                     "--overwrite", "--dataset=MER2023"])
    assert (a.gpu, a.model_name, a.feature_level, a.overwrite, a.dataset) == (1, "chinese-hubert-base", "UTTERANCE",
                                                                               True, "MER2023")


def test_main_names_the_directory_and_hands_over(tmp_path, monkeypatch):
    audio = tmp_path / "audio"
    audio.mkdir()
    (audio / "a.wav").write_bytes(b"")
    cfg = types.SimpleNamespace(PATH_TO_RAW_AUDIO={"MER2023": str(audio)},
                                PATH_TO_FEATURES={"MER2023": str(tmp_path / "features")})
    seen = {}
    monkeypatch.setattr(M, "extract", lambda *a, **k: seen.update(args=a, kw=k))
    M.main(M.build_parser().parse_args(["--model_name=chinese-wav2vec2-base", "--dataset=MER2023",
                                        "--feature_level=UTTERANCE"]), config=cfg)
    save_dir = str(tmp_path / "features" / "chinese-wav2vec2-base-UTT")
    assert os.path.isdir(save_dir)
    assert seen["args"] == ("chinese-wav2vec2-base", [str(audio / "a.wav")], save_dir, "UTTERANCE")
    assert seen["kw"]["layer_ids"] == [-1] and seen["kw"]["gpu"] == 0
    with pytest.raises(ValueError, match="unbound"):   # refused before the directory is made
        M.main(M.build_parser().parse_args(["--model_name=wavlm-base", "--dataset=MER2023"]), config=cfg)
    assert not os.path.exists(tmp_path / "features" / "wavlm-base-FRA")


def test_stereo_is_refused_with_a_message():
    ext = M.Mer2023AudioExtractor.__new__(M.Mer2023AudioExtractor)   # no device: the check runs first
    with pytest.raises(ValueError, match=r"clip 1: mono audio only"):
        ext.extract_waves([np.zeros(16000), np.zeros((16000, 2))])


def test_every_clip_takes_the_ragged_path_and_one_frame_clips_are_squeezed():
    """Clips of any length (here 1 s and 40 s, beyond the 10 s split of the MERBench extractor) go to the ragged
    launches unsplit; a one-frame clip comes back as [D] like the reference's feature[0].squeeze()."""
    ext = M.Mer2023AudioExtractor.__new__(M.Mer2023AudioExtractor)
    calls = []

    def fake(waves, clips, level, res):
        calls.append((list(clips), level))
        for i in clips:
            res[i] = np.ones((max(1, (len(waves[i]) - 400) // 320 + 1), 4), np.float32)
    ext._extract_ragged = fake
    out = ext.extract_waves([np.zeros(640000), np.zeros(400), np.zeros(16000)], "FRAME")
    assert calls == [([0, 1, 2], "FRAME")]
    assert [o.shape for o in out] == [(1999, 4), (4,), (49, 4)]


# ---- C ABI ------------------------------------------------------------------------------------------------------------
def test_hubert_model_struct_layout_matches_the_header(tmp_path):
    from mertools_b200.encoders import MerHubertModel
    if shutil.which("gcc") is None:
        pytest.skip("no C compiler")
    fields = ["conv_w_f16", "readout"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(
        ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "mer_b200.h")}"',
         "int main(void) {", '  printf("%zu", sizeof(MerHubertModel));']
        + [f'  printf(" %zu", offsetof(MerHubertModel, {f}));' for f in fields]
        + ['  printf(" %d %d %d\\n", MER_HUBERT_READOUT_LAST4, MER_HUBERT_READOUT_LAST, MER_ATT_LONG_MAX);',
           "  return 0;", "}"]))
    subprocess.run(["gcc", "-o", str(tmp_path / "probe"), str(src)], check=True)
    want = [int(v) for v in subprocess.run([str(tmp_path / "probe")], check=True, capture_output=True,
                                           text=True).stdout.split()]
    from mertools_b200 import encoders as En
    got = ([C.sizeof(MerHubertModel)] + [getattr(MerHubertModel, f).offset for f in fields]
           + [En.MER_HUBERT_READOUT_LAST4, En.MER_HUBERT_READOUT_LAST, 4096])
    assert got == want
    assert MerHubertModel().readout == 0   # zero-initialised = the last-four readout of before


def test_abi_version_is_still_4_and_the_export_exists():
    from mertools_b200 import _lib
    dll = C.CDLL(_lib.LIB_PATH)
    assert dll.mer_abi_version() == 4
    assert hasattr(dll, "mer_attention_long") and hasattr(dll, "mer_hubert_forward_ragged")
