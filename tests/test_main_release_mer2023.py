"""CPU tests of the MER2023 baseline trainer (mertools_b200.main_release_mer2023): the golden of the unmodified
MER2023/main-release.py replayed through the trainer's host loop on the oracle's net, the feature reader's rules, the
save_root suffixes, the fold averaging, the report functions and the one-row Attention refusal."""
import os

import numpy as np
import pytest
import torch

import _mer2023_replay as RP
from mertools_b200 import main_release_mer2023 as M
from mertools_b200.fusion_mlp import check_batch, mask_shapes, param_shapes, reference_init
from oracle import mer2023 as O


@pytest.mark.parametrize("tag", ["mlp", "att"])
def test_golden_replayed_through_the_oracle(tag, tmp_path):
    """Fold membership, every step's loss, every pass's F1 / MSE, the best epochs, the fold-0..4 predictions, the
    state_dict layout, the output file names and the submission CSVs of the reference run."""
    make = lambda kind, dims, sd: O.Net(kind, sd)  # noqa: E731
    rp, written, folder_save, name_time, args = RP.run(tag, str(tmp_path), make_net=make, device=torch.device("cpu"))
    RP.check_replay(tag, rp, written, folder_save, name_time, args, str(tmp_path), tol=2e-6)


def test_reader_takes_the_one_glob_match(tmp_path):
    np.save(tmp_path / "clip_01.npy", np.arange(5, dtype=np.float32)[None])
    assert M.func_read_one(str(tmp_path), "clip_01").shape == (5,)
    np.save(tmp_path / "clip_010.npy", np.zeros(5, np.float32))
    with pytest.raises(AssertionError, match="matches 2 entries"):
        M.func_read_one(str(tmp_path), "clip_01")       # clip_01* also matches clip_010.npy
    with pytest.raises(AssertionError, match="matches 0 entries"):
        M.func_read_one(str(tmp_path), "clip_02")


def test_reader_averages_a_directory_of_faces(tmp_path):
    d = tmp_path / "clip_07"
    d.mkdir()
    faces = np.random.default_rng(0).standard_normal((4, 6)).astype(np.float32)
    for i in (2, 0, 3, 1):   # written out of order; read sorted
        np.save(d / f"face_{i}.npy", faces[i][None])
    np.testing.assert_array_equal(M.func_read_one(str(tmp_path), "clip_07"), faces.mean(axis=0))
    d1 = tmp_path / "clip_08"
    d1.mkdir()
    np.save(d1 / "face_0.npy", faces[0])  # one face: squeezed to a vector, no mean
    np.testing.assert_array_equal(M.func_read_one(str(tmp_path), "clip_08"), faces[0])


def test_save_root_suffixes():
    assert M.save_root_suffix("./s", "A", "A", "A") == "./s-unimodal"
    assert M.save_root_suffix("./s", "A", "T", "A") == "./s-bimodal"
    assert M.save_root_suffix("./s", "A", "T", "V") == "./s-trimodal"


def test_average_folder_results_means_logits_then_argmax():
    folds = [{"t_names": ["b", "a"], "t_emoprobs": np.array([[0., 2, 0, 0, 0, 0], [1., 0, 0, 0, 0, 0]]),
              "t_valpreds": np.array([[1.0], [2.0]])},
             {"t_names": ["a", "b"], "t_emoprobs": np.array([[0., 0, 3, 0, 0, 0], [0., 0, 0, 3, 0, 0]]),
              "t_valpreds": np.array([[4.0], [-1.0]])}]
    out = M.average_folder_results(folds, "t")
    assert list(out) == ["b", "a"]
    assert out["a"]["emo"] == 2 and out["a"]["val"] == pytest.approx(3.0)
    assert out["b"]["emo"] == 3 and out["b"]["val"] == pytest.approx(0.0)   # mean logits (0, 1, 0, 1.5, ..)
    np.testing.assert_allclose(out["b"]["emoprob"], [0, 1, 0, 1.5, 0, 0])


def test_report_functions(tmp_path):
    from sklearn.metrics import f1_score
    lab, pred = tmp_path / "label.csv", tmp_path / "pred.csv"
    lab.write_text("name,discrete,valence\nx,happy,1.0\ny,sad,-2.0\nz,angry,0.5\n")
    M.write_to_csv_pred({"x": {"emo": 2, "val": 1.5}, "y": {"emo": 2, "val": -2.0}, "z": {"emo": 1, "val": 0.5}},
                        str(pred))
    f1, mse, metric = M.report_results_on_test1_test2(str(lab), str(pred))
    assert f1 == pytest.approx(f1_score([2, 3, 1], [2, 2, 1], average="weighted"))
    assert mse == pytest.approx(0.25 / 3) and metric == pytest.approx(f1 - 0.25 * mse)
    lab.write_text("name,discrete\ny,sad\n")     # test3 labels a subset and has no valence
    assert M.report_results_on_test3(str(lab), str(pred)) == (pytest.approx(0.0), -100, -100)


def test_one_row_attention_batch_is_refused():
    with pytest.raises(ValueError, match="at least 2 rows"):
        check_batch("attention", 1)
    check_batch("attention", 2)
    check_batch("mlp", 1)
    sd = reference_init("attention", 5, 6, 7, "8,4")
    x = [torch.zeros(1, d) for d in (5, 6, 7)]
    with pytest.raises(ValueError, match="at least 2 rows"):
        O.forward(sd, "attention", *x)


def test_layout_and_initial_draw_follow_the_reference_constructors():
    """state_dict order and the generator consumption of MLP(...) / Attention(...): the same draws as building the
    reference's module tree (a restated one here: nn.Sequential of Linear / ReLU / Dropout per chain)."""
    nn = torch.nn

    def chain(k, layers):
        mods = []
        for n in layers:
            mods += [nn.Linear(k, n), nn.ReLU(), nn.Dropout(0.3)]
            k = n
        return nn.Sequential(*mods)

    for kind, layers in (("mlp", [16, 8]), ("attention", [9, 5, 3])):
        torch.manual_seed(3)
        ref = {}
        if kind == "mlp":
            for k, v in chain(10 + 12 + 7, layers).state_dict().items():
                ref[f"module.{k}"] = v
        else:
            for name, k in (("audio_mlp", 10), ("text_mlp", 12), ("video_mlp", 7), ("attention_mlp", 3 * layers[-1])):
                for kk, v in chain(k, layers).state_dict().items():
                    ref[f"{name}.{kk}"] = v
            for kk, v in nn.Linear(layers[-1], 3).state_dict().items():
                ref[f"fc_att.{kk}"] = v
        for head, o in (("fc_out_1", 6), ("fc_out_2", 1)):
            for kk, v in nn.Linear(layers[-1], o).state_dict().items():
                ref[f"{head}.{kk}"] = v
        torch.manual_seed(3)
        sd = reference_init(kind, 10, 12, 7, ",".join(map(str, layers)))
        assert list(sd) == list(ref) == list(param_shapes(kind, 10, 12, 7, layers))
        for k in sd:
            assert torch.equal(sd[k], ref[k]), k
        assert len(mask_shapes(kind, layers, 4)) == len(layers) * (1 if kind == "mlp" else 4)


def test_cli_refuses_other_corpora_and_data_parallel(monkeypatch, tmp_path):
    args = M.build_parser().parse_args(["--dataset=MER2024", f"--save_root={tmp_path}/s"])
    with pytest.raises(AssertionError, match="MER2023-format corpora only"):
        M.main(args, config=object(), device=torch.device("cpu"))
    monkeypatch.setenv("WORLD_SIZE", "2")
    args = M.build_parser().parse_args(["--dataset=MER2023"])
    with pytest.raises(SystemExit, match="one GPU"):
        M.main(args, config=object(), device=torch.device("cpu"))
    assert not os.path.exists(f"{tmp_path}/s-unimodal")
