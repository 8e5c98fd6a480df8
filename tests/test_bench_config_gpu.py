"""Parity AT the benchmarked configuration (BASELINE.json configs[1..3]; VERDICT r1 'weak' item 1) and on stress
checkpoints at full depth.

test_parity_at_the_benchmarked_configuration builds exactly what bench.py times -- the same models
(bench.build_models), the same 256-clip step inputs (bench.make_inputs) -- and runs the same three calls
(VitEncoder.clip_features on 256 x 8 frames, HubertEncoder.forward on 256 x 80,000 samples,
BertEncoder.forward_packed on 256 x 32 ids) plus TriModalPipeline.step_host.  Eight sampled clips per modality are
compared with the oracle (1e-3 relative, north_star), the fusion loss of the step with the oracle trainer on the
device-extracted features, and the GEMM instantiations the bench runs on (gemm_kernel<256, F16> for the ViT / HuBERT /
BERT layers, gemm_kernel<256, BF16X3> for the HuBERT conv stack) are asserted to have launched.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from mertools_b200 import synthetic as S
from oracle import encoders as E
from oracle import fusion as OF
from oracle import pipeline as P

pytestmark = pytest.mark.gpu
TOL = 1e-3
SAMPLE = [0, 37, 91, 128, 170, 201, 230, 255]


def _rel(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(got - ref).max() / np.abs(ref).max())


def test_parity_at_the_benchmarked_configuration(cuda):
    import bench
    from mertools_b200 import _lib as L
    from mertools_b200.pipeline import TriModalPipeline
    lib = L.lib()
    lib.mer_gemm_variant_launches.restype = C.c_longlong
    variant = lambda bn, mode, cl, two: int(lib.mer_gemm_variant_launches(bn, mode, cl, two))  # noqa: E731
    clips = 256
    vit, hub, bert, fus = models = bench.build_models(cuda)
    host_in = bench.make_inputs(0, clips)
    frames, wave, ids, emo, val = dev_in = [x.to(cuda) for x in host_in]
    n_f16, n_x3 = variant(256, 2, 1, 0), variant(256, 1, 1, 0)
    vfeat = vit.clip_features(frames, bench.FRAMES).clone()
    assert variant(256, 2, 1, 0) - n_f16 >= 48, "the ViT linears did not run on gemm_kernel<256, F16>"
    n_f16 = variant(256, 2, 1, 0)
    afeat = hub.forward(wave, normalize=True)[0].clone()
    tfeat = bert.forward_packed(ids, bench.TOKENS)[0].clone()
    assert hub.stack_precision == "f16" and hub.conv_precision == "f16" and bert.precision == "f16"
    # conv3..6 + the feature projection on split operands; conv1 / conv2 and the 12 layers on fp16 operands
    assert variant(256, 1, 1, 0) - n_x3 >= 5, "HuBERT conv3..6 / projection did not run on gemm_kernel<256, BF16X3>"
    assert variant(256, 2, 1, 0) - n_f16 >= 50, "HuBERT conv1 / conv2 / layers did not run on gemm_kernel<256, F16>"
    torch.cuda.synchronize()
    assert vfeat.shape == afeat.shape == tfeat.shape == (clips, 768)
    for t in (vfeat, afeat, tfeat):
        assert bool(torch.isfinite(t).all())

    to_t = lambda sd: {k: torch.from_numpy(v) for k, v in sd.items()}  # noqa: E731
    sd_v, sd_a = to_t(S.vit_state_dict(seed=0)), to_t(S.hubert_state_dict(seed=1))
    sd_t = to_t(S.bert_state_dict(bench.VOCAB, seed=2))
    fr, wv, idh = host_in[0].numpy(), host_in[1].numpy(), host_in[2].numpy()
    worst = dict(visual=0.0, audio=0.0, text=0.0)
    with torch.no_grad():
        for c in SAMPLE:
            ref = P.visual_clip_features(sd_v, fr[c * bench.FRAMES:(c + 1) * bench.FRAMES], nframe=None)
            worst["visual"] = max(worst["visual"], _rel(vfeat[c].cpu().numpy(), ref))
            ref = P.audio_clip_features(sd_a, wv[c].astype(np.float64))
            worst["audio"] = max(worst["audio"], _rel(afeat[c].cpu().numpy(), ref))
            ref = P.text_clip_features(sd_t, idh[c].tolist(), 1, -1)
            worst["text"] = max(worst["text"], _rel(tfeat[c].cpu().numpy(), ref))
    print(f"bench configuration, 8 of {clips} clips per modality, max-rel vs oracle: {worst}")
    assert all(v < TOL for v in worst.values()), worst

    # the fusion step of the same bench step (dropout 0.3, masks from the counter hash -> compare at dropout 0 too)
    sd_f = S.fusion_state_dict(seed=3)
    from mertools_b200.fusion import FusionNet
    net = FusionNet(dropout=0.0, device=cuda).load_state_dict(sd_f)
    loss, _, _ = net.train_step(afeat, tfeat, vfeat, emo, val, lr=1e-3, weight_decay=1e-5)
    ref = OF.Trainer(sd_f, lr=1e-3, l2=1e-5).step(afeat.cpu(), tfeat.cpu(), vfeat.cpu(), emo.cpu(), val.cpu())
    assert abs(float(loss[2].cpu()) - ref[2]) <= 1e-3 * max(1.0, abs(ref[2])), (float(loss[2]), ref[2])

    # the end-to-end call of the bench: host buffers in, loss out; same features -> same kind of loss
    pipe = TriModalPipeline(vit, hub, bert, fus, frames_per_clip=bench.FRAMES, seqlen=bench.TOKENS)
    a2, t2, v2 = pipe.extract_host(*host_in[:3])
    assert _rel(a2.numpy(), afeat.cpu().numpy()) < 2e-4 and _rel(v2.numpy(), vfeat.cpu().numpy()) < 2e-4
    assert _rel(t2.numpy(), tfeat.cpu().numpy()) < 2e-4
    l_host = pipe.step_host(*host_in)
    assert np.isfinite(l_host) and 0.5 < l_host < 50.0


# ---- stress checkpoints --------------------------------------------------------------------------------------
# Scaling every matrix weight by s multiplies the network's condition number: the fp32 reference itself drifts from
# a float64 evaluation by 2e-7 (s = 1), 7e-7 (3), 6e-6 (5), 7e-4 (10) on the ViT readout and 3e-7 / 5e-6 / 1.5e-3 on
# HuBERT (measured with the oracle, dtype=float64 against float32).  A tensor-core product with u-bit operands
# carries 2^(24-u) times the operand rounding of fp32, so the honest bar on such a checkpoint is
#     err <= max(1e-3, SLACK * 2^(24-u) * |fp32 reference - fp64 reference|)
# (u = 11 for fp16 / TF32 operands, 17 for the bf16 hi+lo split): the first term is north_star's tolerance, the
# second says "no worse than the operand format allows on THIS checkpoint".  Both terms and the margin are printed.
SLACK = 4.0


def _bar(noise, mantissa_bits):
    return max(TOL, SLACK * 2.0 ** (24 - mantissa_bits) * noise)


@pytest.mark.parametrize("precision", ["f16", "tf32"])
@pytest.mark.parametrize("scale", [3.0, 5.0, 10.0])
def test_vit_stress_checkpoint_at_full_depth(cuda, precision, scale):
    """SURVEY.md Appendix A: every matrix weight of the 12 layers x3 / x5 / x10 (peaky softmax rows, large GELU
    arguments, LayerNorm inputs with large means; fp16 operands saturate at 65,504)."""
    from mertools_b200.encoders import VitEncoder
    sd = S.vit_state_dict(seed=0, layers=12, scale=scale)
    frames = S.synth_frames(1, 3, seed=11)[0]
    enc = VitEncoder(sd, device=cuda, precision=precision)
    feats, hidden = enc.frame_features(torch.from_numpy(frames).to(cuda), return_hidden=True)
    x = P.vit_preprocess(frames)
    with torch.no_grad():
        ref_hs = E.vit_hidden_states(sd, x, layers=12)
        ref64 = torch.stack(E.vit_hidden_states(sd, x, layers=12, dtype=torch.float64))[-1].sum(dim=1)
    ref = torch.stack(ref_hs)[-1].sum(dim=1)
    noise = _rel(ref.numpy(), ref64.numpy())
    m = _rel(feats.cpu().numpy(), ref.numpy())
    bar = _bar(noise, 11)
    print(f"ViT x{scale:g} {precision}: readout max-rel {m:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e}); margin "
          f"{bar / max(m, 1e-12):.1f}x; |x| max {float(ref_hs[-1].abs().max()):.0f}")
    assert bool(torch.isfinite(feats).all()) and m < bar


@pytest.mark.parametrize("precision,bits", [("f16", 11), ("bf16x3", 17)])
@pytest.mark.parametrize("scale", [3.0, 5.0, 10.0])
def test_hubert_stress_checkpoint_at_full_depth(cuda, scale, precision, bits):
    """Both operand formats of the 12 layers (the conv feature encoder is BF16X3 in both): fp16 (default since round
    2, 11 significant bits) and the bf16 (hi, lo) split (17)."""
    from mertools_b200.encoders import HubertEncoder
    sd = S.hubert_state_dict(seed=1, layers=12, scale=scale)
    wav = (S.synth_waves(2, 48000, seed=29).astype(np.float64) / 32768.0).astype(np.float32)
    enc = HubertEncoder(sd, device=cuda, stack_precision=precision)
    utt, _ = enc.forward(torch.from_numpy(wav).to(cuda), normalize=True)
    worst, noise = 0.0, 0.0
    with torch.no_grad():
        for i in range(2):
            ref = P.audio_clip_features(sd, wav[i].astype(np.float64), layers=12)
            worst = max(worst, _rel(utt[i].cpu().numpy(), ref))
            if i == 0:
                noise = _rel(ref, P.audio_clip_features(sd, wav[i].astype(np.float64), layers=12, dtype=torch.float64))
    bar = _bar(noise, bits)
    print(f"HuBERT x{scale:g} {precision}: readout max-rel {worst:.2e}; bar {bar:.2e} (fp32-vs-fp64 {noise:.1e}); margin "
          f"{bar / max(worst, 1e-12):.1f}x")
    assert bool(torch.isfinite(utt).all()) and worst < bar
