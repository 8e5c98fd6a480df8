#!/usr/bin/env python
"""bench.py — clips/sec of the MERTools hot path on one or more H100s.

One "step" = one pass of the hot path over one batch of synthetic clips per GPU:
  tri-modal feature extraction (ViT-B/16 on 8 frames 224x224, HuBERT-base on a 5 s 16 kHz waveform,
  BERT-base on a 32-token sentence) of CLIPS clips, then one Attention-fusion training step on those
  CLIPS clips' features (forward + CE/MSE loss + backward + [NCCL all-reduce] + Adam).
`value`  : whole-job clips/s with the step's inputs already resident in HBM.
`e2e`    : same metric through the public host-buffer API (pinned host inputs -> H2D -> extract ->
           features D2H -> fusion step with H2D of features/labels -> loss D2H), copies timed.
`--impl reference` times the reference's algorithm on the host CPU cores (the oracle port: the
reference is pure Python over torch/transformers).
`--dump-outputs DIR` writes what the last timed step computed (the loss and the three clip-feature arrays) as
DIR/<name>.npy; the inputs and weights are seeded, so two builds can be compared output for output.

Weak scaling: every rank processes its own CLIPS clips per step; the only collective is the fusion
gradient all-reduce (1.9 MB).  Random-init weights (no network), synthetic inputs.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

CLIPS = int(os.environ.get("MER_BENCH_CLIPS", "256"))     # clips per GPU per step
FRAMES, SAMPLES, TOKENS, VOCAB = 8, 80000, 32, 2629
GF_PER_CLIP = dict(visual=281.0, audio=71.66, text=5.47)   # SURVEY.md §8d (2*MAC)
METRIC = "clips/sec tri-modal feature-extract + fusion-train step"


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d["hbm_gbs"], bf16=d["bf16_tflops"], bf16_sustained=d["bf16_tflops_sustained"],
                    src="measured")
    # NVIDIA H100 SXM data sheet (700 W): HBM3 3.35 TB/s, dense fp16 / bf16 989 TFLOP/s; not reached figures
    return dict(hbm=3350.0, bf16=989.0, bf16_sustained=989.0, src="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.index), "-lms", "100"], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc is None:
            return None
        self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        if not sm:
            return None
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 2 + i and r[2 + i] == "Active" for r in self.rows)]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        return dict(sm_mhz=float(np.median(sm)), sm_max_mhz=max(mx) if mx else None, reasons=reasons,
                    samples=len(sm))


def make_inputs(rank, clips):
    """Synthetic step inputs in pinned host memory (SURVEY.md §8d shapes)."""
    g = torch.Generator().manual_seed(1234 + rank)
    frames = torch.randint(0, 256, (clips * FRAMES, 224, 224, 3), dtype=torch.uint8, generator=g).pin_memory()
    wave = (torch.randn(clips, SAMPLES, generator=g) * (3000.0 / 32768.0)).pin_memory()
    ids = torch.randint(5, VOCAB, (clips, TOKENS), dtype=torch.int32, generator=g)
    ids[:, 0], ids[:, -1] = 2, 3  # [CLS] ... [SEP]
    emo = torch.randint(0, 6, (clips,), dtype=torch.int64, generator=g).pin_memory()
    val = ((torch.rand(clips, 1, generator=g) * 6.0) - 3.0).pin_memory()
    return frames, wave, ids.pin_memory(), emo, val


def build_models(device):
    from mertools_b200 import synthetic as S
    from mertools_b200.encoders import BertEncoder, HubertEncoder, VitEncoder
    from mertools_b200.fusion import FusionNet
    vit = VitEncoder(S.vit_state_dict(seed=0), device=device)
    hub = HubertEncoder(S.hubert_state_dict(seed=1), device=device)
    hub._bench_sd = S.hubert_state_dict(seed=1)
    bert = BertEncoder(S.bert_state_dict(VOCAB, seed=2), device=device)
    fus = FusionNet(dropout=0.3, device=device, seed=7).load_state_dict(S.fusion_state_dict(seed=3))
    return vit, hub, bert, fus


def device_step(models, dev_in, clips, world):
    """The hot path on device-resident inputs.  Returns the loss tensor (device)."""
    vit, hub, bert, fus = models
    frames, wave, ids, emo, val = dev_in
    vfeat = vit.clip_features(frames, FRAMES)
    afeat, _ = hub.forward(wave, normalize=True)
    tfeat, _ = bert.forward_packed(ids, TOKENS)
    loss, _, _ = fus.train_step(afeat, tfeat, vfeat, emo, val, lr=1e-3, weight_decay=1e-5,
                                world_size=world)
    return loss, dict(visual_features=vfeat, audio_features=afeat, text_features=tfeat)


def dump_outputs(out_dir, loss, feats):
    """The last timed step's results as float32 .npy files (3 x clips x 768 features + the loss vector)."""
    os.makedirs(out_dir, exist_ok=True)
    arrays = dict(feats, loss=loss)
    for name, t in arrays.items():
        np.save(os.path.join(out_dir, f"{name}.npy"), t.detach().float().cpu().numpy())


def _log(msg):
    if os.environ.get("MER_BENCH_VERBOSE"):
        print(f"[bench rank {os.environ.get('RANK', '0')} {time.strftime('%H:%M:%S')}] {msg}", file=sys.stderr, flush=True)


def fusion_latency(device):
    """SURVEY.md §8d: the fusion step is latency-bound -> microseconds per step on CUDA-graph replay, B = 32 / 256."""
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    from bench_fusion_step import fusion_step_us
    out = {}
    for B in (32, 256):
        r = fusion_step_us(B, iters=200, device=str(device))
        out[f"B{B}"] = {"graph_replay_us": r["graph_replay_us"], "clips_per_s": r["clips_per_s"],
                        "kernels_per_step": r["kernels_per_step"]}
    out["what"] = ("one Attention-fusion training step (forward + CE/MSE + backward + Adam; hidden 128, dropout 0.3) as a "
                   "CUDA-graph replay of fus_rows_fast_kernel + fus_wgrad_kernel, CUDA events over 200 replays, measured before "
                   "the extraction loop (un-capped SM clock, as in a training run of the fusion net on its own)")
    return out


def mixed_length_audio(hub_sd, device, clips=256, seed=5):
    """The workload users see (reference loop extract_audio_huggingface.py:72-110: a different length per file):
    `clips` waveforms of U(2 s, 10 s) from host memory through AudioExtractor (ragged batches, H2D inside)."""
    from mertools_b200.extract.audio import AudioExtractor
    rng = np.random.default_rng(seed)
    lens = rng.integers(2 * 16000, 10 * 16000 + 1, clips)
    waves = [(rng.standard_normal(int(n)) * (3000.0 / 32768.0)) for n in lens]
    ext = AudioExtractor(hub_sd, device=device)
    ext.extract_waves(waves[:32])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ext.extract_waves(waves)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return {"workload": f"{clips} waveforms of U(2 s, 10 s) (mean {lens.mean() / 16000:.2f} s), host numpy in, UTTERANCE features "
                        "out, ragged batches (AudioExtractor default); HuBERT-base only",
            "clips_per_s": clips / dt, "audio_seconds_per_s": float(lens.sum()) / 16000 / dt,
            "frames_over_249": int((lens > 80079).sum())}


def run_ours(args):
    import torch.distributed as dist
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world} (launch with torch.distributed.run)"
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=device)
        _log("process group up")
    from mertools_b200 import _lib as L
    L.check(L.lib().mer_check_device())
    L.lib().mer_launch_count.restype = __import__("ctypes").c_longlong
    clips = args.clips
    models = build_models(device)
    host_in = make_inputs(rank, clips)
    dev_in = [x.to(device) for x in host_in]
    _log("models and inputs ready")

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    # the fusion step is latency-bound (its time follows the SM clock), and a training run executes it on its own: take
    # its number BEFORE the extraction loop has driven the GPU into its power cap (after the loop the same replay
    # measures 1.4x longer at the capped ~1.35 GHz)
    extras = {}
    if rank == 0 and not args.no_extras:
        try:
            extras["fusion_step_us"] = fusion_latency(device)
        except Exception as ex:  # noqa: BLE001 -- the headline line must not depend on the side measurements
            extras["error"] = repr(ex)

    # ---------------- device-resident arm ----------------
    for _ in range(args.warmup):
        device_step(models, dev_in, clips, world)
    barrier()
    _log("warm-up done")
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    import ctypes as C
    L.lib().mer_profile_enable(1)
    l0 = L.lib().mer_launch_count()
    g0 = models[3].graph_launches
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.steps):
        loss, feats = device_step(models, dev_in, clips, world)
    ev[1].record()
    barrier()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, feats)
    ms = ev[0].elapsed_time(ev[1])
    launches = int(L.lib().mer_launch_count() - l0 + models[3].graph_launches - g0)
    prof = {}
    for name, mode in (("tf32", 0), ("bf16x3", 1), ("f16", 2), ("f16_small", 3), ("conv_f16", 4), ("att_f16", 10), ("att_tc", 11), ("ln", 12),
                       ("posconv", 13), ("conv0", 14)):
        t, f, n = C.c_double(), C.c_double(), C.c_int()
        L.lib().mer_profile_collect(mode, C.byref(t), C.byref(f), C.byref(n))
        prof[name] = (t.value, f.value, n.value)
    L.lib().mer_profile_enable(0)
    clocks = sampler.stop() if rank == 0 else None
    tmax = torch.tensor([ms], device=device)
    if world > 1:
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    ms_dev = float(tmax.item())
    _log(f"device arm done: {ms_dev:.1f} ms")

    # ---------------- end-to-end arm (host buffers, copies timed) ----------------
    vit, hub, bert, fus = models

    from mertools_b200.pipeline import TriModalPipeline
    pipe = TriModalPipeline(vit, hub, bert, fus, frames_per_clip=FRAMES, seqlen=TOKENS, world_size=world)

    def e2e_step():
        return pipe.step_host(*host_in)

    for _ in range(max(1, args.warmup // 2)):
        e2e_step()
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        e2e_step()
    barrier()
    e2e_ms = (time.perf_counter() - t0) * 1e3
    tmax = torch.tensor([e2e_ms], device=device)
    if world > 1:
        dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    e2e_ms = float(tmax.item())
    h2d = sum(x.numel() * x.element_size() for x in host_in) + 3 * clips * 768 * 4
    d2h = 3 * clips * 768 * 4 + 4
    if world > 1:  # data-parallel replicas must agree: the all-reduced loss and the parameters are identical on every rank
        sig = torch.stack([loss[2].double(), fus.params.double().sum()])
        lo, hi = sig.clone(), sig.clone()
        dist.all_reduce(lo, op=dist.ReduceOp.MIN)
        dist.all_reduce(hi, op=dist.ReduceOp.MAX)
        assert torch.equal(lo, hi), f"ranks disagree on the fusion loss / parameters: {lo.tolist()} vs {hi.tolist()}"
    if rank == 0 and not args.no_extras:
        try:
            extras["mixed_length_audio"] = mixed_length_audio(hub._bench_sd, device)
            # the same step with the ViT linears on TF32 operands (MER_VIT_PRECISION=tf32), same inputs
            from mertools_b200 import synthetic as S2
            from mertools_b200.encoders import VitEncoder
            vit32 = VitEncoder(S2.vit_state_dict(seed=0), device=device, precision="tf32")
            m32 = (vit32, hub, bert, fus)
            for _ in range(2):
                device_step(m32, dev_in, clips, 1)
            torch.cuda.synchronize()
            e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            e[0].record()
            for _ in range(max(2, args.steps // 2)):
                device_step(m32, dev_in, clips, 1)
            e[1].record()
            torch.cuda.synchronize()
            ms32 = e[0].elapsed_time(e[1]) / max(2, args.steps // 2)
            extras["tf32_vit"] = {"value": clips / (ms32 * 1e-3), "unit": "clips/s (this GPU alone)", "ms_per_step": ms32,
                                  "what": "the device-resident step with VitEncoder(precision='tf32'): ViT linears on TF32 "
                                          "operands at half the fp16 tensor rate; audio / text / fusion unchanged"}
            del vit32
        except Exception as ex:  # noqa: BLE001 -- the headline line must not depend on the side measurements
            extras["error"] = repr(ex)
    if world > 1:
        dist.barrier()

    if rank == 0:
        pk = peaks()
        total_clips = clips * world * args.steps
        # dominant kernel: the ViT stack's linear layers, fp16 operands by default (MER_VIT_PRECISION=tf32
        # selects the TF32 variant).  Denominator: the kernel is timed inside a long step -> the SUSTAINED bf16
        # figure of MEASURED_PEAKS when present (fp16 and bf16 share the tensor-pipe rate; tf32 runs at half of it);
        # the fraction of the burst figure is given beside it.
        use_f16 = prof["f16"][2] > 0
        t_ms, t_fl, t_n = prof["f16"] if use_f16 else prof["tf32"]
        div = 1.0 if use_f16 else 2.0
        tf32_peak = pk["bf16_sustained"] / div
        burst_peak = pk["bf16"] / div
        ach = t_fl / (t_ms * 1e-3) / 1e12 if t_ms > 0 else 0.0
        # every other kernel class of the encoders, event-timed the same way over the same timed region
        def entry(key, kernel, bound, peak, unit, scale):
            k_ms, k_work, k_n = prof[key]
            if k_n == 0 or k_ms <= 0:
                return None
            a = k_work / (k_ms * 1e-3) / scale
            return {"kernel": kernel, "bound": bound, "achieved": a, "peak": peak, "unit": unit, "frac": a / peak,
                    "launches_timed": k_n, "share_of_step": k_ms / ms_dev if ms_dev else None}
        sus = pk["bf16_sustained"]
        other = [e for e in (
            entry("bf16x3", "gemm_kernel<*, BF16X3> (3 bf16 MMAs per product; HuBERT conv3-6 + feature projection)", "tensor",
                  sus / 3.0, "TFLOP/s (useful)", 1e12),
            entry("conv_f16", "gemm_kernel<256, F16> as HuBERT conv1 / conv2 (implicit GEMM over time-major fp16 "
                  "rows, k = 3, stride 2)", "tensor", sus, "TFLOP/s", 1e12),
            entry("f16_small", "gemm_kernel<*, F16> on the HuBERT (63,744 rows) and BERT (8,192 rows) layers: 10 / 1.3 waves of "
                  "tiles at N = 768", "tensor", sus, "TFLOP/s", 1e12),
            entry("att_f16", "attention_vt_kernel<f16> (mma.sync f16; ViT 197, HuBERT 249, BERT 32 tokens)", "tensor", sus,
                  "TFLOP/s", 1e12),
            entry("att_tc", "attention_vt_kernel<tf32> (mma.sync tf32; HuBERT 249 tokens, BERT)", "tensor", sus / 2.0,
                  "TFLOP/s", 1e12),
            entry("ln", "layernorm_kernel (warp per row, 128-bit I/O)", "hbm", pk["hbm"], "GB/s", 1e9),
            entry("conv0", "conv0 moments + coefficients + apply (HuBERT conv0 + GroupNorm + GELU; statistics from the "
                  "waveform's tap moments, one pass over the output, fp16 rows out: 4.2 GB)", "hbm", pk["hbm"],
                  "GB/s", 1e9),
            entry("posconv", "HuBERT positional conv (grouped k=128) as a windowed block-diagonal F16 GEMM; algorithmic FLOPs "
                  "(the GEMM executes 6.67x as many)", "tensor", sus, "TFLOP/s", 1e12),
            entry("tf32" if use_f16 else "f16", "gemm_kernel<256, TF32> (ViT patch embedding)", "tensor", sus / 2.0,
                  "TFLOP/s", 1e12),
        ) if e]
        line = {
            "metric": METRIC, "value": total_clips / (ms_dev * 1e-3), "unit": "clips/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_dev / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": ("f16 operands (ViT / HuBERT / BERT layers, ViT attention) / tf32 (audio + text "
                                          "attention, patch embed)" if use_f16 else "tf32 (ViT)") +
                                          " / f16 (HuBERT conv1-2) / bf16x3 (HuBERT conv3-6, feature projection) tensor-core products, fp32 accumulate; fp32 elsewhere",
            "data": "synthetic inputs, seeded random-init weights (no network)",
            "config": {"workload": f"tri-modal extract (ViT-B/16 {FRAMES}x224x224 frames + HuBERT-base 5 s @16 kHz + "
                                   f"BERT-base {TOKENS} tokens) + Attention-fusion train step (hidden 128, dropout 0.3), "
                                   f"{clips} clips per GPU per step",
                       "clips_per_gpu_per_step": clips, "l2": "step inputs + activations (>10 GB) exceed the 50 MB L2",
                       "text_inputs": "pre-tokenised ids (the HF tokenizer is host code on both arms)",
                       "parallelism": f"clip-sharded x{world}, one NCCL all-reduce of the fusion gradient per step"},
            "e2e": {"value": total_clips / (e2e_ms * 1e-3), "unit": "clips/s",
                    "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h)},
            "gpu_launches": launches,
            "clocks": clocks,
            "roofline": {"kernel": ("gemm_kernel<256, F16> (wgmma f16; the 48 linear layers of the ViT stack, 403,456 rows)"
                                    if use_f16 else
                                    "gemm_kernel<256, TF32> (wgmma tf32; ViT linear layers)"),
                         "bound": "tensor", "achieved": ach, "peak": tf32_peak, "unit": "TFLOP/s",
                         "frac": ach / tf32_peak if tf32_peak else None,
                         "frac_vs_burst": ach / burst_peak if burst_peak else None,
                         "launches_timed": t_n, "share_of_step": t_ms / ms_dev if ms_dev else None,
                         "peak_source": (f"{pk['src']} MEASURED_PEAKS bf16_tflops_sustained (kernel timed inside a long "
                                         f"step; fp16 = bf16 pipe rate); burst = {burst_peak:.1f}") if use_f16 else
                                        (f"{pk['src']} MEASURED_PEAKS bf16_tflops_sustained / 2 (tf32 pipe rate = half "
                                         f"the bf16 rate); burst / 2 = {burst_peak:.1f}")},
            "roofline_other": other,
        }
        line.update(extras)
        line["cpu_baseline"] = cpu_baseline(sample_clips=args.cpu_clips)
        if not args.no_extras:
            line["cpu_baseline"]["whole_host"] = cpu_whole_host(line["cpu_baseline"]["cores"])
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------
# CPU baseline: the oracle port of the reference path on the host cores
# ------------------------------------------------------------------------------------------------
_CPU_STATE = {}


def _pick_threads():
    """torch intra-op threads that maximise the reference path's throughput on this host: the
    reference runs one clip per forward, and on a many-core box torch's default (all cores) can be
    far slower than a moderate count (measured 24 s/clip at 128 threads).  Quick calibration on a
    4-layer ViT forward of one 8-frame clip."""
    from mertools_b200 import synthetic as S
    from oracle import encoders as E
    sd = {k: torch.from_numpy(v) for k, v in S.vit_state_dict(seed=0, layers=4).items()}
    x = torch.randn(FRAMES, 3, 224, 224)
    ncpu = os.cpu_count() or 1
    best, best_t = 1, float("inf")
    for n in sorted({min(ncpu, c) for c in (8, 16, 32, 64, ncpu)}):
        torch.set_num_threads(n)
        with torch.no_grad():
            E.vit_hidden_states(sd, x, layers=4)
            t0 = time.perf_counter()
            E.vit_hidden_states(sd, x, layers=4)
            dt = time.perf_counter() - t0
        if dt < best_t:
            best, best_t = n, dt
        if dt > 4 * best_t:
            break
    torch.set_num_threads(best)
    return best


def _cpu_setup():
    if _CPU_STATE:
        return _CPU_STATE
    from mertools_b200 import synthetic as S
    _CPU_STATE["threads"] = _pick_threads()
    to_t = lambda sd: {k: torch.from_numpy(v) for k, v in sd.items()}  # noqa: E731
    _CPU_STATE.update(vit=to_t(S.vit_state_dict(seed=0)), hub=to_t(S.hubert_state_dict(seed=1)),
                      bert=to_t(S.bert_state_dict(VOCAB, seed=2)), fus=S.fusion_state_dict(seed=3))
    return _CPU_STATE


def cpu_step(n_clips, seed=0):
    """Reference algorithm (oracle port) for n_clips clips on the CPU: per-clip extraction loops as in
    the reference scripts (one clip per forward), then one fusion step.  Returns seconds."""
    from mertools_b200 import synthetic as S
    from oracle import fusion as OF
    from oracle import pipeline as P
    st = _cpu_setup()
    frames = S.synth_frames(n_clips, FRAMES, seed=seed)
    waves = S.synth_waves(n_clips, SAMPLES, seed=seed).astype(np.float64) / 32768.0
    rng = np.random.default_rng(seed)
    ids = rng.integers(5, VOCAB, (n_clips, TOKENS))
    t0 = time.perf_counter()
    with torch.no_grad():
        v = np.stack([P.visual_clip_features(st["vit"], frames[i]) for i in range(n_clips)])
        a = np.stack([P.audio_clip_features(st["hub"], waves[i]) for i in range(n_clips)])
        t = np.stack([P.text_clip_features(st["bert"], ids[i].tolist(), 1, -1) for i in range(n_clips)])
    tr = OF.Trainer(st["fus"], lr=1e-3, l2=1e-5)
    emo = torch.from_numpy(rng.integers(0, 6, n_clips))
    val = torch.from_numpy(rng.uniform(-3, 3, (n_clips, 1)).astype(np.float32))
    tr.step(torch.from_numpy(a), torch.from_numpy(t), torch.from_numpy(v), emo, val)
    return time.perf_counter() - t0


def cpu_baseline(sample_clips=48):
    _cpu_setup()        # weight generation + thread calibration, untimed
    cpu_step(1)         # warm-up
    sec1 = cpu_step(1)  # sizing of the bounded sample: about 15 s of CPU work
    n = int(max(2, min(sample_clips, 15.0 / max(sec1, 1e-3))))
    sec = cpu_step(n)
    return {"value": n / sec, "unit": "clips/s", "cores": torch.get_num_threads(), "kind": "port",
            "sample": f"{n} synthetic clips, tri-modal extract (one clip per forward, as the reference scripts "
                      f"do) + one fusion step, torch CPU fp32, {torch.get_num_threads()} threads (best of a "
                      f"calibration over 8..{os.cpu_count()} on this {os.cpu_count()}-core host), {sec:.1f} s"}


def cpu_whole_host(threads_per_proc, clips_per_proc=2):
    """The whole host, not one process: P = cores // threads independent processes of the reference port, each on
    `threads_per_proc` torch threads, started together; value = total clips / wall time of the slowest."""
    ncpu = os.cpu_count() or 1
    procs = max(1, min(16, ncpu // max(1, threads_per_proc)))
    cmd = [sys.executable, os.path.abspath(__file__), "--cpu-worker", str(clips_per_proc), "--cpu-threads", str(threads_per_proc)]
    try:
        t0 = time.perf_counter()
        ps = [subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True) for _ in range(procs)]
        secs = [float(p.communicate(timeout=600)[0].strip().splitlines()[-1]) for p in ps]
        wall = time.perf_counter() - t0
        return {"value": procs * clips_per_proc / max(secs), "unit": "clips/s", "processes": procs,
                "threads_per_process": threads_per_proc, "cores_used": procs * threads_per_proc, "host_cores": ncpu,
                "sample": f"{procs} processes x {clips_per_proc} clips, slowest {max(secs):.1f} s (wall incl. start-up {wall:.0f} s)"}
    except Exception as ex:  # noqa: BLE001
        return {"value": None, "error": repr(ex)}


def cpu_worker(n_clips, threads, steps=1):
    _CPU_STATE["threads"] = threads
    torch.set_num_threads(threads)
    from mertools_b200 import synthetic as S
    to_t = lambda sd: {k: torch.from_numpy(v) for k, v in sd.items()}  # noqa: E731
    _CPU_STATE.update(vit=to_t(S.vit_state_dict(seed=0)), hub=to_t(S.hubert_state_dict(seed=1)),
                      bert=to_t(S.bert_state_dict(VOCAB, seed=2)), fus=S.fusion_state_dict(seed=3))
    cpu_step(1)
    for k in range(steps):
        print(cpu_step(n_clips, seed=k), flush=True)


def run_reference(args):
    """The reference's CPU implementation of the path on ALL the host cores: P = cores // T processes of the oracle
    port (T = the calibrated torch thread count at which one process is fastest), every process running the same
    bounded K-step sample; a step's time is the slowest process's, value = P * n * K / sum of step times."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    _cpu_setup()
    threads = _CPU_STATE["threads"]
    cpu_step(1)
    sec1 = cpu_step(1)
    ncpu = os.cpu_count() or 1
    procs = max(1, min(16, ncpu // max(1, threads)))
    # bounded sample: keep the whole K-step run within a few minutes (contended processes run ~1.5x slower)
    n = int(max(1, min(args.cpu_clips, 90.0 / max(args.steps, 1) / max(sec1, 1e-3))))
    warm = max(1, args.warmup - 2)
    cmd = [sys.executable, os.path.abspath(__file__), "--cpu-worker", str(n), "--cpu-threads", str(threads),
           "--cpu-steps", str(warm + args.steps)]
    ps = [subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True) for _ in range(procs)]
    per_proc = []
    for p_ in ps:
        lines = p_.communicate(timeout=3000)[0].strip().splitlines()
        per_proc.append([float(x) for x in lines[-(warm + args.steps):]][warm:])
    secs = [max(t[k] for t in per_proc) for k in range(args.steps)]
    total = sum(secs)
    value = procs * n * args.steps / total
    sample = (f"{procs} processes x {threads} torch threads = {procs * threads} of {ncpu} host cores; {n} clips per process "
              f"and step x {args.steps} steps; oracle port of the reference path (the reference is pure Python); one process "
              f"alone: {1.0 / sec1:.2f} clips/s")
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "clips/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": total / args.steps * 1e3,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32 (torch CPU)",
        "data": "synthetic inputs, seeded random-init weights (no network)",
        "config": {"workload": f"tri-modal extract (ViT-B/16 {FRAMES}x224x224 + HuBERT-base 5 s + BERT-base {TOKENS} tok) "
                               f"+ Attention-fusion train step; bounded sample of {procs} x {n} clips per step on the host CPU"},
        "cpu_baseline": {"value": value, "unit": "clips/s", "cores": procs * threads, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": "clips/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", type=str, default="ours", choices=["ours", "reference"])
    ap.add_argument("--clips", type=int, default=CLIPS, help="clips per GPU per step")
    ap.add_argument("--cpu-clips", type=int, default=48, help="upper bound of clips in the bounded CPU sample")
    ap.add_argument("--no-extras", action="store_true", help="skip the side measurements (fusion latency, mixed-length "
                    "audio, TF32 ViT, whole-host CPU figure)")
    ap.add_argument("--dump-outputs", type=str, default=None, metavar="DIR",
                    help="write the last timed step's loss and clip features to DIR/<name>.npy (float32)")
    ap.add_argument("--cpu-worker", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--cpu-threads", type=int, default=16, help=argparse.SUPPRESS)
    ap.add_argument("--cpu-steps", type=int, default=1, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.cpu_worker:
        cpu_worker(a.cpu_worker, a.cpu_threads, a.cpu_steps)
    elif a.impl == "reference":
        run_reference(a)
    else:
        run_ours(a)
