"""Throughput of the decoder-LLM text-feature paths (LLaMA at 7 B and 13 B shapes; BLOOM-7B1, OPT-13B, Falcon-7B and the
two GPT-2 models on request) against the reference's loop.

Packed path: LlamaNet on the CUDA backend (fp16 weights and operands, fp32 residual), sentences packed back to back,
up to --tokens per pass.  Reference loop (extract_text_huggingface.py:193-231): batch 1, one sentence per forward, fp16,
output_hidden_states and the last-four sum; HF LlamaModel when transformers imports, else the torch restatement
(LlamaNet + TorchOps) in fp16 on the GPU — the output says which ran.  Weights are seeded random fp16 tensors generated
on the device (no checkpoint on disk); sentence lengths are seeded draws shaped like the MER2023 transcripts under a
Chinese sentencepiece tokenizer (mean ~20 tokens, p99 ~53, capped at 128).  The time shares of GEMM / attention /
RMSNorm / RoPE / SwiGLU (LayerNorm for BLOOM / OPT) come from CUDA events around every launch, in a separate pass.
``bloom-7b1`` / ``opt-13b`` run LnDecoderNet (extract/ln_decoder_text.py) against HF BloomModel / OPTModel in fp16 at
batch 1 (a 32000-token vocabulary here: the embedding gather is not part of the timed work that matters).
``falcon-7b`` (32 x 4544, 71 query heads of 64 sharing one K / V head, FFN 18176, no biases) runs LnDecoderNet against
HF FalconModel in fp16 at batch 1, as the reference halves it.
``gpt2-chinese`` (gpt2-chinese-cluecorpussmall: 12 x 768, 12 heads of 64) and ``wenzhong-3.5b`` (Wenzhong2.0-GPT2-3.5B:
30 x 3072, 32 heads of 96) run LnDecoderNet against HF GPT2Model at batch 1 in fp32, the precision the reference runs
these two in: their speed-up includes fp16 against fp32.

    python scripts/bench_llm_text.py [--shapes 7b,13b,bloom-7b1,opt-13b,falcon-7b,gpt2-chinese,wenzhong-3.5b]
        [--sentences 1024]
        [--ref-sentences 64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mertools_b200.extract import llama_text as LT  # noqa: E402
from mertools_b200.extract import ln_decoder_text as LD  # noqa: E402

SHAPES = {"7b": dict(hidden=4096, heads=32, ffn=11008, layers=32, eps=1e-6),
          "13b": dict(hidden=5120, heads=40, ffn=13824, layers=40, eps=1e-5),
          "bloom-7b1": dict(family="bloom", hidden=4096, heads=32, ffn=16384, layers=30, eps=1e-5),
          "opt-13b": dict(family="opt", hidden=5120, heads=40, ffn=20480, layers=40, eps=1e-5),
          "falcon-7b": dict(family="falcon", hidden=4544, heads=71, ffn=18176, layers=32, eps=1e-5),
          "gpt2-chinese": dict(family="gpt2", hidden=768, heads=12, ffn=3072, layers=12, eps=1e-5),
          "wenzhong-3.5b": dict(family="gpt2", hidden=3072, heads=32, ffn=12288, layers=30, eps=1e-5)}
MAX_POS = {"bloom": None, "opt": 2048, "gpt2": 1024, "falcon": 2048}
VOCAB = 32000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f"unavailable ({e})"
    return name, q


def sentence_lengths(n, seed):
    rng = np.random.default_rng(seed)
    return np.clip(np.round(rng.lognormal(2.85, 0.45, n)), 2, 128).astype(int).tolist()


def random_weights(s, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    D, I = s["hidden"], s["ffn"]

    def w(*shape, std=0.02):
        return (torch.randn(*shape, generator=g, device=dev, dtype=torch.float16) * std)
    if "family" in s:
        return ln_decoder_weights(s, w)
    sd = {"embed_tokens.weight": w(VOCAB, D, std=1.0), "norm.weight": 1 + w(D, std=0.1)}
    for i in range(s["layers"]):
        p = f"layers.{i}."
        sd.update({p + f"self_attn.{n}.weight": w(D, D) for n in ("q_proj", "k_proj", "v_proj", "o_proj")})
        sd.update({p + "mlp.gate_proj.weight": w(I, D), p + "mlp.up_proj.weight": w(I, D),
                   p + "mlp.down_proj.weight": w(D, I)})
        sd.update({p + n + ".weight": 1 + w(D, std=0.1) for n in ("input_layernorm", "post_attention_layernorm")})
    return sd


def ln_decoder_weights(s, w):
    """BloomModel / OPTModel (decoder.*) / GPT2Model (Conv1D weights [in, out]) keys, biases on every linear and
    LayerNorm; FalconModel keys (multi-query query_key_value, no linear biases)."""
    D, F = s["hidden"], s["ffn"]

    def ln(p):
        return {p + ".weight": 1 + w(D, std=0.1), p + ".bias": w(D, std=0.1)}

    def lin(p, o, i):   # GPT-2's Conv1D: (p, in, out) -> weight [in, out]
        return {p + ".weight": w(o, i), p + ".bias": w(i if s["family"] == "gpt2" else o)}
    sd = {}
    if s["family"] == "bloom":
        sd.update({"word_embeddings.weight": w(VOCAB, D, std=1.0), **ln("word_embeddings_layernorm"), **ln("ln_f")})
        for i in range(s["layers"]):
            p = f"h.{i}."
            sd.update({**ln(p + "input_layernorm"), **ln(p + "post_attention_layernorm"),
                       **lin(p + "self_attention.query_key_value", 3 * D, D), **lin(p + "self_attention.dense", D, D),
                       **lin(p + "mlp.dense_h_to_4h", F, D), **lin(p + "mlp.dense_4h_to_h", D, F)})
    elif s["family"] == "falcon":
        sd.update({"word_embeddings.weight": w(VOCAB, D, std=1.0), **ln("ln_f")})
        for i in range(s["layers"]):
            p = f"h.{i}."
            sd.update({**ln(p + "input_layernorm"), p + "self_attention.query_key_value.weight": w(D + 128, D),
                       p + "self_attention.dense.weight": w(D, D), p + "mlp.dense_h_to_4h.weight": w(F, D),
                       p + "mlp.dense_4h_to_h.weight": w(D, F)})
    elif s["family"] == "gpt2":
        sd.update({"wte.weight": w(VOCAB, D, std=1.0), "wpe.weight": w(MAX_POS["gpt2"], D, std=0.1), **ln("ln_f")})
        for i in range(s["layers"]):
            p = f"h.{i}."
            sd.update({**ln(p + "ln_1"), **ln(p + "ln_2"), **lin(p + "attn.c_attn", D, 3 * D),
                       **lin(p + "attn.c_proj", D, D), **lin(p + "mlp.c_fc", D, F), **lin(p + "mlp.c_proj", F, D)})
    else:
        sd.update({"decoder.embed_tokens.weight": w(VOCAB, D, std=1.0), "decoder.embed_positions.weight":
                   w(2050, D, std=0.1), **ln("decoder.final_layer_norm")})
        for i in range(s["layers"]):
            p = f"decoder.layers.{i}."
            sd.update({**ln(p + "self_attn_layer_norm"), **ln(p + "final_layer_norm"), **lin(p + "fc1", F, D),
                       **lin(p + "fc2", D, F)})
            for n in ("q", "k", "v", "out"):
                sd.update(lin(p + f"self_attn.{n}_proj", D, D))
    return sd


def hf_config(s):
    from transformers import BloomConfig, FalconConfig, GPT2Config, LlamaConfig, OPTConfig
    if s.get("family") == "falcon":
        return FalconConfig(vocab_size=VOCAB, hidden_size=s["hidden"], num_attention_heads=s["heads"],
                            ffn_hidden_size=s["ffn"], num_hidden_layers=s["layers"], layer_norm_epsilon=s["eps"],
                            max_position_embeddings=MAX_POS["falcon"])
    if s.get("family") == "gpt2":
        return GPT2Config(vocab_size=VOCAB, n_positions=MAX_POS["gpt2"], n_embd=s["hidden"], n_layer=s["layers"],
                          n_head=s["heads"], n_inner=s["ffn"], layer_norm_epsilon=s["eps"])
    if s.get("family") == "bloom":
        return BloomConfig(vocab_size=VOCAB, hidden_size=s["hidden"], n_head=s["heads"], n_layer=s["layers"])
    if s.get("family") == "opt":
        return OPTConfig(vocab_size=VOCAB, hidden_size=s["hidden"], num_attention_heads=s["heads"], ffn_dim=s["ffn"],
                         num_hidden_layers=s["layers"], max_position_embeddings=2048, word_embed_proj_dim=s["hidden"])
    return LlamaConfig(vocab_size=VOCAB, hidden_size=s["hidden"], num_attention_heads=s["heads"],
                       intermediate_size=s["ffn"], num_hidden_layers=s["layers"], rms_norm_eps=s["eps"],
                       max_position_embeddings=4096)


def packed_batches(ids, max_tokens):
    b = 0
    while b < len(ids):
        e, tok = b, 0
        while e < len(ids) and (e == b or tok + len(ids[e]) <= max_tokens):
            tok += len(ids[e])
            e += 1
        yield ids[b:e]
        b = e


def run_packed(net, ids, max_tokens):
    for batch in packed_batches(ids, max_tokens):
        net.forward(np.concatenate(batch), [len(x) for x in batch])


def reference_loop(s, sd, ids, dev):
    """Batch-1 forwards with output_hidden_states and the last-four sum, as the reference script does: fp16, except
    GPT-2, which the reference does not halve."""
    try:
        from transformers import BloomModel, FalconModel, GPT2Model, LlamaModel, OPTModel
        cls = {"bloom": BloomModel, "opt": OPTModel, "gpt2": GPT2Model, "falcon": FalconModel}.get(s.get("family"),
                                                                                                  LlamaModel)
        cfg = hf_config(s)
        dt = torch.get_default_dtype()
        ref_dtype = torch.float32 if s.get("family") == "gpt2" else torch.float16
        torch.set_default_dtype(ref_dtype)
        try:
            with torch.device(dev):
                m = cls(cfg).eval()
        finally:
            torch.set_default_dtype(dt)
        m.load_state_dict(sd, strict=True)
        which = f"HF {cls.__name__} {'fp32' if ref_dtype == torch.float32 else 'fp16'}"
        start = 0 if s.get("family") in ("bloom", "falcon") else 1

        def fwd(x):
            hs = m(torch.from_numpy(x)[None].to(dev), output_hidden_states=True).hidden_states
            return torch.stack(hs)[[-4, -3, -2, -1]].sum(0)[0, start:].cpu().numpy()
    except ImportError:
        assert "family" not in s, "the BLOOM / OPT / GPT-2 / Falcon reference loop needs transformers"
        net = LT.LlamaNet(dict(sd), LT.TorchOps(dev, torch.float16), s["layers"], s["heads"], s["eps"], 10000.0, 4096)
        which = "torch restatement fp16 (transformers not importable)"

        def fwd(x):
            return net.forward(x, [len(x)])[1:].cpu().numpy()
    with torch.no_grad():
        for x in ids[:2]:
            fwd(x)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for x in ids:
            fwd(x)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    return which, dt


def rmsnorm_bandwidth(dev, rows=16384, dim=5120, reps=50):
    """mer_rmsnorm at the 13 B width, fp16 output: compulsory bytes (fp32 x in, fp16 y out) over event time."""
    from mertools_b200 import _lib as L
    ops = LT.CudaOps(dev)
    x = torch.randn(rows, dim, device=dev)
    w = torch.ones(dim, device=dev)
    for _ in range(3):
        ops.rmsnorm(x, w, 1e-5)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    y = torch.empty(rows, dim, dtype=torch.float16, device=dev)
    e0.record()
    for _ in range(reps):
        L.check(ops._rms(L.ptr(x), L.ptr(w), L.ptr(y), None, rows, dim, 1e-5, L.stream_ptr()))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return ms, rows * dim * 6 / (ms * 1e-3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="7b,13b")
    ap.add_argument("--sentences", type=int, default=1024)
    ap.add_argument("--ref-sentences", type=int, default=64)
    ap.add_argument("--tokens", type=int, default=16384, help="tokens per packed pass")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="JSON file for the results")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}")
    lens = sentence_lengths(a.sentences, a.seed)
    q = np.percentile(lens, [50, 90, 99])
    print(f"sentence lengths (tokens, BOS included): n {len(lens)} mean {np.mean(lens):.1f} p50 {q[0]:.0f} "
          f"p90 {q[1]:.0f} p99 {q[2]:.0f} max {max(lens)} total {sum(lens)}")
    rng = np.random.default_rng(a.seed + 1)
    ids = [np.concatenate([[1], rng.integers(3, VOCAB, n - 1)]).astype(np.int64) for n in lens]
    results = dict(card=name, power=power, lengths=dict(n=len(lens), mean=float(np.mean(lens)), total=int(sum(lens))))
    ms, gbs = rmsnorm_bandwidth(dev)
    results["rmsnorm_16384x5120"] = dict(ms=ms, GBps=gbs, of_3350=gbs / 3350)
    print(f"mer_rmsnorm 16384 x 5120 (fp32 in, fp16 out): {ms:.3f} ms, {gbs:.0f} GB/s = {gbs / 3350:.2f} of 3.35 TB/s")
    for shape in a.shapes.split(","):
        s = SHAPES[shape]
        sd = random_weights(s, a.seed + 7, dev)
        ref_ids = ids[:a.ref_sentences]
        which, ref_dt = reference_loop(s, sd, ref_ids, dev)
        ref_tok = sum(len(x) for x in ref_ids)
        if "family" in s:
            ops = LD.CudaOps(dev)
            conv1d = s["family"] == "gpt2"   # as load_ln_decoder_weights lays GPT-2's Conv1D weights out
            net = LD.LnDecoderNet({LD._strip(k, s["family"]): (v.T if conv1d and k.endswith(LD.GPT2_CONV1D) else v)
                                   for k, v in sd.items()}, ops, s["family"], s["layers"], s["heads"], s["eps"],
                                  MAX_POS[s["family"]])
            if s["family"] == "falcon":   # q | one k | one v, dense, the two FFN matrices
                linear_flops = s["hidden"] * (s["hidden"] + 128) + s["hidden"] ** 2 + 2 * s["hidden"] * s["ffn"]
            else:
                linear_flops = 4 * s["hidden"] ** 2 + 2 * s["hidden"] * s["ffn"]
        else:
            ops = LT.CudaOps(dev)
            net = LT.LlamaNet(sd, ops, s["layers"], s["heads"], s["eps"], 10000.0, 4096)
            linear_flops = 4 * s["hidden"] ** 2 + 3 * s["hidden"] * s["ffn"]
        del sd
        with torch.no_grad():
            run_packed(net, ids, a.tokens)                      # warm-up: every shape of the timed window
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                run_packed(net, ids, a.tokens)
            e1.record()
            torch.cuda.synchronize()
            dt = e0.elapsed_time(e1) / 1e3 / a.steps
            ops.timing = []                                     # separate pass: per-launch events
            run_packed(net, ids, a.tokens)
            torch.cuda.synchronize()
        shares = {}
        for klass, b, e in ops.timing:
            shares[klass] = shares.get(klass, 0.0) + b.elapsed_time(e)
        ops.timing = None
        tot = sum(shares.values())
        r = dict(packed_sentences_per_s=len(ids) / dt, packed_tokens_per_s=sum(lens) / dt,
                 reference=which, reference_sentences_per_s=len(ref_ids) / ref_dt,
                 reference_tokens_per_s=ref_tok / ref_dt, speedup=(len(ids) / dt) / (len(ref_ids) / ref_dt),
                 shares={k: v / tot for k, v in sorted(shares.items())},
                 tflops=2.0 * sum(lens) * s["layers"] * linear_flops / dt / 1e12)
        results[shape] = r
        print(f"{shape}: packed {r['packed_sentences_per_s']:.1f} sentences/s, {r['packed_tokens_per_s']:.0f} tokens/s "
              f"({r['tflops']:.0f} TFLOP/s in the linears); reference loop ({which}) "
              f"{r['reference_sentences_per_s']:.2f} sentences/s, {r['reference_tokens_per_s']:.0f} tokens/s; "
              f"x{r['speedup']:.1f}" + (" (includes fp16 against the reference's fp32)" if "fp32" in which else ""))
        print(f"{shape}: time shares (per-launch events) " + ", ".join(f"{k} {v:.3f}" for k, v in r["shares"].items()))
        del net, ops
        torch.cuda.empty_cache()
    print(json.dumps(results))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
