"""Throughput of the ELECTRA text-feature path (BertEncoder over mer_bert_forward / mer_bert_forward_projected) at the
published small / base / large shapes and LERT-small, and the achieved bandwidth of the 256-wide LayerNorm.

Packed path: BertEncoder with its default operand format, sentences packed up to --tokens per pass.  Weights are seeded
random fp32 tensors (synthetic.electra_state_dict); sentence lengths are bench_llm_text.py's seeded draws (MER2023-like),
capped at 512 tokens.  Times come from CUDA events around --steps passes over all sentences after a warm-up pass over the
same batches; every step is timed on its own so that the spread is reported next to the median.  LayerNorm: the
post-LN stack's form at 256 columns (fp32 out + split copy, the MER_LN_ACC_ADD readout form), algorithmic bytes (fp32 row
in, each output row, the accumulator read and written) over the median event time of 200 launches.  The card's name and
power limit are read in the same run.

    python scripts/bench_electra_text.py [--shapes chinese-electra-180g-small,...] [--sentences 2048]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_llm_text import card, packed_batches, sentence_lengths  # noqa: E402

from mertools_b200 import _lib as L  # noqa: E402
from mertools_b200 import synthetic as S  # noqa: E402
from mertools_b200.encoders import BertEncoder  # noqa: E402


def layernorm_bandwidth(dev, rows, dim=256, reps=200):
    x = torch.randn(rows, dim, device=dev)
    g, b = torch.ones(dim, device=dev), torch.zeros(dim, device=dev)
    y, ys, acc = torch.empty_like(x), torch.empty(rows, dim, dtype=torch.float16, device=dev), torch.zeros_like(x)
    forms = {"fp32 + fp16 copy, acc add": (ys, acc, L.MER_LN_SPLIT_F16 | L.MER_LN_ACC_ADD, 4 + 4 + 2 + 8),
             "fp32 + split bf16 copy": (torch.empty_like(x), None, 0, 4 + 4 + 4),
             "fp32 only": (None, None, 0, 4 + 4)}
    out = {}
    for name, (second, a, fl, bpe) in forms.items():
        def launch():
            L.check(L.lib().mer_layernorm(L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(y), L.ptr(second), L.ptr(a), rows, dim,
                                          1e-12, fl, L.stream_ptr()))
        for _ in range(10):
            launch()
        ts = []
        for _ in range(reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 1e3)
        t = float(np.median(ts))
        gbs = rows * dim * bpe / t / 1e9
        out[name] = dict(rows=rows, bytes_per_element=bpe, median_us=t * 1e6, p10_us=float(np.percentile(ts, 10)) * 1e6,
                         p90_us=float(np.percentile(ts, 90)) * 1e6, achieved_GBps=gbs, share_of_3350_GBps=gbs / 3350)
        print(f"LayerNorm 256 x {rows} rows, {name}: {t * 1e6:.1f} us median, {gbs:.0f} GB/s "
              f"({gbs / 3350:.2f} of the 3.35 TB/s data-sheet HBM3 bandwidth)")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default=",".join(S.ELECTRA_PUBLISHED_CFGS))
    ap.add_argument("--sentences", type=int, default=2048)
    ap.add_argument("--tokens", type=int, default=16384, help="tokens per packed pass")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="JSON file for the results")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power.limit, clocks.max.sm: {power}")
    lens = [min(n, 512) for n in sentence_lengths(a.sentences, a.seed)]
    results = dict(card=name, power=power, lengths=dict(n=len(lens), mean=float(np.mean(lens)), total=int(sum(lens))))
    for shape in a.shapes.split(","):
        kw = S.ELECTRA_PUBLISHED_CFGS[shape]
        ekw = dict(kw, embedding_size=kw["hidden_size"]) if "lert" in shape else kw
        rng = np.random.default_rng(a.seed + 1)
        ids = [np.concatenate([[2], rng.integers(10, kw["vocab_size"], n - 2), [3]]).astype(np.int64) for n in lens]
        enc = BertEncoder(S.electra_state_dict(ekw, seed=a.seed + 7), device=dev, ln_eps=kw["layer_norm_eps"])
        batches = list(packed_batches(ids, a.tokens))

        def run():
            for batch in batches:
                enc.forward(batch, start=1, end=-1)
        run()                                               # warm-up: every shape of the timed window
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / 1e3)
        dt = float(np.median(ts))
        r = dict(precision=enc.precision, hidden=enc.hidden, embedding=enc.emb_dim, layers=enc.n_layers,
                 sentences_per_s=len(ids) / dt, tokens_per_s=sum(lens) / dt,
                 step_s_median=dt, step_s_min=float(min(ts)), step_s_max=float(max(ts)))
        results[shape] = r
        print(f"{shape} ({r['precision']}, E {enc.emb_dim} / H {enc.hidden} x {enc.n_layers}): "
              f"{r['sentences_per_s']:.0f} sentences/s ({r['tokens_per_s']:.0f} tokens/s); step "
              f"{dt * 1e3:.1f} ms median, {min(ts) * 1e3:.1f}-{max(ts) * 1e3:.1f} ms over {a.steps}")
        del enc
        torch.cuda.empty_cache()
    results["layernorm_256"] = layernorm_bandwidth(dev, a.tokens * 8)
    print(json.dumps(results))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
