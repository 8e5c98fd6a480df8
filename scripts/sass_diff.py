#!/usr/bin/env python
"""SASS-level diff of the kernels in mertools_b200/csrc/*.cu between a git revision and the working tree (no GPU
needed: nvcc cross-compiles sm_90a cubins, cuobjdump lists them).  Used at the end of round 1 to show that the default
kernels were untouched by the work done after the last GPU run:

    python scripts/sass_diff.py a914b7b attention_f16 attention_tc hubert_frontend helpers rowwise gemm

For every kernel of the old revision: identical instruction stream in the new build, or the opcode counts that were
removed / added.  Scratch files go under gpurun_out/sasscmp/ (git-ignored).
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRATCH = os.path.join(ROOT, "gpurun_out", "sasscmp")
NVCC = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-DMER_BUILD=1"]


def kernels(cubin):
    out = subprocess.run(["cuobjdump", "-sass", cubin], capture_output=True, text=True, check=True).stdout
    ks, cur = collections.OrderedDict(), None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", m.group(1))   # the anonymous-namespace hash differs per build
            ks[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur:
            ks[cur].append(re.sub(r"\s+", " ", m.group(1)))
    return ks


def build(tag, rev, names):
    src = os.path.join(SCRATCH, tag, "m", "csrc")
    inc = os.path.join(SCRATCH, tag, "include")
    os.makedirs(src, exist_ok=True)
    os.makedirs(inc, exist_ok=True)
    files = [f"mertools_b200/csrc/{n}.cu" for n in names] + ["mertools_b200/csrc/mer_common.cuh", "mertools_b200/csrc/mer_kernels.h"]
    for rel, dst in [(f, src) for f in files] + [("include/mer_b200.h", inc)]:
        if rev is None:
            data = open(os.path.join(ROOT, rel), "rb").read()
        else:
            data = subprocess.run(["git", "-C", ROOT, "show", f"{rev}:{rel}"], capture_output=True, check=True).stdout
        open(os.path.join(dst, os.path.basename(rel)), "wb").write(data)
    procs = [subprocess.Popen(NVCC + ["-cubin", "-o", f"{n}.cubin", f"{n}.cu"], cwd=src) for n in names]
    assert all(p.wait() == 0 for p in procs), "nvcc failed"
    return {n: kernels(os.path.join(src, f"{n}.cubin")) for n in names}


def opcodes(stream):
    return collections.Counter((x.split()[1] if x.startswith("@") else x.split()[0]) for x in stream)


def main():
    rev, names = sys.argv[1], sys.argv[2:]
    old, new = build("old", rev, names), build("new", None, names)
    for n in names:
        same = 0
        for k, v in old[n].items():
            cand = new[n].get(k)
            if cand is None:   # templates added since: look for the same stream under another name
                cand = next((s for s in new[n].values() if s == v), None)
            if cand == v:
                same += 1
            elif cand is None:   # signature changed (new parameter / template): closest kernel with the same base name
                base = re.search(r"\d+([A-Za-z_0-9]+_kernel)", k)
                near = [(kk, s) for kk, s in new[n].items() if base and base.group(1) in kk]
                if not near:
                    print(f"{n}: {k[:100]}: no counterpart in the new build")
                    continue
                kk, s = min(near, key=lambda t: sum(((opcodes(t[1]) - opcodes(v)) + (opcodes(v) - opcodes(t[1]))).values()))
                rem, add = opcodes(v) - opcodes(s), opcodes(s) - opcodes(v)
                print(f"{n}: {base.group(1)}: signature changed; {len(v)} -> {len(s)} instructions; removed {dict(rem)}; "
                      f"added {dict(add.most_common(8))}")
            else:
                rem, add = opcodes(v) - opcodes(cand), opcodes(cand) - opcodes(v)
                print(f"{n}: {k[:100]}: {len(v)} -> {len(cand)} instructions; removed {dict(rem)}; added {dict(add.most_common(8))}")
        print(f"{n}: {same} of {len(old[n])} kernels of {rev} have identical SASS ({len(new[n])} kernels now)")


if __name__ == "__main__":
    main()
