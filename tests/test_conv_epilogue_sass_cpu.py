"""Instruction count of conv_tc_kernel's staged epilogue, read from the SASS ptxas makes of csrc/conv_tc.cu (no GPU
needed).

While the two consumer warpgroups run a tile's epilogue no MMA is issued, so every instruction of it adds to every tile.
A full tile takes an epilogue with the layer's flags as compile-time constants and no per-pair row or column checks
(DESIGN.md §4, Epilogue); ragged tiles keep the general path.  In the SASS each staged chunk starts at the wait for its
slot (SYNCS.PHASECHK) and ends at the proxy fence that hands the slot to the TMA store (FENCE.VIEW.ASYNC.S).  A chunk is
64 rows x 64 columns over the warpgroup's 128 threads: 16 output pairs per thread, one STS per pair and plane.  The
general path is the kernel's BN / 64 largest chunks; every other chunk belongs to a full-tile variant and must stay
within the bound below.  Swish chunks also carry expf and the correctly rounded reciprocal of every sigmoid."""
import os
import re
import shutil
import subprocess

import pytest

from object_detection_tracking_b200 import build

MAX_PER_OUTPUT = {False: 20.0, True: 45.0}   # by SWISH; the general path takes ~31 (split) and ~60 (split + swish)
PAIRS_PER_CHUNK = 16


def _tool(name):
    nvcc = build._nvcc()
    path = shutil.which(nvcc) or nvcc
    cand = os.path.join(os.path.dirname(path), name) if os.path.sep in path else name
    return cand if os.path.exists(cand) or shutil.which(cand) else None


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    if _tool("nvcc") is None or _tool("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not found")
    cubin = tmp_path_factory.mktemp("sass") / "conv_tc.cubin"
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", os.path.join(build.CSRC, "conv_tc.cu"), "-o", str(cubin)]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    r = subprocess.run([_tool("cuobjdump"), "-sass", str(cubin)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


def _functions(text):
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def _opcode(ins):
    words = ins.split()
    return words[1] if words[0].startswith("@") else words[0]


def _chunks(ins):
    """(instructions, STS count) of every span from a slot wait to the proxy fence that ends it"""
    out, start = [], None
    for k, t in enumerate(ins):
        op = _opcode(t)
        if op.startswith("SYNCS.PHASECHK"):
            start = k
        elif op == "FENCE.VIEW.ASYNC.S" and start is not None:
            body = ins[start:k + 1]
            out.append((len(body), sum(1 for x in body if _opcode(x).split(".")[0] == "STS")))
            start = None
    return out


def test_full_tile_staged_chunks_are_short(sass):
    funcs = {k: v for k, v in _functions(sass).items() if "conv_tc_kernel" in k}
    assert len(funcs) == 12, list(funcs)
    report, bad = [], []
    for name, ins in sorted(funcs.items()):
        bn, split, acc, swish = re.search(r"conv_tc_kernelILi(\d+)ELb(\d)ELb(\d)ELb(\d)E", name).groups()
        bn, split, swish = int(bn), split == "1", swish == "1"
        planes = 2 if split else 1
        chunks = sorted(_chunks(ins))
        assert chunks, name
        per_output = []
        for n, sts in chunks:
            assert sts == PAIRS_PER_CHUNK * planes, (name, n, sts)
            per_output.append(n / (2 * sts // planes))
        general, fast = per_output[-(bn // 64):], per_output[:-(bn // 64)]
        tag = "BN=%d split=%d acc=%s swish=%d" % (bn, split, acc, swish)
        report.append("%s: general %s, full tile %s" % (tag, ["%.1f" % x for x in general],
                                                         ["%.1f" % x for x in fast]))
        if not fast or max(fast) > MAX_PER_OUTPUT[swish]:
            bad.append(tag)
    assert not bad, "full-tile chunks missing or over %s instructions per output in %s\n%s" % (
        MAX_PER_OUTPUT, bad, "\n".join(report))
