#!/usr/bin/env python
"""Regenerate profiles/sass_summary.md: per-kernel counts of the SASS instructions that prove the NVSwitch / TMA / wgmma
paths, taken from `cuobjdump -sass` of the in-tree libraries (works without a GPU).

    python tools/sass_summary.py            # writes profiles/sass_summary.md
"""
import os
import re
import subprocess
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "mpi_operator_b200", "lib")

COLLECTIVE_COLS = OrderedDict([
    ("LDGMC (multimem.ld_reduce)", re.compile(r"\bLDGMC\b")),
    ("128-bit global stores (multicast VA, peer or local)", re.compile(r"\bSTG\.E\.(\w+\.)*128")),
    ("128-bit global loads (peer, staging or user)", re.compile(r"\bLDG\.E\.(\w+\.)*128")),
    ("UBLKCP (cp.async.bulk, TMA copy engine)", re.compile(r"\bUBLKCP\b")),
    ("SYNCS (mbarrier)", re.compile(r"\bSYNCS\b")),
    ("32-bit flag LD/ST .SYS", re.compile(r"\b(LDG|STG)\.E\.STRONG\.SYS\b|\b(LD|ST)\.E\.STRONG\.SYS\b")),
    ("MEMBAR.*SYS", re.compile(r"\bMEMBAR\.\S*SYS")),
])
GEMM_COLS = OrderedDict([
    ("HGMMA (wgmma.mma_async)", re.compile(r"\bHGMMA\b")),
    ("WARPGROUP.ARRIVE (wgmma.fence)", re.compile(r"\bWARPGROUP\.ARRIVE\b")),
    ("WARPGROUP.DEPBAR (wgmma.wait_group)", re.compile(r"\bWARPGROUP\.DEPBAR\b")),
    ("UTMALDG (TMA tensor load)", re.compile(r"\bUTMALDG\b")),
    ("UTMASTG (TMA tensor store)", re.compile(r"\bUTMASTG\b")),
    ("SYNCS (mbarrier)", re.compile(r"\bSYNCS\b")),
    ("BPT.TRAP (bounded waits)", re.compile(r"\bBPT\.TRAP\b")),
])


def demangle(names):
    try:
        out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
        return dict(zip(names, out))
    except Exception:
        return {n: n for n in names}


def kernels(lib):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    cur, out = None, OrderedDict()
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur is not None and "/*" in line:
            out[cur].append(line)
    return out


def short(name):
    name = re.sub(r"\(.*$", "", name)                     # drop the argument list
    name = name.replace("b200mpi::", "").replace("__nv_bfloat16", "bf16").replace("__half", "f16")
    return re.sub(r"^void ", "", name)


def table(ks, cols, only=None):
    names = demangle(list(ks))
    rows = ["| kernel | instructions | " + " | ".join(cols) + " |", "|---|---|" + "---|" * len(cols)]
    for k, lines in ks.items():
        nm = short(names[k])
        if only and not only(nm):
            continue
        body = "\n".join(lines)
        n_ins = sum(1 for ln in lines if re.match(r"\s+/\*[0-9a-f]{4,6}\*/", ln))
        rows.append(f"| `{nm}` | {n_ins} | " + " | ".join(str(len(rx.findall(body))) for rx in cols.values()) + " |")
    return "\n".join(rows)


def main():
    out = ["# SASS evidence (`cuobjdump -sass`, sm_90a; regenerate with `python tools/sass_summary.py`)", ""]
    lib = os.path.join(LIBDIR, "libb200mpi.so")
    ks = kernels(lib)
    out += ["## `libb200mpi.so`: collective kernels (`csrc/kernels/collectives.cu`, `p2p.cu`)", "",
            table(ks, COLLECTIVE_COLS, only=lambda n: not n.startswith("bn::") and "scale_cast" not in n), "",
            "Reading: every `<..., 1>` (MODE_NVLS) instantiation of the reducing kernels carries `LDGMC` (the switch adds) and no "
            "peer pulls; the `<..., 0>` (MODE_P2P) ones pull with 128-bit loads and push with one 128-bit store per peer instead. `k_pipe` (the "
            "user-pointer pipeline: copy-in / reduce / copy-out CTAs chained by flags) is the only collective with `UBLKCP`: "
            "its staging copies run on the TMA copy engine.", "",
            "## `libb200mpi.so`: fused BatchNorm(+add)+ReLU kernels (`csrc/kernels/bn_act.cu`)", "",
            table(ks, OrderedDict([("128-bit global loads", re.compile(r"\bLDG\.E\.(\w+\.)*128")),
                                   ("128-bit global stores", re.compile(r"\bSTG\.E\.(\w+\.)*128")),
                                   ("SHFL (warp reductions)", re.compile(r"\bSHFL\b")),
                                   ("ATOM/RED", re.compile(r"\b(ATOMG|RED)\b"))]), only=lambda n: n.startswith("bn::")), ""]
    glib = os.path.join(LIBDIR, "libb200mpi_gemm.so")
    if os.path.exists(glib):
        out += ["## `libb200mpi_gemm.so`: wgmma / TMA GEMM with BN statistics (`csrc/kernels/gemm_bnstats.cu`)", "",
                "Numerics: `tests/test_zz_gemm_bnstats_gpu.py`; on by default for eligible 1x1 convolutions.", "",
                table(kernels(glib), GEMM_COLS), ""]
    path = os.path.join(ROOT, "profiles", "sass_summary.md")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write("\n".join(out))
    print(f"wrote {path}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
