"""The wgmma 1x1-convolution GEMM (csrc/kernels/gemm_bnstats.cu) bit for bit against the float64 oracle of gemm_oracle.py.

Entry points: the training forward ``b200mpi_gemm_bnstats`` (tile widths 128 and 64) and the dgrad
``b200mpi_gemm_dgrad_res`` with and without the BN-backward partials of the layer below (``Xb``). Every shape runs the three
operand families of the oracle: E (``Y`` / ``dX`` bit-exact), S (partial rows bit-exact, also through ``gemm_bnstats_raw``)
and R (within one rounding plus ``2^-20 sum |terms|``; partial rows within ``1e-5 sum |terms|``). On every case:

* ``Y`` / ``dX`` have 128 NaN rows past M that must stay NaN; the partials buffer is NaN-filled, rows ``>= parts`` must stay
  NaN and rows ``< parts`` must be finite; ``parts`` follows the planning rule;
* the operands have 128 poisoned rows past M (NaN for bf16, 0xFF for masks); a second call with those rows zeroed gives the
  same bits;
* dgrad: ``R`` = NaN / ±Inf wherever its mask bit is 0 leaves ``dX`` unchanged, and ``dX`` with the partials equals ``dX``
  without them.

The shapes cover both tile widths with several column blocks, 1 to 64 k-blocks (either side of the 4-stage forward ring and
the 3-stage ring of the partials), ``groups = 1`` (N = 8384), ``num_m < groups``, one partial row past the last full
m-group, ResNet-101's stride-1 1x1 forward shapes and linked-conv1 dgrad shapes at batch 64 and 256, and one case with
``M * N >= 2^31``. Several shapes share one subprocess; each case runs in a subprocess so that a trap in the kernel cannot
poison the CUDA context of the test session, and the file sorts after the other GEMM files. B200MPI_SKIP_GEMM_TESTS=1
skips it. Each case prints the largest family-R ``err / bound`` it saw."""
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("B200MPI_SKIP_GEMM_TESTS") == "1", reason="B200MPI_SKIP_GEMM_TESTS=1")]

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))

# ResNet-101's stride-1 1x1 convolutions as (H*W, K = Cin, N = Cout), and its linked conv1 dgrads as (H*W, N = Cin,
# K = width): M = batch * H * W
RESNET_FWD = [(56 * 56, 64, 64), (56 * 56, 64, 256), (56 * 56, 256, 64), (28 * 28, 256, 128), (28 * 28, 128, 512),
              (28 * 28, 512, 128), (14 * 14, 512, 256), (14 * 14, 256, 1024), (14 * 14, 1024, 256), (7 * 7, 1024, 512),
              (7 * 7, 512, 2048), (7 * 7, 2048, 512)]
RESNET_DGRAD = [(56 * 56, 256, 64), (28 * 28, 512, 128), (14 * 14, 1024, 256), (7 * 7, 2048, 512)]

# (M, N, K). 5633 = 128 * 44 + 1, 16897 = 128 * 132 + 1, 257 = 128 * 2 + 1: one row past the last full m-group for N = 192,
# 64 / 128 and 8448
FWD_SHAPES = {
    "bn64": [(128, 64, 64), (129, 192, 192), (255, 320, 320), (256, 192, 2048), (1000, 8384, 128), (5633, 192, 256),
             (1000, 64, 4096), (16897, 64, 64), (200704, 320, 64)],
    "bn128": [(128, 128, 128), (256, 128, 64), (1000, 128, 256), (4096, 256, 64), (12544, 512, 128), (50176, 2048, 512),
              (129, 8448, 4096), (257, 8448, 320), (16897, 128, 192), (255, 2048, 320), (1000, 256, 2048)],
    "resnet_b64": [(64 * hw, n, k) for hw, k, n in RESNET_FWD],
    "resnet_b256": [(256 * hw, n, k) for hw, k, n in RESNET_FWD],
}
DGRAD_SHAPES = {
    "edges": [(128, 128, 64), (129, 384, 192), (255, 2048, 320), (256, 8448, 4096), (257, 8448, 128), (1000, 128, 256),
              (980, 1024, 256), (4096, 256, 64), (12544, 512, 128), (16897, 128, 2048), (1000, 384, 64)],
    "resnet_b64": [(64 * hw, n, k) for hw, n, k in RESNET_DGRAD],
    "resnet_b256": [(256 * hw, n, k) for hw, n, k in RESNET_DGRAD],
}

PRELUDE = r"""
import ctypes as C, sys, torch
sys.path.insert(0, {repo!r}); sys.path.insert(0, {tests!r})
import gemm_oracle as go
from mpi_operator_b200.ops import gemm_bnstats
L = gemm_bnstats.lib()
dev = torch.device("cuda")
SMS = torch.cuda.get_device_properties(dev).multi_processor_count
STREAM = torch.cuda.current_stream().cuda_stream
NAN = float("nan")
BIG = 1 << 28                      # outputs with more elements are re-checked against the oracle instead of cloned
worst = {{}}

def note(key, v):
    worst[key] = max(worst.get(key, 0.0), v)

def make(fam, M, N, K, seed, residual=False):
    if fam == "E":
        return go.family_e(M, N, K, x_full=seed % 2 == 0, residual=residual, seed=seed, device=dev)
    if fam == "S":
        return go.family_s(M, N, K, residual=residual, scale=not residual, seed=seed, device=dev)
    return go.family_r(M, N, K, residual=residual, seed=seed, device=dev)

def into_guarded(t, rows):
    buf, view = go.guarded(rows, t.shape[1], t.dtype, dev)
    view.copy_(t)
    return buf, view

def nan_out(M, N):
    return torch.full((M + go.GUARD_ROWS, N), NAN, dtype=torch.bfloat16, device=dev)

def nan_partials(N):
    return torch.full((int(L.b200mpi_gemm_bnstats_partial_floats(N)),), NAN, dtype=torch.float32, device=dev)

def check_guards(what, out, pbuf, M, N, parts):
    assert bool(out[M:].isnan().all()), f"{{what}}: rows of the output past M were written"
    if pbuf is not None:
        P = pbuf.view(go.MAX_PARTS, N, 2)
        assert bool(P[parts:].isnan().all()), f"{{what}}: partial rows at index >= parts={{parts}} were written"
        assert bool(P[:parts].isfinite().all()), f"{{what}}: partial rows below parts={{parts}} are not all finite"

def same_bits(a, b, what):
    go.assert_bits(a, b, what)
"""

FWD_CASE = r"""
def run(x, w, M, N, K):
    y, pbuf, parts = nan_out(M, N), nan_partials(N), C.c_int(-1)
    rc = L.b200mpi_gemm_bnstats(x.data_ptr(), w.data_ptr(), y.data_ptr(), pbuf.data_ptr(), C.byref(parts), M, N, K, STREAM)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return y, pbuf, parts.value

def case(M, N, K, fam, seed):
    what = f"forward M={{M}} N={{N}} K={{K}} family {{fam}}"
    op = make(fam, M, N, K, seed)
    xbuf, op.x = into_guarded(op.x, M)
    y, pbuf, parts = run(op.x, op.w, M, N, K)
    assert parts == go.plan_parts(M, N, SMS), (what, "parts", parts, go.plan_parts(M, N, SMS))
    check_guards(what, y, pbuf, M, N, parts)
    note(("b200mpi_gemm_bnstats Y", fam), go.check_y(y[:M], op, what))
    P = pbuf.view(go.MAX_PARTS, N, 2)[:parts]
    sh, mg, pl = go.stats_ref(y[:M], parts)
    if fam == "S":
        unit = torch.exp2(op.eb.double())[:, None].repeat(1, 2)
        unit[:, 1] = unit[:, 0] ** 2
        go.check_exact_sums(sh, mg, unit, what)
        go.check_rows(P, sh, mg, True, what + " shifted partial rows")
    if fam == "S" and y.numel() <= BIG:
        y2, p2, parts2 = gemm_bnstats.gemm_bnstats_raw(op.x, op.w)
        torch.cuda.synchronize()
        assert parts2 == parts
        same_bits(y2, y[:M], what + " gemm_bnstats_raw Y")
        same_bits(p2, pl.float(), what + " gemm_bnstats_raw plain partial rows")
        del y2, p2
    if fam != "S":
        note(("b200mpi_gemm_bnstats partials", fam), go.check_rows(P, sh, mg, False, what))
    # the same call with the operand's guard rows zeroed gives the same bits
    keep = y.clone() if y.numel() <= BIG else None
    pkeep = pbuf.clone()
    del y
    go.set_guard(xbuf, M, poison=False)
    y, pbuf, _ = run(op.x, op.w, M, N, K)
    if keep is not None:
        same_bits(y, keep, what + " second call")
    else:
        assert fam != "R"
        go.check_y(y[:M], op, what + " second call")
        check_guards(what, y, None, M, N, parts)
    same_bits(pbuf, pkeep, what + " second call partials")

for i, (M, N, K) in enumerate({shapes}):
    for fam in {families}:
        case(M, N, K, fam, seed=i)
        torch.cuda.empty_cache()
print("WORST", {{f"{{k[0]}} [{{k[1]}}]": round(v, 4) for k, v in worst.items()}})
print("OK")
"""

DGRAD_CASE = r"""
def run(dy, wt, r, mbytes, M, N, K, below=None):
    dx, parts = nan_out(M, N), C.c_int(-1)
    xb = mb = mean = pbuf = None
    if below is not None:
        xb, mb, mean = below
        pbuf = nan_partials(N)
    p = lambda t: t.data_ptr() if t is not None else None
    rc = L.b200mpi_gemm_dgrad_res(dy.data_ptr(), wt.data_ptr(), dx.data_ptr(), r.data_ptr(), mbytes.data_ptr(), p(xb), p(mb),
                                  p(mean), p(pbuf), C.byref(parts), M, N, K, STREAM)
    assert rc == 0, rc
    torch.cuda.synchronize()
    return dx, pbuf, parts.value

def masked_poison(r, mask):
    # NaN, +Inf and -Inf in turn wherever the mask bit is 0
    idx = torch.arange(r.numel(), device=dev).view(r.shape) % 3
    bad = torch.where(idx == 0, NAN, torch.where(idx == 1, float("inf"), float("-inf"))).to(r.dtype)
    return torch.where(mask, r, bad)

def case(M, N, K, fam, seed, mask=None):
    what = f"dgrad M={{M}} N={{N}} K={{K}} family {{fam}}" + (f" mask {{mask[0]}}" if mask is not None else "")
    op = make(fam, M, N, K, seed, residual=True)
    if mask is not None:
        op.mask = mask[1]
    dybuf, dy = into_guarded(op.x, M)
    rbuf, r = into_guarded(op.r, M)
    mbuf, mbytes = into_guarded(go.pack_mask(op.mask), M)
    xb, maskb, mean = go.below_operands(M, N, fam=fam, seed=seed, device=dev)
    xbbuf, xbv = into_guarded(xb, M)
    mbbuf, mbb = into_guarded(go.pack_mask(maskb), M)
    below = (xbv, mbb, mean)

    dx, _, parts0 = run(dy, op.w, r, mbytes, M, N, K)
    plan = go.plan_parts(M, N, SMS)
    assert parts0 == plan, (what, "parts", parts0, plan)
    check_guards(what, dx, None, M, N, plan)
    note(("b200mpi_gemm_dgrad_res dX", fam), go.check_y(dx[:M], op, what))

    # a masked-out residual is never read into dX, even NaN / Inf
    rpbuf, rp = into_guarded(masked_poison(op.r, op.mask), M)
    dxp, _, _ = run(dy, op.w, rp, mbytes, M, N, K)
    same_bits(dxp, dx, what + " with NaN / Inf residual where the mask is 0")
    del dxp, rpbuf, rp

    # with the BN-backward partials: the same dX, partial rows against float64 on the kernel's own dX
    dx2, pbuf, parts = run(dy, op.w, r, mbytes, M, N, K, below)
    assert parts == plan, (what, "parts with Xb", parts, plan)
    check_guards(what + " with Xb", dx2, pbuf, M, N, parts)
    same_bits(dx2, dx, what + " dX with the partials vs without")
    del dx2
    P = pbuf.view(go.MAX_PARTS, N, 2)[:parts]
    rows, mg = go.gst_ref(dx[:M], xbv, maskb, mean, parts)
    if fam == "S":
        assert float(mg[..., 1].max()) < 2 ** 22, (what, "oracle precondition: sum |g| |xb - mean| >= 2^22")
        go.check_exact_sums(rows, mg, torch.tensor([1.0, 0.25], dtype=torch.float64, device=dev), what)
        go.check_rows(P, rows, mg, True, what + " GST partial rows")
    else:
        note(("b200mpi_gemm_dgrad_res partials", fam), go.check_rows(P, rows, mg, False, what + " GST partial rows"))

    # the same calls with every operand's guard rows zeroed give the same bits
    keep = dx.clone() if dx.numel() <= BIG else None
    pkeep = pbuf.clone()
    del dx, pbuf
    for b in (dybuf, rbuf, mbuf, xbbuf, mbbuf):
        go.set_guard(b, M, poison=False)
    dx, pbuf, _ = run(dy, op.w, r, mbytes, M, N, K, below)
    if keep is not None:
        same_bits(dx, keep, what + " second call")
    else:
        assert fam != "R"
        go.check_y(dx[:M], op, what + " second call")
    same_bits(pbuf, pkeep, what + " second call partials")

{body}
print("WORST", {{f"{{k[0]}} [{{k[1]}}]": round(v, 4) for k, v in worst.items()}})
print("OK")
"""

DGRAD_LOOP = r"""
for i, (M, N, K) in enumerate({shapes}):
    for fam in {families}:
        case(M, N, K, fam, seed=i)
        torch.cuda.empty_cache()
"""

MASK_LOOP = r"""
# every mask pattern: all zero, all one, the single-bit bytes 1 << j, random
for i, (M, N, K) in enumerate([(1000, 384, 192), (129, 128, 64)]):
    patterns = [("zero", 0), ("one", 0xFF)] + [(f"1<<{{j}}", 1 << j) for j in range(8)]
    for name, byte in patterns:
        bits = go.unpack_mask(torch.full((M, N // 8), byte, dtype=torch.uint8, device=dev), N)
        case(M, N, K, "E", seed=i, mask=(name, bits))
    case(M, N, K, "E", seed=i + 10)
    case(M, N, K, "S", seed=i + 10)
"""

SUPPORT_CASE = r"""
OK_CODE, INVALID, UNSUPPORTED = 0, -1, -5
fwd, dgrad = {fwd}, {dgrad}
for M, N, K in fwd:
    assert L.b200mpi_gemm_bnstats_supported(M, N, K) == 1, ("forward shape refused", M, N, K)
for M, N, K in dgrad:
    assert L.b200mpi_gemm_dgrad_res_supported(M, N, K) == 1, ("dgrad shape refused", M, N, K)
assert L.b200mpi_gemm_bnstats_supported((1 << 24) + 37, 128, 64) == 1
refused = [(1000, 8512, 64), (1000, 96, 64), (1000, 128, 32), (127, 128, 64)]
for M, N, K in refused:
    assert L.b200mpi_gemm_bnstats_supported(M, N, K) == 0, ("accepted", M, N, K)
    assert L.b200mpi_gemm_dgrad_res_supported(M, N, K) == 0, ("dgrad accepted", M, N, K)
for N in (64, 192, 320, 8384):
    assert L.b200mpi_gemm_bnstats_supported(1000, N, 64) == 1
    assert L.b200mpi_gemm_dgrad_res_supported(1000, N, 64) == 0, ("dgrad with N % 128 = 64 accepted", N)

def buf(nbytes):
    return torch.zeros(nbytes + 64, dtype=torch.uint8, device=dev)

# the launches agree: refused shapes return UNSUPPORTED and write nothing
M, N, K = 1000, 256, 128
X, W, Y, R, MK, XB, MB = (buf(M * K * 2), buf(N * K * 2), buf(M * N * 2), buf(M * N * 2), buf(M * N // 8), buf(M * N * 2),
                          buf(M * N // 8))
mean = torch.zeros(N, dtype=torch.float32, device=dev)
P = nan_partials(N)
Y.fill_(0xAB)
parts = C.c_int(-7)
def fwd_call(x, w, y, p, m, n, k):
    return L.b200mpi_gemm_bnstats(x, w, y, p, C.byref(parts), m, n, k, STREAM)
def dgrad_call(dy, wt, dx, r, mk, xb, mb, mu, p, m, n, k):
    return L.b200mpi_gemm_dgrad_res(dy, wt, dx, r, mk, xb, mb, mu, p, C.byref(parts), m, n, k, STREAM)
a = lambda t, off=0: t.data_ptr() + off
for m, n, k in [(127, N, K), (M, 96, K), (M, N, 32)]:
    assert fwd_call(a(X), a(W), a(Y), a(P), m, n, k) == UNSUPPORTED
    assert dgrad_call(a(X), a(W), a(Y), a(R), a(MK), a(XB), a(MB), a(mean), a(P), m, n, k) == UNSUPPORTED
assert dgrad_call(a(X), a(W), a(Y), a(R), a(MK), a(XB), a(MB), a(mean), a(P), M, 192, K) == UNSUPPORTED
# a pointer misaligned by 2 bytes is refused, for every operand
for i in range(3):
    ptrs = [a(X), a(W), a(Y)]
    ptrs[i] += 2
    assert fwd_call(*ptrs, a(P), M, N, K) == INVALID, ("forward misaligned operand", i)
for i in range(7):
    ptrs = [a(X), a(W), a(Y), a(R), a(MK), a(XB), a(MB)]
    ptrs[i] += 2
    assert dgrad_call(*ptrs, a(mean), a(P), M, N, K) == INVALID, ("dgrad misaligned operand", i)
# the partials need Xb, maskB, mean_b and the partials buffer together
assert dgrad_call(a(X), a(W), a(Y), a(R), a(MK), a(XB), None, a(mean), a(P), M, N, K) == INVALID
assert dgrad_call(a(X), a(W), a(Y), a(R), a(MK), a(XB), a(MB), None, a(P), M, N, K) == INVALID
assert dgrad_call(a(X), a(W), a(Y), a(R), a(MK), a(XB), a(MB), a(mean), None, M, N, K) == INVALID
torch.cuda.synchronize()
assert bool((Y == 0xAB).all()) and bool(P.isnan().all()), "a refused call wrote its output"
print("OK")
"""

HUGE_CASE = r"""
M, N, K = (1 << 24) + 37, 128, 64
assert M * N >= 1 << 31
free, _ = torch.cuda.mem_get_info()
if free < 10 * 2 ** 30:
    print("SKIP free memory", free / 2 ** 30, "GiB")
else:
    case(M, N, K, "S", seed=0)
    print("OK")
"""


def _run(src, timeout=900):
    r = subprocess.run([sys.executable, "-c", src], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and ("OK" in r.stdout or "SKIP" in r.stdout), r.stdout[-3000:] + r.stderr[-3000:]
    for line in r.stdout.splitlines():
        if line.startswith(("WORST", "SKIP")):
            print(line)
    if "SKIP" in r.stdout:
        pytest.skip(r.stdout.strip().splitlines()[-1])
    return r.stdout


def _src(template, **fmt):
    return PRELUDE.format(repo=REPO, tests=TESTS) + template.format(**fmt)


@pytest.mark.parametrize("group", list(FWD_SHAPES))
def test_forward_matches_oracle(group):
    _run(_src(FWD_CASE, shapes=FWD_SHAPES[group], families=["E", "S", "R"]))


@pytest.mark.parametrize("group", list(DGRAD_SHAPES))
def test_dgrad_matches_oracle(group):
    body = DGRAD_LOOP.format(shapes=DGRAD_SHAPES[group], families=["E", "S", "R"])
    _run(_src(DGRAD_CASE, body=body))


def test_dgrad_mask_patterns_and_masked_out_nan_residual():
    _run(_src(DGRAD_CASE, body=MASK_LOOP.replace("{{", "{").replace("}}", "}")))


def test_supported_shapes_and_argument_checks():
    fwd = sorted({s for v in FWD_SHAPES.values() for s in v})
    dgrad = sorted({s for v in DGRAD_SHAPES.values() for s in v})
    _run(_src(SUPPORT_CASE, fwd=fwd, dgrad=dgrad))


def test_forward_beyond_2g_elements():
    _run(_src(FWD_CASE.split("for i, (M, N, K)")[0] + HUGE_CASE))
