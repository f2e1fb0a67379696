"""Shared harness of the element-by-element GPU tests (the gemm_epilogue, train_bwd, fwd_kernels, text_kernels, sam_kernels,
vit_kernels and amg files): covering designs, per-element bound checks with a worst err/bound report, NaN-sentinel output buffers,
NaN-padded strided operands, and the calling primitives -- the library, stream and pointers, repeat runs that must be bit-identical,
and declined shapes that must write nothing."""
import itertools
import random
import zlib

import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24                 # unit roundoff of fp32
L_ACT = {None: 1.0, "relu": 1.0, "hswish": 1.5, "gelu": 1.13, "sigmoid": 0.25}
EPS_GELU = 3e-7                # es3_gelu_fast: 0.5 |x| * (1.5e-7 erf approximation + a few ulp of MUFU rcp / ex2), per |x|
EPS_SIGMOID = 1e-6             # 1 / (1 + __expf(-x)): __expf is within (2 + 1.16 |x|) ulp; sigmoid' <= 1/4
TAIL = 256                     # sentinel cells past the end of a flat output buffer
_INT = {torch.bfloat16: torch.int16, torch.float32: torch.int32}
WORST: dict = {}               # section -> max err/bound over the current module


def report_worst(title):
    """A module-scoped autouse fixture that prints the worst err/bound of every section the module checked."""
    @pytest.fixture(scope="module", autouse=True)
    def _report_worst():
        WORST.clear()
        yield
        for k in sorted(WORST):
            print(f"\n{title}, section {k}: max err/bound = {WORST[k]:.3g}", end="")
    return _report_worst


def _pairwise(factors: dict, seed: int = 0) -> list:
    """Rows of a strength-2 covering design: every value pair of every two factors appears in some row (greedy)."""
    names = list(factors)
    sizes = [len(factors[n]) for n in names]
    nf = len(names)
    todo = {(i, a, j, b) for i, j in itertools.combinations(range(nf), 2) for a in range(sizes[i]) for b in range(sizes[j])}
    rng = random.Random(seed)
    rows = []

    def key(k, v, m, u):
        return (k, v, m, u) if k < m else (m, u, k, v)

    while todo:
        i, a, j, b = min(todo)
        row = {i: a, j: b}
        for k in range(nf):
            if k in row:
                continue
            gains = [sum(key(k, v, m, u) in todo for m, u in row.items()) for v in range(sizes[k])]
            row[k] = rng.choice([v for v in range(sizes[k]) if gains[v] == max(gains)])
        todo -= {(p, row[p], q, row[q]) for p, q in itertools.combinations(range(nf), 2)}
        rows.append(tuple(factors[names[k]][row[k]] for k in range(nf)))
    return rows


def _bf(t):
    return t.to(torch.bfloat16)


def _gen(cuda, *key):
    return torch.Generator(device=cuda).manual_seed(zlib.crc32(repr(key).encode()))


def _act64(x, act):
    if act is None:
        return x
    return {"relu": F.relu, "hswish": F.hardswish, "gelu": F.gelu, "sigmoid": torch.sigmoid}[act](x)


def _eps_act(x, act):
    if act == "gelu":
        return EPS_GELU * x.abs()
    if act == "sigmoid":
        return EPS_SIGMOID * (1.0 + x.abs())
    return 0.0


def _check(section, got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                   # NaN (a cell never written) is outside any bound
    nbad = int(bad.sum())
    if nbad:
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {nbad} of {err.numel()} elements outside their bound ({int(torch.isnan(got).sum())} unwritten); "
                             f"first at {idx}: got {got[idx].item():.6g}, ref {ref[idx].item():.6g}, bound {bound[idx].item():.3g}")
    WORST[section] = max(WORST.get(section, 0.0), (err / bound).max().item())


def _sentinel(dtype):
    return torch.full((1,), float("nan"), dtype=dtype).view(_INT[dtype]).item()


def _assert_untouched(buf, inside, what):
    bits = buf.view(_INT[buf.dtype])[~inside]
    changed = int((bits != _sentinel(buf.dtype)).sum())
    assert changed == 0, f"{what}: {changed} cells outside the output region were written"


def _flat_out(n, dtype, cuda):
    """A NaN-filled flat buffer of n + TAIL cells; returns (buffer, inside-mask)."""
    buf = torch.full((n + TAIL,), float("nan"), dtype=dtype, device=cuda)
    inside = torch.zeros(n + TAIL, dtype=torch.bool, device=cuda)
    inside[:n] = True
    return buf, inside


def _matrix_out(M, N, dtype, strided, cuda):
    """(buffer, [M, N] view, inside-mask): `strided` puts the view at column 8 of a [M + 2, N + 24] buffer."""
    if not strided:
        buf, inside = _flat_out(M * N, dtype, cuda)
        return buf, buf[:M * N].view(M, N), inside
    buf = torch.full((M + 2, N + 24), float("nan"), dtype=dtype, device=cuda)
    inside = torch.zeros(buf.shape, dtype=torch.bool, device=cuda)
    inside[:M, 8:8 + N] = True
    return buf, buf[:M, 8:8 + N], inside


def _padded(t, strided):
    """`t` itself, or the same values as a column-8 slice of a NaN-padded buffer 16 columns wider (row stride != width)."""
    if not strided:
        return t.contiguous()
    big = torch.full((t.shape[0], t.shape[1] + 16), float("nan"), dtype=t.dtype, device=t.device)
    big[:, 8:8 + t.shape[1]] = t
    return big[:, 8:8 + t.shape[1]]


def _st():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _lib(cuda):
    from efficientsam3_b200 import _lib
    _lib.init(cuda.index or 0)
    return _lib


def _bits_equal(a, b, what):
    a, b = a.contiguous(), b.contiguous()
    if a.dtype in _INT:
        a, b = a.view(_INT[a.dtype]), b.view(_INT[b.dtype])
    assert torch.equal(a, b), what


def _twice(run, buf):
    """run(buffer) on two copies of the prefilled buffer; both must be bit-identical.  Returns the first."""
    a, b = buf.clone(), buf.clone()
    run(a)
    run(b)
    _bits_equal(a, b, "two runs differ")
    return a


def _prefilled(n, cuda, g):
    """A flat fp32 buffer of n + TAIL cells: n random values (an accumulating output's prior contents), then NaN sentinels."""
    buf, inside = _flat_out(n, torch.float32, cuda)
    buf[:n] = torch.randn(n, device=cuda, generator=g)
    return buf, inside


def _declined(lib, name, args, bufs, what):
    """A shape `name` declines: the call raises and every buffer keeps its bits."""
    from efficientsam3_b200._lib import Es3Error
    before = [b.clone() for b in bufs]
    with pytest.raises(Es3Error):
        lib.call(name, *args)
    torch.cuda.synchronize()
    for b, b0 in zip(bufs, before):
        _bits_equal(b, b0, f"{what}: a declined call wrote")


def _qkv(cuda, B, L, heads, kind, g):
    """bf16 qkv rows [B L, 3 C] (head_dim 64): normal, peaked (scores spread by ~100), flat (q = 0) or tied (keys of period 5)."""
    C = 64 * heads
    x = torch.randn(B * L, 3 * C, device=cuda, generator=g) * 1.5
    if kind == "peaked":                                   # scores spread by ~100: near one-hot rows
        x[:, :2 * C] *= 5
    elif kind == "flat":                                   # q = 0: every score 0, p = 1
        x[:, :C] = 0
    elif kind == "tied":                                   # keys repeat with period 5: tied maxima in every row, across KV tiles
        k = x[:, C:2 * C].view(B, L, C)
        x[:, C:2 * C] = k[:, torch.arange(L, device=cuda) % 5].reshape(B * L, C)
    return _bf(x)
