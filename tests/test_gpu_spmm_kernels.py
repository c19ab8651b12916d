"""The graph propagation kernels of csrc/spmm.cu called directly through the C-ABI and compared with float64:
``b200_spmm_csr`` (K6, the CSR SpMM of LightGCN and NGCF), ``b200_ngcf_combine`` and ``b200_mul_elementwise``.

The long-row plan is built here with numpy (tests/_spmm_plan.py), not with ``SpmmGraph``.

Exact-arithmetic cases: values k/8 with integer k in [-4, 4] and embeddings that are integers in [-16, 16]. Every
partial sum is then a multiple of 1/8, and ``_exact_inputs`` asserts that 8 times each row's sum of |v e| (plus the
base the epilogue adds) stays below 2^24, so every partial sum is exact in any order. The kernel must then equal the
float64 product exactly: a lost, doubled or misrouted non-zero fails, whichever path the row takes. Random-float
cases are held to a per-element summation bound instead of one tolerance for the whole matrix."""
import numpy as np
import pytest
from scipy import sparse as sp

from _spmm_plan import long_row_plan

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
VEC4_WIDTHS = [4, 12, 20, 32, 36, 64, 100, 128]          # vec4 LPR 4, 4, 8, 8, 16, 16, 32, 32
SCALAR_WIDTHS = [1, 3, 5, 10, 17, 132, 255, 256]          # lpr 1, 4, 8, 16, 32; T = 5, 8, 8


def _lanes(d):
    """Lanes per row of the branch b200_spmm_csr takes for width d with aligned operands."""
    if d % 4 == 0 and d <= 128:
        q = d // 4
        return 4 if q <= 4 else 8 if q <= 8 else 16 if q <= 16 else 32
    lpr = 1
    while lpr < d and lpr < 32:
        lpr *= 2
    return lpr


def _torch():
    import torch

    return torch


def _dev(a):
    return _torch().as_tensor(np.ascontiguousarray(a)).cuda()


def _strided(rows, d, ld, offset=0, fill=np.nan):
    """A [rows, d] device view with row stride ``ld`` starting ``offset`` floats into a fresh allocation whose other
    entries hold ``fill`` (sentinels the kernel must not touch)."""
    torch = _torch()
    base = torch.full((rows * ld + offset + 4,), float(fill), dtype=torch.float32, device="cuda")
    return base, base[offset: offset + rows * ld].view(rows, ld)[:, :d]


class Graph:
    def __init__(self, deg, n_e, rng, exact=True, col=None):
        self.deg = np.asarray(deg, dtype=np.int64)
        self.n_rows, self.n_e = len(self.deg), int(n_e)
        self.indptr = np.zeros(self.n_rows + 1, dtype=np.int64)
        self.indptr[1:] = np.cumsum(self.deg)
        nnz = int(self.indptr[-1])
        self.col = (rng.integers(0, n_e, nnz) if col is None else np.asarray(col)).astype(np.int32)
        if exact:
            self.val = (rng.integers(-4, 5, nnz) / 8.0).astype(np.float32)
        else:
            self.val = rng.standard_normal(nnz).astype(np.float32)
        self.rows = np.repeat(np.arange(self.n_rows), self.deg)

    def product64(self, E, absolute=False):
        """L @ E (or |L| @ |E|) in float64; duplicate columns add up."""
        v = np.abs(self.val) if absolute else self.val
        E = np.abs(E) if absolute else E
        L = sp.coo_matrix((v.astype(np.float64), (self.rows, self.col)), shape=(self.n_rows, self.n_e)).tocsr()
        return L @ np.asarray(E, dtype=np.float64)


def _exact_inputs(g, E, base=None):
    assert np.all(np.abs(E) <= 16) and np.array_equal(E, np.round(E))
    assert np.array_equal(g.val * 8, np.round(g.val * 8)) and np.all(np.abs(g.val) <= 0.5)
    bound = g.product64(E, absolute=True).max(initial=0.0)
    if base is not None:
        bound += np.abs(base).max(initial=0.0)
    assert 8 * bound < 2 ** 24, "inputs too large for exact float32 partial sums"


def spmm(g, E, out=None, acc=None, acc_init=0, final_div=0.0, plan=True, null_col_val=False):
    """b200_spmm_csr on device views (unit column stride); returns the C-ABI's return code."""
    from librecommender_b200 import _lib

    torch = _torch()
    d = int(E.shape[1])
    for t in (E, out, acc):
        assert t is None or t.stride(1) == 1
    lib = _lib.lib
    p = long_row_plan(g.indptr, lib.b200_spmm_long_row_threshold(), lib.b200_spmm_chunk())
    indptr = _dev(g.indptr)
    if null_col_val:
        assert g.indptr[-1] == 0
        col = val = None
    else:
        col, val = _dev(g.col), _dev(g.val)
    lr = lcp = cr = ck = part = None
    if p["n_long"] and plan:
        lr, lcp, cr, ck = (_dev(p[k]) for k in ("long_rows", "long_chunk_ptr", "chunk_row", "chunk_k"))
        part = torch.empty(p["n_chunks"] * d, dtype=torch.float32, device="cuda")
    rc = lib.b200_spmm_csr(_lib.ptr(indptr), _lib.ptr(col), _lib.ptr(val), g.n_rows, _lib.ptr(E), E.stride(0), d,
                           _lib.ptr(out), out.stride(0) if out is not None else 0,
                           _lib.ptr(acc), acc.stride(0) if acc is not None else 0, acc_init, final_div,
                           _lib.ptr(lr), _lib.ptr(lcp), p["n_long"], _lib.ptr(cr), _lib.ptr(ck), p["n_chunks"],
                           _lib.ptr(part), _lib.current_stream())
    torch.cuda.synchronize()
    return rc


def _run_ok(*a, **k):
    from librecommender_b200 import _lib

    _lib.check(spmm(*a, **k))


def _int_matrix(rng, rows, d):
    return rng.integers(-16, 17, (rows, d)).astype(np.float32)


def _check_out_and_acc(g, E, d):
    """One call writing out and acc (acc_init = 1, final_div = 4); both must equal the float64 values exactly."""
    ref = g.product64(E)
    _exact_inputs(g, E, base=E[: g.n_rows])
    Ed = _dev(E)
    out, acc = _strided(g.n_rows, d, d)[1], _strided(g.n_rows, d, d)[1]
    _run_ok(g, Ed, out=out, acc=acc, acc_init=1, final_div=4.0)
    np.testing.assert_array_equal(out.cpu().numpy(), ref.astype(np.float32))
    want = (E[: g.n_rows].astype(np.float64) + ref).astype(np.float32) / np.float32(4)
    np.testing.assert_array_equal(acc.cpu().numpy(), want)
    return out, acc


def torch_isnan_all(t):
    return _torch().isnan(t).all()


def _mixed_degrees(rng, d, n_short=300):
    """Short rows of every unroll tail around this width's lanes per row, long rows at the first and last row and
    in the middle (1025: a second chunk of one non-zero; 2049: three chunks)."""
    lpr = _lanes(d)
    tails = [0, 1, 3, 4, 5, 8, 9, lpr - 1, lpr, lpr + 1, 2 * lpr + 1, 1023, 1024]
    deg = rng.integers(0, 40, n_short)
    deg[1: 1 + len(tails)] = tails
    deg[0] = 1025
    deg[n_short // 2] = 2049
    deg[-1] = 1500
    return deg


# ---- widths: every dispatch branch ----------------------------------------------------------------------------------

@pytest.mark.parametrize("d", VEC4_WIDTHS + SCALAR_WIDTHS)
def test_spmm_exact_every_width(d):
    """Each width's branch (vec4 LPR 4 / 8 / 16 / 32; scalar lpr 1 / 4 / 8 / 16 / 32 and T = 5 / 8), its short-row
    kernel and its long-row chunk kernel plus the ordered reduction, out and acc written in one call."""
    rng = np.random.default_rng(100 + d)
    g = Graph(_mixed_degrees(rng, d), 320, rng)
    _check_out_and_acc(g, _int_matrix(rng, 320, d), d)


def _misaligned_runs(how, g, E, d):
    """Device views that turn the vec4 path off in one way each; returns (E, out, acc) views."""
    n = g.n_rows
    if how == "E_offset":                      # E starts 4 bytes past a 16-byte boundary, ld_e a multiple of 4
        _, Ev = _strided(E.shape[0], d, d + 4, offset=1, fill=0.0)
        Ev.copy_(_dev(E))
        assert Ev.data_ptr() % 16 == 4 and Ev.stride(0) % 4 == 0
        return Ev, _strided(n, d, d)[1], _strided(n, d, d)[1]
    if how == "ld_e":                          # aligned E, ld_e = d + 1
        _, Ev = _strided(E.shape[0], d, d + 1, fill=0.0)
        Ev.copy_(_dev(E))
        assert Ev.data_ptr() % 16 == 0 and Ev.stride(0) == d + 1
        return Ev, _strided(n, d, d)[1], _strided(n, d, d)[1]
    if how == "out_offset":
        out = _strided(n, d, d + 4, offset=1)[1]
        assert out.data_ptr() % 16 == 4
        return _dev(E), out, _strided(n, d, d)[1]
    assert how == "acc_offset"
    acc = _strided(n, d, d + 4, offset=3)[1]
    assert acc.data_ptr() % 16 == 12
    return _dev(E), _strided(n, d, d)[1], acc


@pytest.mark.parametrize("how", ["E_offset", "ld_e", "out_offset", "acc_offset"])
@pytest.mark.parametrize("d", VEC4_WIDTHS)
def test_spmm_vec4_forced_off_matches_aligned(d, how):
    """A vec4 width whose E, out or acc breaks the 16-byte preconditions takes the scalar kernels (short rows and the
    long-row chunk kernel): its results must equal the aligned vec4 run bit for bit, and the float64 product."""
    rng = np.random.default_rng(200 + d)
    g = Graph(_mixed_degrees(rng, d, n_short=120), 130, rng)
    E = _int_matrix(rng, 130, d)
    out_a, acc_a = _check_out_and_acc(g, E, d)
    Ev, out, acc = _misaligned_runs(how, g, E, d)
    _run_ok(g, Ev, out=out, acc=acc, acc_init=1, final_div=4.0)
    assert np.array_equal(out.cpu().numpy().view(np.int32), out_a.cpu().numpy().view(np.int32))
    assert np.array_equal(acc.cpu().numpy().view(np.int32), acc_a.cpu().numpy().view(np.int32))


# ---- row structure ----------------------------------------------------------------------------------------------

def _structure(name, lpr, rng):
    """(degrees, column override or None, number of E rows)."""
    n_e = 400
    if name == "unroll_tails":
        return np.array([0, 1, 3, 4, 5, 8, 9, 0, 2, 7, lpr - 1, lpr, lpr + 1, 0, 0, 33]), None, n_e
    if name == "threshold_edge":           # the last short row and a long row whose second chunk has 1 nnz
        return np.array([1023, 1024, 1025, 3, 0, 1024]), None, n_e
    if name == "many_chunks":              # 2, 3, 8 (one chunk per reduce warp) and 17 chunks (the second
        return np.array([2048, 5, 2049, 8 * 1024, 0, 16 * 1024 + 1]), None, n_e   # accumulator wraps)
    if name == "forty_chunks":
        return np.array([7, 40 * 1024 + 17, 2]), None, n_e
    if name == "long_rows_in_sub_warp_group":   # row 0, rows 8q + j next to short rows, last row
        deg = rng.integers(0, 12, 43)
        deg[[0, 19, 20, 42]] = [1100, 2500, 1030, 1200]
        return deg, None, n_e
    if name == "duplicate_columns":
        deg = np.array([5, 33, 1500, 2, 4100])
        return deg, rng.choice([3, 3, 3, 11, 399], int(deg.sum())).astype(np.int32), n_e
    if name == "last_row_columns":
        deg = np.array([1, 6, 1200, 40, 0, 9])
        col = rng.integers(0, n_e, int(deg.sum()))
        col[::2] = n_e - 1
        return deg, col, n_e
    if name == "single_short_row":
        return np.array([7]), None, 5
    if name == "single_long_row":
        return np.array([3001]), None, 64
    assert name == "ragged_row_count"      # 8 * 13 + 5 rows: not a multiple of any rows-per-warp above 1
    return rng.integers(0, 40, 8 * 13 + 5), None, n_e


STRUCTURES = ["unroll_tails", "threshold_edge", "many_chunks", "forty_chunks", "long_rows_in_sub_warp_group",
              "duplicate_columns", "last_row_columns", "single_short_row", "single_long_row", "ragged_row_count"]


@pytest.mark.parametrize("d", [4, 36, 3, 132])
@pytest.mark.parametrize("structure", STRUCTURES)
def test_spmm_exact_row_structure(structure, d):
    """Row shapes where gathers, unroll tails, chunk boundaries and the reduce kernel's warp assignment go wrong, on
    vec4 LPR 4 / LPR 16 and scalar lpr 4 / T = 5 (each with its own long-row chunk kernel)."""
    rng = np.random.default_rng(500 + 10 * STRUCTURES.index(structure) + d)
    deg, col, n_e = _structure(structure, _lanes(d), rng)
    n_e = max(n_e, len(deg))              # acc_init = 1 reads E's row r
    g = Graph(deg, n_e, rng, col=col)
    _check_out_and_acc(g, _int_matrix(rng, n_e, d), d)


# ---- epilogue modes ---------------------------------------------------------------------------------------------

EPILOGUES = ["out", "acc_init", "both", "block_acc_fewer_E_rows", "block_both_more_E_rows", "acc_init_div3",
             "block_div3", "strided_nan_gaps"]


@pytest.mark.parametrize("d", [16, 17, 64, 132])
@pytest.mark.parametrize("mode", EPILOGUES)
def test_spmm_exact_epilogue(mode, d):
    """out only, acc only (acc = E row + sum), both, the accumulate mode acc += sum (acc_init = 0) with E's row count
    different from n_rows as the sharded propagations use it, final_div 3 and ld_out / ld_acc / ld_e > d whose gap
    columns keep NaN sentinels; vec4 (16, 64) and scalar (17, 132) branches, long rows included."""
    rng = np.random.default_rng(300 + d + 1000 * EPILOGUES.index(mode))
    n = 200
    n_e = {"block_acc_fewer_E_rows": 77, "block_both_more_E_rows": 451}.get(mode, n)
    g = Graph(_mixed_degrees(rng, d, n_short=n), n_e, rng)
    E = _int_matrix(rng, n_e, d)
    ref = g.product64(E)
    block = mode.startswith("block")
    acc0 = _int_matrix(rng, n, d)
    base = acc0 if block else E[:n]
    _exact_inputs(g, E, base=base)
    div = 3.0 if mode.endswith("div3") else 0.0
    ld = d + 8 if mode == "strided_nan_gaps" else d
    if mode == "strided_nan_gaps":
        _, Ed = _strided(n_e, d, d + 4, fill=0.0)
        Ed.copy_(_dev(E))
    else:
        Ed = _dev(E)
    want_out = mode in ("out", "both", "block_both_more_E_rows", "strided_nan_gaps")
    want_acc = mode != "out"
    ob, out = _strided(n, d, ld) if want_out else (None, None)
    ab, acc = _strided(n, d, ld + 4) if want_acc else (None, None)
    if acc is not None and block:
        acc.copy_(_dev(acc0))
    _run_ok(g, Ed, out=out, acc=acc, acc_init=0 if block else 1, final_div=div)
    if want_out:
        np.testing.assert_array_equal(out.cpu().numpy(), ref.astype(np.float32))
        assert bool(torch_isnan_all(ob[: n * ld].view(n, ld)[:, d:]))
    if want_acc:
        x = (base.astype(np.float64) + ref).astype(np.float32)
        want = x / np.float32(div) if div else x
        np.testing.assert_array_equal(acc.cpu().numpy(), want)
        assert bool(torch_isnan_all(ab[: n * (ld + 4)].view(n, ld + 4)[:, d:]))


@pytest.mark.parametrize("d", [4, 3, 64, 132])
def test_spmm_all_empty_graph_null_col_val(d):
    """nnz = 0 with NULL col / val: out is all zero, acc = E row (acc_init = 1) or acc / final_div (acc_init = 0)."""
    rng = np.random.default_rng(d)
    g = Graph(np.zeros(37, dtype=np.int64), 37, rng)
    E = _int_matrix(rng, 37, d)
    out = _strided(37, d, d)[1]
    acc = _strided(37, d, d)[1]
    _run_ok(g, _dev(E), out=out, acc=acc, acc_init=1, null_col_val=True)
    assert (out.cpu().numpy() == 0).all()
    np.testing.assert_array_equal(acc.cpu().numpy(), E)
    _run_ok(g, _dev(E), acc=acc, acc_init=0, final_div=4.0, null_col_val=True)
    np.testing.assert_array_equal(acc.cpu().numpy(), E / np.float32(4))


# ---- random floats: per-element bound, determinism ----------------------------------------------------------------

@pytest.mark.parametrize("d", [3, 16, 64, 100, 132, 256])
def test_spmm_random_float_bound_and_determinism(d):
    """Random values: |got - ref64| <= (nnz_r + 2) u sum_j |v_j e_j| per element (any summation tree of the short
    and chunked paths stays within that height), plus one rounding of |E| + sum|v e| per epilogue add / divide.
    A second identical call is bit-identical, long rows included (the kernels use no float atomics)."""
    rng = np.random.default_rng(400 + d)
    g = Graph(_mixed_degrees(rng, d, n_short=250), 250, rng, exact=False)
    E = rng.standard_normal((250, d)).astype(np.float32)
    ref = g.product64(E)
    S = g.product64(E, absolute=True)
    nnz = g.deg[:, None].astype(np.float64)
    out, acc = _strided(250, d, d)[1], _strided(250, d, d)[1]
    _run_ok(g, _dev(E), out=out, acc=acc, acc_init=1, final_div=3.0)
    got_out, got_acc = out.cpu().numpy(), acc.cpu().numpy()
    sum_err = (nnz + 2) * U * S
    assert (np.abs(got_out - ref) <= sum_err).all()
    x = E.astype(np.float64) + ref
    acc_err = (sum_err + 2 * U * (np.abs(E) + S)) / 3.0
    assert (np.abs(got_acc - x / 3.0) <= acc_err).all()
    # the bound is tight enough to see one non-zero of a row lost
    assert (np.abs(g.val)[:, None] * np.abs(E[g.col]) > sum_err[g.rows]).mean() > 0.5
    out2, acc2 = _strided(250, d, d)[1], _strided(250, d, d)[1]
    _run_ok(g, _dev(E), out=out2, acc=acc2, acc_init=1, final_div=3.0)
    assert np.array_equal(out2.cpu().numpy().view(np.int32), got_out.view(np.int32))
    assert np.array_equal(acc2.cpu().numpy().view(np.int32), got_acc.view(np.int32))


# ---- envelope -------------------------------------------------------------------------------------------------------

def test_spmm_envelope_rejects_without_launch():
    """n_rows = 0 returns 0 and launches nothing; d = 0, d = 257 and a long-row count without its plan return -2
    before any launch.  Every device pointer passed is valid."""
    from librecommender_b200 import _lib

    rng = np.random.default_rng(7)
    empty = Graph(np.zeros(0, dtype=np.int64), 4, rng)
    E = _dev(_int_matrix(rng, 4, 8))
    n0 = _lib.launch_count()
    assert spmm(empty, E, out=_strided(1, 8, 8)[1]) == 0
    assert _lib.launch_count() == n0
    g = Graph([3, 1500], 4, rng)
    torch = _torch()
    for d in (0, 257):
        Ed = torch.zeros((4, max(d, 1)), dtype=torch.float32, device="cuda")[:, :d]
        outd = torch.zeros((2, max(d, 1)), dtype=torch.float32, device="cuda")[:, :d]
        assert spmm(g, Ed, out=outd) == -2
        assert _lib.launch_count() == n0
    assert spmm(g, _dev(_int_matrix(rng, 4, 8)), out=_strided(2, 8, 8)[1], plan=False) == -2
    assert b"plan missing" in _lib.lib.b200_last_error()
    assert _lib.launch_count() == n0


# ---- NGCF epilogue kernels ------------------------------------------------------------------------------------------

def _combine_rows(rng, d):
    a = rng.standard_normal((70, d)).astype(np.float32)
    b = rng.standard_normal((70, d)).astype(np.float32)
    a[3], b[3] = 0.0, 0.0                                  # all-zero row: exactly 0, not NaN
    a[4] = rng.uniform(0.5, 1.0, d) * 1e-14                # norm < 1e-12: m / 1e-12 (F.normalize's eps)
    b[4] = -rng.uniform(0.0, 0.4, d) * 1e-14
    a[5] = rng.standard_normal(d) * 1e17                   # large rows: m^2 summed without overflow
    b[5] = rng.standard_normal(d) * 1e17
    a[6], b[6] = -np.abs(a[6]), -np.abs(b[6])              # all negative: only the slope branch
    a[7], b[7] = a[7], -a[7]                               # cancels to exactly zero
    return a, b


@pytest.mark.parametrize("slope", [0.2, 0.0, 1.0])
@pytest.mark.parametrize("d", [1, 7, 32, 33, 64, 130, 256])
def test_ngcf_combine_vs_float64(d, slope):
    """normalize(leaky_relu(a + b, slope)) per row with strided lda / ldb / ld_out; m = float32(a) + float32(b) as
    the kernel forms it, the rest in float64.  Bound per element: ((L + 7) / 2 + 4) u |ref| with L = ceil(d / 32),
    the fma chain per lane: L + 5 roundings in the sum of squares (chain + butterfly) and 2 from the squared slope
    product, halved by the square root, then the square root, the reciprocal, the final product and the slope
    product in the numerator."""
    from librecommender_b200 import _lib

    rng = np.random.default_rng(d * 10 + int(slope * 10))
    a, b = _combine_rows(rng, d)
    R = len(a)
    ab, av = _strided(R, d, d + 3, fill=0.0)
    bb, bv = _strided(R, d, d + 1, fill=0.0)
    av.copy_(_dev(a))
    bv.copy_(_dev(b))
    ob, out = _strided(R, d, d + 5)
    _lib.check(_lib.lib.b200_ngcf_combine(_lib.ptr(av), d + 3, _lib.ptr(bv), d + 1, R, d, slope, _lib.ptr(out), d + 5,
                                          _lib.current_stream()))
    got = out.cpu().numpy()
    assert bool(torch_isnan_all(ob[: R * (d + 5)].view(R, d + 5)[:, d:]))
    m = (a + b).astype(np.float64)
    m = np.where(m > 0, m, float(np.float32(slope)) * m)
    ref = m / np.maximum(np.sqrt((m * m).sum(1, keepdims=True)), 1e-12)
    L = -(-d // 32)
    bound = ((L + 7) / 2 + 4) * U * np.abs(ref)
    assert not np.isnan(got).any()
    assert (got[3] == 0).all() and (got[7] == 0).all()
    assert (np.abs(got - ref) <= bound).all(), np.abs(got - ref).max()
    np.testing.assert_allclose(got[4], m[4] / 1e-12, rtol=8 * U)
    n0 = _lib.launch_count()
    _lib.check(_lib.lib.b200_ngcf_combine(_lib.ptr(av), d + 3, _lib.ptr(bv), d + 1, 0, d, slope, _lib.ptr(out), d + 5,
                                          _lib.current_stream()))
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 1_000_003])
def test_mul_elementwise_bit_exact(n):
    """a * b elementwise equals numpy's float32 product bit for bit at block-boundary sizes; n = 0 launches
    nothing."""
    from librecommender_b200 import _lib

    rng = np.random.default_rng(n)
    a = rng.standard_normal(max(n, 1)).astype(np.float32)
    b = rng.standard_normal(max(n, 1)).astype(np.float32)
    ad, bd = _dev(a), _dev(b)
    out = _torch().full((max(n, 1) + 1,), float("nan"), device="cuda")
    n0 = _lib.launch_count()
    _lib.check(_lib.lib.b200_mul_elementwise(_lib.ptr(ad), _lib.ptr(bd), n, _lib.ptr(out), _lib.current_stream()))
    got = out.cpu().numpy()
    assert _lib.launch_count() == n0 + (1 if n else 0)
    assert np.array_equal(got[:n].view(np.int32), (a[:n] * b[:n]).view(np.int32))
    assert np.isnan(got[n:]).all()
