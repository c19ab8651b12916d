"""K1, ``b200_feat_forward``, held directly against float64 (tests/_feat_gather_ref.py) on hand-built layouts:
* every kernel family at every template argument: the generic kernel (sub-warp rows for K < 32, several passes up to
  K = 256), lane-per-field <1..8>, field-group / software-pipelined / cp.async staged / bulk-copy (TMA) <1, 2, 4, 8>;
  a profiler check per family that the kernel that ran is the one ``expected_kernel`` names;
* every output (concat, pw, lin, fm_out with and without BN, ssum + sqsum), all together and alone;
* outputs inside NaN-filled buffers with extra columns and rows: nothing outside is touched, nothing inside is skipped;
* grid mode in chunks whose offsets are no multiple of the item count, explicit feature rows with wide strides, tower /
  ids-only / dense-only layouts, OOV and repeated ids, dense values 0, negative and ~1e3, heavy cancellation in pw;
* dispatch edges: R = 0, 1, 2047 / 2048, 4095 / 4096, 16 / 17 staged steps, 258 fields, misaligned pointers;
* bit-for-bit repeatability, one concat across all families, and errors raised before any launch.
concat must match bit for bit (copies and one float32 product); the sums and heads are held to the per-element bounds
of ``_feat_gather_ref.bounds``."""
import numpy as np
import pytest

import _feat_gather_ref as fr

pytestmark = pytest.mark.gpu

SENT = np.int32(0x7FC0FFEE)      # quiet NaN with a payload no kernel writes
PAD_ROWS = 5
TUNE = {"generic": 0, "lanefield": 2, "fieldgroup": 4, "pipe": 0, "async": 8, "tma": 1}
TABLES = ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds",
          "user_linear", "item_linear", "sparse_linear", "dense_linear")


@pytest.fixture
def tune():
    """Sets the process-wide K1 kernel switch; always restores the default."""
    from librecommender_b200 import _lib

    def set_code(code):
        _lib.check(_lib.lib.b200_feat_forward_tune(int(code)))

    try:
        yield set_code
    finally:
        set_code(0)


class Dev:
    """Device copy of a case: FeatLayoutStruct, FeatTablesStruct, head tensors.  ``misalign``: the sparse table is
    placed 4 bytes past a 16-byte boundary (the fast kernels need 16-byte rows)."""

    def __init__(self, case, sparse_rows=None, dense_rows=None, misalign=False):
        import torch

        from librecommender_b200.feat_models import FeatLayoutStruct, tables_struct

        cu = lambda a, dt=torch.float32: torch.as_tensor(np.ascontiguousarray(a)).to("cuda", dt)
        self.case, self.K, self.F = case, int(case["K"]), fr.n_fields(case)
        self.t = {n: cu(case[n]) for n in TABLES}
        if misalign:
            se = self.t["sparse_embeds"]
            buf = torch.empty(se.numel() + 1, dtype=torch.float32, device="cuda")
            buf[1:] = se.reshape(-1)
            self.t["sparse_embeds"] = buf[1:].view(se.shape)
        self.uniq = {n: cu(case[n], torch.int32 if "sparse" in n else torch.float32)
                     for n in ("user_sparse_unique", "item_sparse_unique", "user_dense_unique", "item_dense_unique")}
        L = FeatLayoutStruct()
        L.embed_size, L.id_mask = self.K, int(case["id_mask"])
        L.n_sparse, L.n_dense = len(case["sparse_side"]), len(case["dense_side"])
        for f in range(L.n_sparse):
            L.sparse_side[f], L.sparse_col[f] = int(case["sparse_side"][f]), int(case["sparse_col"][f])
        for f in range(L.n_dense):
            L.dense_side[f], L.dense_col[f] = int(case["dense_side"][f]), int(case["dense_col"][f])
            L.dense_embed_row[f] = int(case["dense_embed_row"][f])
        for n, ld in (("user_sparse_unique", "ld_us"), ("item_sparse_unique", "ld_is"),
                      ("user_dense_unique", "ld_ud"), ("item_dense_unique", "ld_id")):
            setattr(L, n, self.uniq[n].data_ptr())
            setattr(L, ld, self.uniq[n].stride(0))
        self.rows = []
        for name, ld, a, dt in (("sparse_rows", "ld_sparse_rows", sparse_rows, torch.int32),
                                ("dense_rows", "ld_dense_rows", dense_rows, torch.float32)):
            if a is None:
                setattr(L, name, None)
                continue
            # explicit rows inside a wider matrix: the stride is larger than the field count
            buf = torch.zeros((a.shape[0], a.shape[1] + 3), dtype=dt, device="cuda")
            buf[:, : a.shape[1]] = cu(a, dt)
            self.rows.append(buf)
            setattr(L, name, buf.data_ptr())
            setattr(L, ld, buf.stride(0))
        self.L, self.T = L, tables_struct(self.t)
        self.lin_kernel = cu(case["lin_kernel"])
        self.head_bn = dict(bn_scale=cu(case["bn_scale"]), bn_shift=cu(case["bn_shift"]), pw_kernel=cu(case["pw_kernel"]),
                            pw_bias=float(case["pw_bias"]))
        self.head_nobn = dict(pw_kernel=self.head_bn["pw_kernel"], pw_bias=float(case["pw_bias"]))


def _buf(rows, cols):
    import torch

    shape = (rows + PAD_ROWS,) + ((cols,) if cols else ())
    return torch.full(shape, int(SENT), dtype=torch.int32, device="cuda").view(torch.float32)


def run(dev, users, items, R, outs=("concat", "pw", "lin", "fm_out", "ss"), bn=True, grid_items=0, row_offset=0,
        pad=(4, 3, 5), concat_off=0):
    """One b200_feat_forward call; every output inside a sentinel buffer with ``pad`` extra columns (concat, pw,
    ssum / sqsum) and PAD_ROWS extra rows.  ``concat_off``: the concat view starts that many floats into its
    buffer.  Returns {name: (whole buffer as numpy, width or None)}."""
    import torch

    from librecommender_b200 import feat_models as fm

    K, F = dev.K, dev.F
    bufs, kw = {}, {}
    if "concat" in outs:
        b = _buf(R, F * K + pad[0] + (4 if concat_off else 0))     # ld % 4 unchanged by the offset
        bufs["concat"] = (b, F * K, concat_off)
        kw["concat"] = b[:R, concat_off: concat_off + F * K]
    if "pw" in outs:
        b = _buf(R, K + pad[1])
        bufs["pw"] = (b, K, 0)
        kw["pw"] = b[:R, :K]
    for name in ("lin", "fm_out"):
        if name in outs:
            b = _buf(R, 0)
            bufs[name] = (b, None, 0)
            kw[name] = b[:R]
    if "ss" in outs:
        for name in ("ssum", "sqsum"):
            b = _buf(R, K + pad[2])
            bufs[name] = (b, K, 0)
            kw[name] = b[:R, :K]
    if "lin" in outs or "fm_out" in outs:
        kw.update(lin_kernel=dev.lin_kernel, lin_bias=float(dev.case["lin_bias"]))
    if "fm_out" in outs:
        kw["head"] = dev.head_bn if bn else dev.head_nobn
    fm.feat_forward(dev.L, dev.T, users, items, R, grid_items=grid_items, row_offset=row_offset, **kw)
    torch.cuda.synchronize()
    return {n: (b.cpu().numpy(), w, off) for n, (b, w, off) in bufs.items()}


def check(got, want, R, label=""):
    """Sentinels untouched, every in-range element written, concat bit-exact, the rest within the bounds."""
    for name, (buf, width, off) in got.items():
        bits = buf.view(np.int32)
        inside = np.zeros(bits.shape, dtype=bool)
        if width is None:
            inside[:R] = True
        else:
            inside[:R, off: off + width] = True
        assert (bits[~inside] == SENT).all(), f"{label} {name}: write outside the output"
        v = buf[inside].reshape((R, width) if width else (R,))
        assert not (v.view(np.int32) == SENT).any(), f"{label} {name}: element left unwritten"
        if name == "concat":
            np.testing.assert_array_equal(v.view(np.int32), want["concat"].view(np.int32), err_msg=f"{label} concat")
        else:
            ratio = fr.worst(v, want[name], want["bound"][name])
            assert ratio <= 1.0, f"{label} {name}: error {ratio:.3g} x the bound"


def ids(rng, case_users, case_items, R):
    """Row ids with repeats and the OOV rows (n_users / n_items) included."""
    u = rng.integers(0, case_users + 1, R)
    it = rng.integers(0, case_items + 1, R)
    u[::97], it[::89] = case_users, case_items
    return u, it


def cuda_ids(*a):
    import torch

    return [torch.as_tensor(np.asarray(x, dtype=np.int64)).cuda() for x in a]


def _same(a, b, label):
    for n in a:
        np.testing.assert_array_equal(a[n][0].view(np.int32), b[n][0].view(np.int32), err_msg=f"{label} {n}")


# ---- the path matrix ---------------------------------------------------------------------------------------------------
# (family, K, R): every instantiation; field counts of the staged cases give 1 to 9 steps of 32 / K4 fields.
PATHS = ([("generic", K, 1000 + K) for K in (1, 2, 3, 5, 7, 10, 17, 30, 33, 64, 100, 256)] +
         [("lanefield", 4 * k4, 1237) for k4 in range(1, 9)] +
         [("fieldgroup", 4 * k4, 5003) for k4 in (1, 2, 4, 8)] +
         [("pipe", 4 * k4, 4099) for k4 in (1, 2, 4, 8)] +
         [("async", 4 * k4, 4133) for k4 in (1, 2, 4, 8)] +
         [("tma", 4 * k4, 2053) for k4 in (1, 2, 4, 8)])


def _path_case(family, K):
    rng = np.random.default_rng(K * 31 + len(family))
    if family in ("pipe", "async", "tma"):
        return rng, fr.make_case(rng, K, 10, 14, 4, 5, dense_row_perm=True)      # F = 35
    return rng, fr.make_case(rng, K, 5, 7, 2, 3, dense_row_perm=True)            # F = 19


@pytest.mark.parametrize("family,K,R", PATHS, ids=[f"{f}-K{K}" for f, K, _ in PATHS])
def test_path_matrix(family, K, R, tune):
    rng, case = _path_case(family, K)
    F = fr.n_fields(case)
    code = TUNE[family]
    want_k = (family, K // 4 if family != "generic" else None)
    assert fr.expected_kernel(K, R, F, tune=code) == want_k
    dev = Dev(case)
    u, it = ids(rng, 300, 400, R)
    ud, itd = cuda_ids(u, it)
    tune(code)
    w_bn, w_nobn = fr.ref(case, u, it), fr.ref(case, u, it, bn=False)
    a = run(dev, ud, itd, R)
    check(a, w_bn, R, f"{family} K={K} all")
    _same(a, run(dev, ud, itd, R), f"{family} K={K} repeat")
    check(run(dev, ud, itd, R, outs=("fm_out",), bn=False), w_nobn, R, f"{family} K={K} fm_out alone, no BN")
    check(run(dev, ud, itd, R, outs=("concat",)), w_bn, R, f"{family} K={K} concat alone")
    check(run(dev, ud, itd, R, outs=("pw", "lin")), w_bn, R, f"{family} K={K} pw + lin")


def _k1_kernels(prof):
    import torch

    out = []
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            k = fr.kernel_of(e.name)
            if k is not None:
                out.append(k)
    return out


@pytest.mark.parametrize("family", list(TUNE))
def test_dispatch_names_the_kernel_that_ran(family, tune):
    """torch.profiler's CUDA kernel records of one call per path-matrix case of the family: exactly the kernel
    ``expected_kernel`` names, at every template argument."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    cases = [(K, R) for f, K, R in PATHS if f == family]
    prepared = []
    for K, R in cases:
        rng, case = _path_case(family, K)
        u, it = ids(rng, 300, 400, R)
        prepared.append((K, R, case, Dev(case), *cuda_ids(u, it)))
    tune(TUNE[family])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for K, R, case, dev, ud, itd in prepared:
            run(dev, ud, itd, R)
    want = [fr.expected_kernel(K, R, fr.n_fields(case), tune=TUNE[family]) for K, R, case, *_ in prepared]
    ran = _k1_kernels(prof)
    key = lambda k: (k[0], k[1] or 0)
    assert sorted(ran, key=key) == sorted(want, key=key), (family, ran)
    if family != "generic":
        assert sorted(k[1] for k in ran) == sorted({K // 4 for K, *_ in prepared})


# ---- grid mode -------------------------------------------------------------------------------------------------------
GRID = [("generic", 7), ("lanefield", 12), ("fieldgroup", 16), ("pipe", 16), ("async", 32), ("tma", 8)]


@pytest.mark.parametrize("family,K", GRID)
def test_grid_chunks(family, K, tune):
    """users x N grid in chunks of odd length starting at offsets that are no multiple of N: each chunk against float64
    of its explicit pairs, and bit for bit against the same call on those pairs."""
    rng = np.random.default_rng(K + 7)
    case = fr.make_case(rng, K, 4, 6, 2, 3, n_users=50, n_items=1021)
    dev = Dev(case)
    N = 1021
    users = rng.integers(0, 51, 11)
    users[3] = 50                                         # the OOV user
    (users_d,) = cuda_ids(users)
    tune(TUNE[family])
    for off, R in ((333, 4099), (4432, 4101), (8533, 2051), (10584, 1), (10585, 3)):
        assert off % N and off + R <= len(users) * N
        want = fr.ref(case, users, R=R, grid_items=N, row_offset=off)
        g = run(dev, users_d, users_d, R, grid_items=N, row_offset=off)
        check(g, want, R, f"{family} grid chunk {off}+{R}")
        pu, pi = fr.row_ids(users, None, R, N, off)
        pud, pid = cuda_ids(pu, pi)
        _same(g, run(dev, pud, pid, R), f"{family} grid chunk {off}+{R} vs pairs")


# ---- explicit feature rows --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family,K,code", [("generic", 7, 0), ("lanefield", 12, 0), ("lanefield", 16, 2),
                                          ("fieldgroup", 16, 0), ("fieldgroup", 32, 8), ("tma", 16, 1)])
def test_explicit_rows(family, K, code, tune):
    """sparse_rows / dense_rows (strides wider than the field count) at R >= 4096: the staged register kernels, which
    read the unique tables only, must not be chosen."""
    rng = np.random.default_rng(K + code)
    case = fr.make_case(rng, K, 5, 4, 2, 2)
    R = 4100
    sr = rng.integers(0, 500, (R, 9)).astype(np.int32)
    sr[::7, 3] = 0
    dr = (rng.standard_normal((R, 4)) * 30).astype(np.float32)
    dr[::5, 1] = 0
    dr[::11, 2] = 1000.5
    dr[::13, 0] = -999.25
    F = fr.n_fields(case)
    assert fr.expected_kernel(K, R, F, explicit_rows=True, tune=code) == (family, K // 4 if family != "generic" else None)
    dev = Dev(case, sparse_rows=sr, dense_rows=dr)
    u, it = ids(rng, 300, 400, R)
    ud, itd = cuda_ids(u, it)
    tune(code)
    check(run(dev, ud, itd, R), fr.ref(case, u, it, sparse_rows=sr, dense_rows=dr), R, f"{family} explicit rows")


# ---- layouts and values ----------------------------------------------------------------------------------------------
def _layout(name, K, rng):
    if name == "ids_only":
        return fr.make_case(rng, K, id_mask=3)
    if name == "user_tower":
        return fr.make_case(rng, K, 6, 0, 3, 0, id_mask=1)
    if name == "item_tower":
        return fr.make_case(rng, K, 0, 5, 0, 2, id_mask=2)
    if name == "dense_only":
        return fr.make_case(rng, K, 0, 0, 3, 4, id_mask=0, dense_row_perm=True)
    if name == "item_dense":
        return fr.make_case(rng, K, 3, 3, 0, 5)
    if name == "dense_1e3":
        return fr.make_case(rng, K, 2, 3, 2, 3, dense_scale=1e3)
    # heavy cancellation: every sparse field appears with its negation, so ssum = 0 and pw = -sqsum / 2
    c = fr.make_case(rng, K, 3, 3, 0, 0, id_mask=0, vocab=64)
    c["sparse_embeds"] = np.concatenate([c["sparse_embeds"][:32], -c["sparse_embeds"][:32]])
    for s in ("user", "item"):
        t = c[f"{s}_sparse_unique"] % 32
        c[f"{s}_sparse_unique"] = np.concatenate([t, t + 32], 1).astype(np.int32)
    c["sparse_side"] = np.array([0, 0, 0, 1, 1, 1] * 2, np.int32)
    c["sparse_col"] = np.array([0, 1, 2, 0, 1, 2, 3, 4, 5, 3, 4, 5], np.int32)
    c["lin_kernel"] = c["lin_kernel"][:12] if len(c["lin_kernel"]) >= 12 else np.resize(c["lin_kernel"], 12)
    return c


LAYOUTS = ("ids_only", "user_tower", "item_tower", "dense_only", "item_dense", "dense_1e3", "cancel")


@pytest.mark.parametrize("family", list(TUNE))
@pytest.mark.parametrize("layout", LAYOUTS)
def test_layouts_and_values(layout, family, tune):
    K = 5 if family == "generic" else (12 if family == "lanefield" else 16)
    rng = np.random.default_rng(10 * LAYOUTS.index(layout) + list(TUNE).index(family))
    case = _layout(layout, K, rng)
    R = 4099
    F = fr.n_fields(case)
    assert fr.expected_kernel(K, R, F, tune=TUNE[family])[0] == family
    dev = Dev(case)
    u, it = ids(rng, 300, 400, R)
    ud, itd = cuda_ids(u, it)
    tune(TUNE[family])
    want = fr.ref(case, u, it)
    if layout == "cancel":
        assert np.abs(want["ssum"]).max() <= 1e-12 * np.abs(want["sqsum"]).max()
    check(run(dev, ud, itd, R), want, R, f"{layout} {family}")


# ---- dispatch edges --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [0, 1, 2047, 2048, 4095, 4096])
@pytest.mark.parametrize("code", [0, 1, 8])
def test_row_count_edges(R, code, tune):
    rng = np.random.default_rng(R + code)
    case = fr.make_case(rng, 16, 3, 4, 1, 2)
    dev = Dev(case)
    u, it = ids(rng, 300, 400, max(R, 1))
    ud, itd = cuda_ids(u[:R], it[:R])
    tune(code)
    check(run(dev, ud, itd, R), fr.ref(case, u[:R], it[:R]), R, f"R={R} tune={code}")


@pytest.mark.parametrize("code,K,n_s,n_d,family", [
    (0, 32, 62, 0, "pipe"), (0, 32, 62, 1, "fieldgroup"),            # 16 / 17 steps of 4 fields
    (8, 32, 62, 0, "async"), (8, 32, 62, 1, "fieldgroup"),
    (0, 4, 126, 128, "pipe"), (8, 4, 126, 128, "async"),           # 256 fields of K = 4: 8 steps of 32
    (2, 32, 128, 128, "lanefield"), (2, 20, 128, 128, "lanefield"),  # 258 fields: three 128-field chunks
    (4, 32, 128, 128, "fieldgroup"), (0, 33, 128, 128, "generic"),
    (1, 32, 128, 128, "tma"),                                      # 33 KB rows: one row per stage
])
def test_field_count_edges(code, K, n_s, n_d, family, tune):
    rng = np.random.default_rng(n_s + n_d + K)
    case = fr.make_case(rng, K, n_s // 2, n_s - n_s // 2, n_d // 2, n_d - n_d // 2)
    F = fr.n_fields(case)
    R = {"pipe": 4096, "async": 4096, "tma": 2048}.get(family, 1500)
    assert fr.expected_kernel(K, R, F, tune=code)[0] == family
    dev = Dev(case)
    u, it = ids(rng, 300, 400, R)
    ud, itd = cuda_ids(u, it)
    tune(code)
    check(run(dev, ud, itd, R), fr.ref(case, u, it), R, f"F={F} K={K} tune={code}")


@pytest.mark.parametrize("what", ["table", "concat_ptr", "ld_concat"])
@pytest.mark.parametrize("code", [0, 1])
def test_misaligned_pointers_take_the_generic_kernel(what, code, tune):
    """A table or concat that is not 16-byte aligned, or ld_concat % 4 != 0: the generic kernel, same results."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    rng = np.random.default_rng(3)
    case = fr.make_case(rng, 16, 4, 4, 2, 2)
    R = 4099
    dev = Dev(case, misalign=what == "table")
    u, it = ids(rng, 300, 400, R)
    ud, itd = cuda_ids(u, it)
    kw = dict(concat_off=1) if what == "concat_ptr" else dict(pad=(5, 3, 5)) if what == "ld_concat" else {}
    tune(code)
    want = fr.ref(case, u, it)
    # torch.profiler occasionally delivers no CUDA kernel record at all for a window this short; such a window says
    # nothing about the dispatch, so it is profiled again.  Any window that records a K1 kernel must show exactly
    # the generic one.
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            got = run(dev, ud, itd, R, **kw)
        check(got, want, R, f"misaligned {what}")
        ran = _k1_kernels(prof)
        if ran:
            break
    assert ran == [("generic", None)]


def test_concat_identical_across_families(tune):
    """One shape through every family (the generic one through a misaligned table): the same concat bits."""
    rng = np.random.default_rng(11)
    case = fr.make_case(rng, 16, 5, 6, 2, 3)
    R = 4099
    u, it = ids(rng, 300, 400, R)
    ud, itd = cuda_ids(u, it)
    dev, dev_mis = Dev(case), Dev(case, misalign=True)
    got = {}
    for family, code in TUNE.items():
        tune(code)
        got[family] = run(dev_mis if family == "generic" else dev, ud, itd, R, outs=("concat", "ss"))
    for family, g in got.items():
        np.testing.assert_array_equal(g["concat"][0].view(np.int32), got["pipe"]["concat"][0].view(np.int32), err_msg=family)
    check(got["pipe"], fr.ref(case, u, it), R, "pipe")


# ---- errors before any launch -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("what", ["K0", "K257", "n_sparse129", "ssum_alone", "fm_out_no_pw_kernel", "items_null"])
def test_errors_before_launch(what):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200 import feat_models as fm
    from librecommender_b200.feat_models import FeatLayoutStruct

    rng = np.random.default_rng(5)
    case = fr.make_case(rng, 16, 2, 2, 1, 1)
    dev = Dev(case)
    R = 64
    ud, itd = cuda_ids(*ids(rng, 300, 400, R))
    L = FeatLayoutStruct.from_buffer_copy(dev.L)
    out = torch.zeros((R, 16), dtype=torch.float32, device="cuda")
    kw = dict(pw=out)
    items = itd
    if what == "K0":
        L.embed_size = 0
    elif what == "K257":
        L.embed_size = 257
    elif what == "n_sparse129":
        L.n_sparse = 129
    elif what == "ssum_alone":
        kw = dict(ssum=out)
    elif what == "fm_out_no_pw_kernel":
        kw = dict(fm_out=out[:, 0].contiguous(), lin_kernel=dev.lin_kernel, head=dict(bn_scale=dev.head_bn["bn_scale"],
                                                                                      bn_shift=dev.head_bn["bn_shift"]))
    else:
        items = None
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    with pytest.raises(_lib.B200Error):
        fm.feat_forward(L, dev.T, ud, items, R, **kw)
    assert _lib.launch_count() == n0
    assert (out == 0).all()
