"""GpuRqEncoder: ResidualQuantizer's beam search on the device, in both distance modes.

On integer-valued data and codebooks (every dot product, norm and partial sum exact in fp32) refine_beam,
refine_beam_LUT and compute_codes equal the CPU's bit for bit: the numpy restatement (oracle/oracle_rq_np.py, pinned to
the reference by tests/test_rq_oracle.py), the reference-minted fixture and, where it is built, the live reference
library.  On float data with CPU-trained codebooks the total encode error agrees with the CPU's to 1e-3.  Results do not
depend on pointer residency, the page budget or how n is split over calls."""
import numpy as np
import pytest

from oracle import oracle_rq_np as ro
from tests.golden import make_golden_rq as g

fb = pytest.importorskip("faiss_b200")

SHAPES = [
    (32, [6] * 4, 5),
    (128, [8] * 8, 32),
    (40, [4, 8, 6, 8, 5, 8, 8, 3, 8, 8], 16),
    (64, [12] * 3, 1),
]


def _ref():
    from oracle import ref_rq

    return ref_rq if ref_rq.available() else None


@pytest.fixture(scope="module")
def res():
    return fb.StandardGpuResources()


def _encoder(res, d, nbits, cb):
    enc = fb.GpuRqEncoder(d, nbits, res)
    enc.setCodebooks(cb)
    return enc


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), b.view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def synthetic(d, n, seed=1338):
    # faiss.contrib.datasets.SyntheticDataset's generator
    rs = np.random.RandomState(seed)
    x = rs.normal(size=(n, 10))
    x = np.dot(x, rs.rand(10, d))
    x = x * (rs.rand(d) * 4 + 0.1)
    return np.sin(x).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("d,nbits,beam", SHAPES, ids=["d32m4", "d128m8b32", "d40m10mixed", "d64nbits12b1"])
def test_integer_data_equals_cpu(res, d, nbits, beam):
    rs = np.random.RandomState(d + beam)
    n = 150
    cb, x, cent = g.int_data(rs, d, nbits, n, False)
    enc = _encoder(res, d, nbits, cb)
    ref = _ref()
    q = ref.RQ(d, nbits, cb) if ref is not None else None

    got = enc.refineBeam(x[:, None], beam)
    want = ro.refine_beam(cb, nbits, x[:, None], beam)
    assert all(_same(a, b) for a, b in zip(got, want))
    if q is not None:
        assert all(_same(a, b) for a, b in zip(got, q.refine_beam(x[:, None], 1, beam)))
    if beam >= 3:  # three input entries per row
        xb = np.stack([x, x + 1, x - 2], 1)
        assert all(_same(a, b) for a, b in zip(enc.refineBeam(xb, beam), ro.refine_beam(cb, nbits, xb, beam)))

    got = enc.refineBeamLUT(x, beam)
    want = ro.refine_beam_lut(cb, nbits, x, beam)
    assert all(_same(a, b) for a, b in zip(got, want))
    if q is not None:
        assert all(_same(a, b) for a, b in zip(got, q.refine_beam_lut(x, beam)))

    lo_, hi = g.NORM_RANGE
    for lut in (0, 1):
        for st in ro.DEVICE_PACKED:
            for cen in (None, cent):
                got = enc.computeCodes(x, lut, beam, st, lo_, hi, cen)
                assert _same(got, ro.compute_codes(cb, nbits, x, lut, beam, st, lo_, hi, cen)), (lut, st, cen is None)
                if q is not None and st in (ro.ST_decompress, ro.ST_norm_float, ro.ST_norm_qint4):
                    qs = ref.RQ(d, nbits, cb, search_type=st, max_beam_size=beam, use_beam_LUT=lut, norm_min=lo_, norm_max=hi)
                    assert _same(got, qs.compute_codes(x, cen)), (lut, st, cen is None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
def test_golden_cases(res, case):
    # the reference-minted fixtures: forced ties, K < 32 and K >= 32 steps, M = 10, beams 1 / 5 / 32
    name, d, nbits, beam, n, _ = case
    c = g.case(g.load(), name)
    enc = _encoder(res, d, nbits, c["cb"])
    codes, resid, dis = enc.refineBeam(c["x"][:, None], beam)
    assert _same(codes, c["codes0"]) and _same(resid, c["resid0"]) and _same(dis, c["dis0"])
    codes, dis = enc.refineBeamLUT(c["x"], beam)
    assert _same(codes, c["codes1"]) and _same(dis, c["dis1"])
    for lut in (0, 1):
        for st in g.SEARCH_TYPES:
            assert _same(enc.computeCodes(c["x"], lut, beam, st, *g.NORM_RANGE), c["packed%d_%d" % (lut, st)])
            got = enc.computeCodes(c["x"], lut, beam, st, *g.NORM_RANGE, centroids=c["cent"])
            assert _same(got, c["packed%d_%d_cent" % (lut, st)])


@pytest.mark.gpu
def test_unpacked_codes(res):
    d, nbits, beam = 24, [5, 7, 6], 8
    cb, x, _ = g.int_data(np.random.RandomState(3), d, nbits, 100, False)
    enc = _encoder(res, d, nbits, cb)
    assert _same(enc.encodeUnpacked(x, 0, beam), ro.refine_beam(cb, nbits, x[:, None], beam)[0][:, 0])
    assert _same(enc.encodeUnpacked(x, 1, beam), ro.refine_beam_lut(cb, nbits, x, beam)[0][:, 0])


def _train_codebooks(d, nbits, xt):
    ref = _ref()
    if ref is not None:
        q = ref.RQ(d, nbits)
        q.train(xt, max_beam_size=5, niter=10)
        return q.tables()[0]
    # a cheap additive codebook: each level is K rows of the previous level's residuals
    rs = np.random.RandomState(0)
    r = xt.astype(np.float64)
    cbs = []
    for nb in nbits:
        c = r[rs.choice(r.shape[0], 1 << nb, replace=False)]
        r = r - c[((r[:, None, :] - c[None]) ** 2).sum(-1).argmin(1)]
        cbs.append(c)
    return np.concatenate(cbs).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("lut", [0, 1])
def test_float_data_error_matches_cpu(res, lut):
    d, nbits, beam = 32, [8] * 4, 8
    x = synthetic(d, 6000)
    xt, xb = x[:4000], x[4000:]
    cb = _train_codebooks(d, nbits, xt)
    enc = _encoder(res, d, nbits, cb)
    got = enc.computeCodes(xb, lut, beam)
    ref = _ref()
    if ref is not None:
        cpu = ref.RQ(d, nbits, cb, max_beam_size=beam, use_beam_LUT=lut).compute_codes(xb)
    else:
        cpu = ro.compute_codes(cb, nbits, xb, lut, beam)

    def err(packed):
        bits = np.unpackbits(packed, axis=1, bitorder="little").astype(np.int64)
        codes = np.stack([(bits[:, 8 * m:8 * m + 8] << np.arange(8)).sum(1) for m in range(len(nbits))], 1)
        return float(((ro.decode_unpacked(cb, nbits, codes).astype(np.float64) - xb) ** 2).sum())

    eg, ec = err(got), err(cpu)
    assert abs(eg - ec) <= 1e-3 * ec, (eg, ec, float((got == cpu).all(1).mean()))


@pytest.mark.gpu
@pytest.mark.parametrize("lut", [0, 1])
def test_invariance_residency_paging_splits(res, lut):
    import torch

    d, nbits, beam, n = 40, [6, 8, 5, 7], 12, 1000
    x = synthetic(d, n, seed=7)
    cb = _train_codebooks(d, nbits, synthetic(d, 3000, seed=8))
    enc = _encoder(res, d, nbits, cb)

    def run(enc, x, **kw):
        if lut:
            return enc.refineBeamLUT(x, beam, **kw) + (enc.computeCodes(x, 1, beam, ro.ST_norm_qint8, 1.0, 30.0, **kw),)
        return enc.refineBeam(x[:, None], beam, **kw) + (enc.computeCodes(x, 0, beam, ro.ST_norm_float, **kw),)

    base = [np.asarray(a) for a in run(enc, x)]
    dev = run(enc, torch.from_numpy(x).cuda())
    assert all(_same(a.cpu().numpy(), b) for a, b in zip(dev, base))
    per_row = 4 * (3 * beam * d + beam * 256 + 4 * beam * len(nbits) + 2 * d)
    for rows in (37, 1):
        assert all(_same(a, b) for a, b in zip(run(enc, x, page_bytes=rows * per_row), base)), rows
    parts = [run(enc, x[a:b]) for a, b in ((0, 1), (1, 400), (400, n))]
    assert all(_same(np.concatenate([p[i] for p in parts]), base[i]) for i in range(len(base)))
    enc2 = fb.GpuRqEncoder(d, nbits, res)
    enc2.setCodebooks(torch.from_numpy(cb).cuda())
    assert all(_same(a, b) for a, b in zip(run(enc2, x), base))


@pytest.mark.gpu
def test_limits_throw_and_leave_the_encoder_usable(res):
    with pytest.raises(fb.FaissError, match="1 <= nbits <= 12"):
        fb.GpuRqEncoder(8, [4, 13], res)
    d, nbits = 8, [4, 5]
    cb, x, _ = g.int_data(np.random.RandomState(0), d, nbits, 50, False)
    enc = fb.GpuRqEncoder(d, nbits, res)
    with pytest.raises(fb.FaissError, match="setCodebooks"):
        enc.computeCodes(x, 0, 5)
    enc.setCodebooks(cb)
    with pytest.raises(fb.FaissError, match="1 <= beam <= 256"):
        enc.computeCodes(x, 0, 257)
    with pytest.raises(fb.FaissError, match="1 <= beam <= 256"):
        enc.refineBeam(np.zeros((2, 300, d), np.float32), 5)
    with pytest.raises(fb.FaissError, match="not packed on the device"):
        enc.computeCodes(x, 0, 5, fb.ST_norm_cqint8)
    assert _same(enc.computeCodes(x, 1, 5), ro.compute_codes(cb, nbits, x, 1, 5))
    # the LUT kernel keeps two int16 beams of M codes per row in shared memory: M = 240 at beam 256 does not fit
    big = fb.GpuRqEncoder(4, [1] * 240, res)
    big.setCodebooks(np.ones((480, 4), np.float32))
    with pytest.raises(fb.FaissError, match="shared memory"):
        big.refineBeamLUT(np.ones((3, 4), np.float32), 256)
    assert big.refineBeamLUT(np.ones((3, 4), np.float32), 2)[0].shape == (3, 2, 240)
    assert _same(enc.refineBeam(x[:, None], 5)[0], ro.refine_beam(cb, nbits, x[:, None], 5)[0])
