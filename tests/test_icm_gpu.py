"""GpuIcmEncoder: LocalSearchQuantizer's ICM encoding on the device, fed the CPU encoder's perturbation draws.

On integer-valued data (every unary, binary and evaluate sum exact in fp32) the codes equal the CPU lsq::IcmEncoder's
byte for byte: the numpy restatement (oracle/oracle_lsq_np.py, pinned to the reference by tests/test_lsq_oracle.py)
and, where it is built, the live reference library.  On float data the total error agrees with the CPU's to 1e-3.
Results do not depend on pointer residency, the page budget, how n is split over calls, or the device count."""
import numpy as np
import pytest

from oracle import oracle_lsq_np as lo
from tests.golden import make_golden_lsq as g

fb = pytest.importorskip("faiss_b200")


def _ref():
    from oracle import ref_lsq

    return ref_lsq if ref_lsq.available() else None


@pytest.fixture(scope="module")
def res():
    return fb.StandardGpuResources()


def _draws(M, K, nperts, n, ils, seed):
    return lo.draws(lo.MT19937(seed), M, K, nperts, n, ils)


def _encoder(res, cb, devices=(0,)):
    M, K, d = cb.shape
    enc = fb.GpuIcmEncoder(M, K, d, res, devices)
    enc.setBinaryTerm(cb)
    return enc


def synthetic(d, n, seed=1338):
    # faiss.contrib.datasets.SyntheticDataset's generator
    rs = np.random.RandomState(seed)
    x = rs.normal(size=(n, 10))
    x = np.dot(x, rs.rand(10, d))
    x = x * (rs.rand(d) * 4 + 0.1)
    return np.sin(x).astype(np.float32)


def residual_codebooks(xt, M, K, seed=0):
    # a cheap additive codebook: each level is K rows of the previous level's residuals
    rs = np.random.RandomState(seed)
    r = xt.astype(np.float64)
    cbs = []
    for _ in range(M):
        c = r[rs.choice(r.shape[0], K, replace=False)]
        a = ((r[:, None, :] - c[None]) ** 2).sum(-1).argmin(1)
        r = r - c[a]
        cbs.append(c)
    return np.stack(cbs).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("M,K,d", [(4, 16, 32), (8, 256, 128), (3, 1024, 20)])
@pytest.mark.parametrize("nperts", [0, 4])
@pytest.mark.parametrize("ils", [1, 8])
def test_integer_data_equals_cpu(res, M, K, d, nperts, ils):
    nperts = min(nperts, M)  # the CPU requires nperts <= M
    n, icm = 300, 4
    rs = np.random.RandomState(M * 1000 + K + nperts + ils)
    cb, x = g.int_data(rs, M, K, d, n, 0)
    codes0 = rs.randint(0, K, (n, M)).astype(np.int32)
    seed = 4321 + ils
    perts = _draws(M, K, nperts, n, ils, seed)
    got = _encoder(res, cb).encode(codes0, x, perts, icm_iters=icm)
    want = lo.icm_encode(cb, codes0, x, perts, icm)
    assert np.array_equal(got, want)
    ref = _ref()
    if ref is not None:
        cpu, _ = ref.LSQ(cb, nperts=nperts, icm_iters=icm).icm_encode(codes0, x, ils, seed)
        assert np.array_equal(got, cpu)


@pytest.mark.gpu
@pytest.mark.parametrize("case", g.CASES, ids=[c[0] for c in g.CASES])
def test_golden_cases(res, case):
    # the reference-minted fixtures, forced ties included
    name, M, K, d, n, ils, nperts, icm, seed, _ = case
    gd = g.load()
    c = {k.split("/", 1)[1]: v for k, v in gd.items() if k.startswith(name + "/")}
    got = _encoder(res, c["cb"]).encode(c["codes0"], c["x"], c["perts"], icm_iters=icm)
    assert np.array_equal(got, c["codes"])


@pytest.mark.gpu
def test_float_data_error_matches_cpu(res):
    M, K, d = 4, 256, 32
    x = synthetic(d, 2000)
    xt, xb = x[:1000], x[1000:]
    cb = residual_codebooks(xt, M, K)
    n, ils, nperts, icm, seed = xb.shape[0], 16, 4, 4, 0x12345
    codes0 = np.random.RandomState(1).randint(0, K, (n, M)).astype(np.int32)
    perts = _draws(M, K, nperts, n, ils, seed)
    got = _encoder(res, cb).encode(codes0, xb, perts, icm_iters=icm)
    err_gpu = float(lo.evaluate(cb, got, xb).astype(np.float64).sum())
    ref = _ref()
    if ref is not None:
        cpu, _ = ref.LSQ(cb, nperts=nperts, icm_iters=icm).icm_encode(codes0, xb, ils, seed)
    else:
        cpu = lo.icm_encode(cb, codes0, xb, perts, icm)
    err_cpu = float(lo.evaluate(cb, cpu, xb).astype(np.float64).sum())
    assert err_gpu <= 1.05 * err_cpu
    # same walk, same draws: only last-bit differences in the sums can make a row take another path
    assert abs(err_gpu - err_cpu) <= 1e-3 * err_cpu, (err_gpu, err_cpu, float((got == cpu).all(1).mean()))


@pytest.mark.gpu
def test_invariance_residency_paging_splits(res):
    import torch

    M, K, d, n, ils, nperts, icm = 8, 64, 40, 1000, 4, 3, 3
    x = synthetic(d, n, seed=7)
    cb = residual_codebooks(x, M, K, seed=3)
    codes0 = np.random.RandomState(2).randint(0, K, (n, M)).astype(np.int32)
    perts = _draws(M, K, nperts, n, ils, 11)
    enc = _encoder(res, cb)
    base = enc.encode(codes0, x, perts, icm_iters=icm)
    # device-resident inputs and output
    dev = enc.encode(torch.from_numpy(codes0).cuda(), torch.from_numpy(x).cuda(), torch.from_numpy(perts).cuda(), icm_iters=icm)
    assert np.array_equal(dev.cpu().numpy(), base)
    # a page budget of a few rows, and of one row
    per_row = 4 * (M * K + d + M) + 8 * ils * nperts
    for rows in (37, 1):
        assert np.array_equal(enc.encode(codes0, x, perts, icm_iters=icm, page_bytes=rows * per_row), base)
    # n split over calls
    parts = [enc.encode(codes0[a:b], x[a:b], perts[:, a:b], icm_iters=icm) for a, b in ((0, 1), (1, 400), (400, n))]
    assert np.array_equal(np.concatenate(parts), base)
    # codebooks given on the device
    enc2 = fb.GpuIcmEncoder(M, K, d, res)
    enc2.setBinaryTerm(torch.from_numpy(cb).cuda())
    assert np.array_equal(enc2.encode(codes0, x, perts, icm_iters=icm), base)


@pytest.mark.gpu
def test_limits_throw_and_leave_the_encoder_usable(res):
    with pytest.raises(fb.FaissError, match="1 <= K <= 1024"):
        fb.GpuIcmEncoder(2, 1025, 8, res)
    M, K, d, n = 3, 16, 8, 50
    rs = np.random.RandomState(0)
    cb, x = g.int_data(rs, M, K, d, n, 0)
    codes0 = rs.randint(0, K, (n, M)).astype(np.int32)
    enc = fb.GpuIcmEncoder(M, K, d, res)
    with pytest.raises(fb.FaissError, match="setBinaryTerm"):
        enc.encode(codes0, x, _draws(M, K, 2, n, 2, 1))
    enc.setBinaryTerm(cb)
    with pytest.raises(fb.FaissError, match="nperts"):
        enc.encode(codes0, x, np.zeros((2, n, M + 1, 2), np.int32))
    bad = _draws(M, K, 2, n, 2, 1)
    bad[1, 7, 0, 0] = M
    with pytest.raises(fb.FaissError, match="perturbation"):
        enc.encode(codes0, x, bad)
    bad_codes = codes0.copy()
    bad_codes[3, 1] = K
    with pytest.raises(fb.FaissError, match="input code"):
        enc.encode(bad_codes, x, _draws(M, K, 2, n, 2, 1))
    perts = _draws(M, K, 2, n, 2, 1)
    assert np.array_equal(enc.encode(codes0, x, perts), lo.icm_encode(cb, codes0, x, perts, 4))


@pytest.mark.gpu
def test_multi_gpu_equals_one_gpu():
    import torch

    ng = torch.cuda.device_count()
    if ng < 2:
        pytest.skip("needs 2 or more GPUs")
    M, K, d, n, ils, nperts, icm = 8, 256, 64, 3001, 4, 4, 4
    x = synthetic(d, n, seed=9)
    cb = residual_codebooks(x, M, K, seed=4)
    codes0 = np.random.RandomState(3).randint(0, K, (n, M)).astype(np.int32)
    perts = _draws(M, K, nperts, n, ils, 5)
    one = _encoder(fb.StandardGpuResources(), cb).encode(codes0, x, perts, icm_iters=icm)
    for k in sorted({2, ng}):
        ress = [fb.StandardGpuResources() for _ in range(k)]
        got = _encoder(ress, cb, devices=list(range(k))).encode(codes0, x, perts, icm_iters=icm)
        assert np.array_equal(got, one), k
    with pytest.raises(fb.FaissError, match="of its own"):
        r = fb.StandardGpuResources()
        fb.GpuIcmEncoder(M, K, d, [r, r], [0, 1])
