"""Device memory of the tensor-core Flat database (DESIGN.md 2): after a search, FlatData holds the stored rows and the
one layout that search scanned, with the byte counts its shapes give.  An int8 database that fails the fitness test
gives the int8 layout's memory back and keeps only its centre beside the fp16 layout."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ALIGN = 256  # every device allocation is rounded up to 256 bytes


def _layout(n, row_bytes, sorted_rows):
    """rows, bias [round_up(n, 256) + 256], tile bias [2 (T + 1)] and, when the rows are sorted, perm [n]"""
    pad_rows = -(-n // 256) * 256 + 256
    sizes = [n * row_bytes, 4 * pad_rows, 4 * 2 * (pad_rows // 256)]
    if sorted_rows:
        sizes.append(4 * n)
    return sizes


def _expected(sizes):
    return len(sizes), sum(-(-s // ALIGN) * ALIGN for s in sizes)


def _int8_unfit(xb):
    out = xb.copy()
    out[7, 3] = 1e6  # one huge coordinate collapses s_y: every ordinary row would quantise to zero
    return out


# metric, d, k, data, operand bits of the search, the FlatData allocations beside the stored rows
CASES = {
    "fp16_l2": ("L2", 96, 10, None, 16, lambda n, d: _layout(n, 2 * 128, True)),
    "fp16_ip": ("IP", 96, 10, None, 16, lambda n, d: _layout(n, 2 * 128, False)),
    "int8": ("L2", 128, 100, None, 8, lambda n, d: _layout(n, 128, True) + [4 * d]),
    "int8_unfit": ("L2", 128, 100, _int8_unfit, 16, lambda n, d: _layout(n, 2 * 128, True) + [4 * d]),
}


@pytest.mark.parametrize("case", list(CASES))
def test_flat_data_bytes_follow_the_layout_shapes(case):
    import faiss_b200 as fb

    metric, d, k, transform, bits, extra = CASES[case]
    rs = np.random.RandomState(d + k)
    n = 70000 + 37  # a partial last tile
    xb = rs.rand(n, d).astype(np.float32)
    if transform is not None:
        xb = transform(xb)
    xq = rs.rand(64, d).astype(np.float32)
    res = fb.StandardGpuResources()  # its own: FlatData then counts this index alone
    idx = (fb.GpuIndexFlatL2 if metric == "L2" else fb.GpuIndexFlatIP)(res, d)
    idx.add(xb)
    rows = [4 * n * d]
    assert res.getMemoryInfo()[0]["FlatData"] == _expected(rows)  # layouts are built by the first search
    for _ in range(2):  # the second search reuses the prepared layout
        idx.search(xq, k)
        assert idx.lastSearchInfo()["tensor_cores"] == 1
        assert idx.lastSearchOperandBits() == bits
        assert res.getMemoryInfo()[0]["FlatData"] == _expected(rows + extra(n, d)), case
    del idx
