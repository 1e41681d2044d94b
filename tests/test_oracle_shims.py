"""The oracle's error path: a reference exception thrown inside a shim library (oracle/_ref/libfaiss_ref_<name>.so)
is caught there by oracle/ref_shim.h, stored in libfaiss_ref.so's one error slot and raised by oracle.ref._ck as a
RuntimeError that carries the reference's own message.  Calls into different shim libraries alternate, so a stale
message from an earlier call would show."""
import numpy as np
import pytest

from oracle import ref_pairwise, ref_rq, ref_sq


def _need(mod):
    if not mod.available():
        pytest.skip("%s not built (needs the reference tree at build time)" % mod.LIB_PATH)


def test_reference_errors_reach_python_from_every_shim_library(ref):
    for mod in (ref_rq, ref_sq, ref_pairwise):
        _need(mod)
    x = np.zeros((4, 8), np.float32)

    # ResidualQuantizer without codebooks is untrained (faiss/impl/ResidualQuantizer.cpp compute_codes_add_centroids,
    # faiss/impl/AdditiveQuantizer.cpp decode)
    rq = ref_rq.RQ(8, [4, 4])
    with pytest.raises(RuntimeError, match="RQ is not trained yet"):
        rq.compute_codes(x)

    # a TurboQuant-MSE scalar quantizer whose trained table has the wrong size: select_quantizer's Lloyd-Max quantizer
    # checks trained.size() == 2 * 2^nbits - 1 (faiss/impl/scalar_quantizer/quantizers.h)
    QT_1bit_tqmse = 10
    sq = ref_sq.IndexIVFScalarQuantizer(8, 1, QT_1bit_tqmse, by_residual=False)
    sq.set_trained(np.zeros(5, np.float32))
    with pytest.raises(RuntimeError, match=r"trained\.size\(\) == 2 \* kCentroidsCount - 1"):
        sq.encode(x, np.full(4, -1, np.int64))

    with pytest.raises(RuntimeError, match="The additive quantizer is not trained yet"):
        rq.decode(np.zeros((4, rq.code_size), np.uint8))

    # a metric the reference does not know (faiss/utils/extra_distances.h with_metric_type)
    with pytest.raises(RuntimeError, match="unknown metric 999"):
        ref_pairwise.pairwise(x, x, 999)
