"""The CPU restatement of the merge step's t-digest fold (tests.util.td_merge_compress / td_fold), checked against the oracle's own
batch update: gyo_td_add_batch is a stable merge of the old centroids with the batch's bin items followed by gyo_td_compress, so the
restatement must reproduce it bit for bit. The GPU merge tests pin fold_td_kernel and finish_td_kernel to this restatement."""
import numpy as np
import pytest

from oracle import pyoracle as po
from tests.util import Digest, td_batch_items, td_fold, td_merge_compress


def _lognormal(rng, n):
    return np.minimum(np.exp(rng.normal(np.log(2000.0), 1.5, n)), 9.0e8).astype(np.uint32)


def _cent(pairs):
    c = np.zeros(len(pairs), dtype=po.CENTROID_DTYPE)
    for i, (m, w) in enumerate(pairs):
        c[i] = (m, w)
    return c


def _same(a, b):
    return len(a) == len(b) and np.array_equal(a["weight"], b["weight"]) and a["mean"].tobytes() == b["mean"].tobytes()


@pytest.mark.parametrize("delta", [10, 100, 200, 256])
def test_merge_compress_restates_add_batch(delta):
    rng = np.random.default_rng(1000 + delta)
    td = po.td_new()
    cent = np.zeros(0, dtype=po.CENTROID_DTYPE)
    for b in range(4):
        vals = _lognormal(rng, 20_000)
        po.td_add(td, vals, float(delta))
        cent = td_merge_compress(cent, td_batch_items(vals), delta)
        want = Digest.of_oracle(td)
        assert _same(cent, want.cent), (delta, b, len(cent), len(want.cent))
        assert want.total == 20_000 * (b + 1)
        assert 0 < len(cent) <= delta
    assert len(cent) > delta // 2


@pytest.mark.parametrize("delta", [10, 200, 256])
def test_merge_with_an_empty_list_is_one_compress(delta):
    rng = np.random.default_rng(delta)
    items = td_batch_items(_lognormal(rng, 50_000))
    assert len(items) > delta                     # the compress pass has to cut the list
    once = po.td_compress(items, delta)
    empty = np.zeros(0, dtype=po.CENTROID_DTYPE)
    assert _same(td_merge_compress(empty, items, delta), once)
    assert _same(td_merge_compress(items, empty, delta), once)
    assert len(td_merge_compress(empty, empty, delta)) == 0
    # the fold of one digest is that compress too (the accumulator starts empty); empty digests are skipped
    d = td_fold([Digest(), Digest(items, int(items["weight"].sum()), 3.0, 9.0e5), Digest()], delta)
    assert _same(d.cent, once) and d.total == int(items["weight"].sum()) and (d.minv, d.maxv) == (3.0, 9.0e5)
    z = td_fold([Digest(), Digest()], delta)
    assert len(z.cent) == 0 and z.total == 0 and np.isnan(z.quantile(0.5))


def test_equal_means_take_the_first_list_first():
    """three unit weights and one weight of 50, all at the same mean: which list goes first decides where the K_1 cells cut"""
    a = _cent([(7.0, 1), (7.0, 1), (7.0, 1)])
    b = _cent([(7.0, 50)])
    a_first = po.td_compress(np.concatenate([a, b]), 10)
    b_first = po.td_compress(np.concatenate([b, a]), 10)
    assert a_first["weight"].tolist() != b_first["weight"].tolist()
    assert _same(td_merge_compress(a, b, 10), a_first)
    assert _same(td_merge_compress(b, a, 10), b_first)
    # ties inside a longer merge: a's entry of an equal pair always precedes b's
    a = _cent([(1.0, 2), (4.0, 1), (4.0, 3), (9.0, 5)])
    b = _cent([(0.5, 1), (4.0, 7), (9.0, 1), (12.0, 2)])
    merged = _cent([(0.5, 1), (1.0, 2), (4.0, 1), (4.0, 3), (4.0, 7), (9.0, 5), (9.0, 1), (12.0, 2)])
    assert _same(td_merge_compress(a, b, 256), po.td_compress(merged, 256))
