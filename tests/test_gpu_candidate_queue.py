"""GPU: the seeded 256-query tensor-core scans (kernels 6, 8, 9) hand candidate chunks from the MMA warps to list warps through a
shared-memory queue; unseeded ones insert in the MMA warps (vec_scan_tc.cu).  Ids and scores against the oracle on both sides: the
seeded scan (>= 65536 rows), the unseeded insert storm (< 65536 rows), a delete set (no seed), an IVF-clustered index (no seed), paging
to k = 100 (seeded) and a corpus where every row is a candidate for every query, so that the queue fills and the MMA warps wait for room."""
import numpy as np
import pytest

from oracle import oracle as O
from seekstorm_b200 import synth
from helpers_ivf import clustered_levels

pytestmark = pytest.mark.gpu

RTOL = 1e-4
KERNELS = [6, 8, 9]


def _check(got, want):
    assert len(got) == len(want), (got, want)
    gs = np.array([s for _, s in got], dtype=np.float64)
    ws = np.array([s for _, s in want], dtype=np.float64)
    assert np.allclose(gs, ws, rtol=RTOL, atol=1e-6), (got, want)
    for (gd, gsc), (wd, wsc) in zip(got, want):
        if gd != wd:   # ids may only differ inside a near-tie group (the score tolerance of allclose above)
            assert abs(gsc - wsc) <= RTOL * abs(wsc) + 1e-6, (got, want)


def _index(kernel, rows):
    from seekstorm_b200 import Index, VectorSimilarity
    ix = Index(0, vector_dims=rows.shape[1], vector_similarity=VectorSimilarity.Cosine, vector_kernel=kernel)
    ix.add_vectors(rows)
    return ix


def _queries(rows, nq, seed):
    qs = synth.gen_vectors(nq, rows.shape[1], seed, "cpu").numpy()
    qs[:8] = rows[:: len(rows) // 8][:8] + 0.05 * qs[:8]     # a few queries with a clear nearest row
    return qs


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("n", [70000, 20000])
def test_queue_seeded_and_unseeded(kernel, n):
    """70000 rows: the threshold-seeded scan; 20000 rows: no seed, every row passes on the first tiles (insert storm)."""
    dims = 96
    rows = synth.gen_vectors(n, dims, 9100 + n, "cpu").numpy()
    qs = _queries(rows, 200, 9200 + n)
    ix = _index(kernel, rows)
    nrows = np.stack([O.normalize(r) for r in rows])
    for k in (1, 10, 16):
        got = ix.search_vector_batch(qs, k)
        for i in list(range(8)) + list(range(8, 200, 13)):
            _check(got[i], O.search_vector(nrows, O.normalize(qs[i]), k, O.SIM_COSINE))
    ix.close()


@pytest.mark.parametrize("kernel", KERNELS)
def test_queue_delete_set(kernel):
    """A delete set turns the seed off: deleted rows never come back."""
    n, dims = 70000, 64
    rows = synth.gen_vectors(n, dims, 9300, "cpu").numpy()
    qs = _queries(rows, 180, 9301)
    ix = _index(kernel, rows)
    nrows = np.stack([O.normalize(r) for r in rows])
    first = ix.search_vector_batch(qs[:8], 1)
    top = [first[i][0][0] for i in range(8)]
    rng = np.random.default_rng(9302)
    deleted = sorted(set(rng.choice(n, size=3000, replace=False).tolist()) | set(top))
    ix.set_deleted(deleted)
    keep = np.ones(n, dtype=bool)
    keep[deleted] = False
    ids = np.nonzero(keep)[0].astype(np.uint32)
    dset = set(deleted)
    got = ix.search_vector_batch(qs, 10)
    for i in range(len(qs)):
        assert not dset.intersection(d for d, _ in got[i]), i
    for i in list(range(8)) + list(range(8, 180, 11)):
        _check(got[i], O.search_vector(nrows[keep], O.normalize(qs[i]), 10, O.SIM_COSINE, doc_ids=ids))
    ix.close()


@pytest.mark.parametrize("kernel", KERNELS)
def test_queue_ivf(kernel):
    """IVF cluster mask per (query, row)."""
    from seekstorm_b200 import Index, VectorSimilarity
    dims = 64
    levels = clustered_levels(dims, [(40000, 24), (30000, 9)], seed=9400)
    ix = Index(0, vector_dims=dims, vector_similarity=VectorSimilarity.Cosine, vector_kernel=kernel)
    olevels = []
    for lid, rows, counts in levels:
        ix.add_vector_level(lid, rows, None, counts)
        olevels.append((lid, np.stack([O.normalize(r) for r in rows]), None, counts))
    rng = np.random.default_rng(9401)
    allr = np.concatenate([lv[1] for lv in levels])
    qs = rng.normal(size=(160, dims)).astype(np.float32)
    qs[:80] = allr[rng.choice(len(allr), size=80, replace=False)] + 0.3 * qs[:80]
    for mode, n_probe, thr in ((1, 3, 0.0), (3, 2, 0.50001)):
        got, _, observed = ix.search_vector_ex(qs, 10, ann_mode=mode, n_probe=n_probe, cluster_threshold=thr)
        for i in range(0, len(qs), 9):
            want, obs = O.search_vector_ivf(olevels, O.normalize(qs[i]), 10, O.SIM_COSINE, mode, n_probe, thr)
            assert int(observed[i]) == obs
            _check(got[i], want)
    ix.close()


def test_queue_paging_kernel6():
    """k = 100 on the exact 256-query scan: pages of 32 whose paging ceilings are applied by the list warps."""
    n, dims = 70000, 64
    rows = synth.gen_vectors(n, dims, 9500, "cpu").numpy()
    qs = _queries(rows, 150, 9501)
    ix = _index(6, rows)
    nrows = np.stack([O.normalize(r) for r in rows])
    got = ix.search_vector_batch(qs, 100)
    for i in list(range(8)) + list(range(8, 150, 17)):
        _check(got[i], O.search_vector(nrows, O.normalize(qs[i]), 100, O.SIM_COSINE))
    ix.close()


@pytest.mark.parametrize("kernel", KERNELS)
def test_queue_backpressure_near_identical_rows(kernel):
    """Every row is a near-copy of one vector (70000 rows: seeded): every row passes for every query on every tile, the queue fills and
    the MMA warps wait.
    The filter scans cannot fit the candidates into 32 entries and hand the queries to the exact fallback."""
    n, dims = 70000, 64
    rng = np.random.default_rng(9600)
    base = synth.gen_vectors(1, dims, 9601, "cpu").numpy()[0]
    rows = (base + 1e-4 * rng.normal(size=(n, dims))).astype(np.float32)
    qs = synth.gen_vectors(140, dims, 9602, "cpu").numpy()
    qs[:4] = base + 0.01 * qs[:4]
    ix = _index(kernel, rows)
    nrows = np.stack([O.normalize(r) for r in rows])
    got = ix.search_vector_batch(qs, 10)
    if kernel in (8, 9):
        assert ix.last_stats()["filter_fallbacks"] > 0
    for i in list(range(4)) + list(range(4, 140, 15)):
        _check(got[i], O.search_vector(nrows, O.normalize(qs[i]), 10, O.SIM_COSINE))
    ix.close()
