"""CPU: host-side logic — synthetic generators, term keys, packed-key order, query parsing helpers."""
import struct

import numpy as np
import torch

from seekstorm_b200 import synth
from seekstorm_b200.index import fnv1a64, synthetic_term_key


def test_term_keys_np_torch_python_agree():
    ids = np.array([0, 1, 2, 12345, 999999, 2**31 - 1], dtype=np.int64)
    a = synth.term_keys_np(ids)
    b = synth.term_keys_torch(torch.from_numpy(ids)).numpy().view(np.uint64)
    c = np.array([synth.splitmix64(int(i)) & ~7 for i in ids], dtype=np.uint64)
    assert (a == b).all() and (a == c).all()
    assert (a & np.uint64(7) == 0).all()
    assert synthetic_term_key("t12345") == int(a[3])
    assert synthetic_term_key("hello") == fnv1a64("hello")


def test_level_generator_invariants():
    lv = synth.gen_level(3, 5000, 2000, 42)
    n = lv.to_numpy()
    offs, ids, tfs = n["posting_offsets"], n["doc_ids"], n["tfs"]
    assert offs[0] == 0 and offs[-1] == len(ids) == len(tfs)
    assert (np.diff(offs.astype(np.int64)) > 0).all()
    for t in range(0, len(offs) - 1, 97):
        seg = ids[offs[t]:offs[t + 1]].astype(np.int64)
        assert (np.diff(seg) > 0).all()          # ascending, unique
        assert seg.max() < 5000
    assert tfs.min() >= 1
    # token conservation: Σ tf == Σ doc lengths (exact lengths before byte4 compression are in [8, 2000])
    lens = np.array([synth.byte4_to_int(int(b)) for b in n["doc_len_bytes"]])
    assert lens.sum() == lv.len_sum_normalized
    assert int(tfs.astype(np.int64).sum()) >= lens.sum()   # byte4 never over-estimates
    # determinism
    lv2 = synth.gen_level(3, 5000, 2000, 42)
    assert torch.equal(lv.doc_ids, lv2.doc_ids) and torch.equal(lv.term_keys, lv2.term_keys)


def test_query_generator():
    qs = synth.gen_queries(200, 5, 20, 20000, (2, 3, 4), (0.4, 0.4, 0.2))
    assert all(len(set(q)) == len(q) for q in qs)
    assert all(19 <= t <= 19999 for q in qs for t in q)
    assert {len(q) for q in qs} == {2, 3, 4}


def _ord(f):
    u = struct.unpack("<I", struct.pack("<f", f))[0]
    return (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)


def test_packed_key_order_is_canonical():
    """key = ord(score)<<32 | (0xFFFFFFFF - doc): larger key <=> (score desc, doc id asc)."""
    rng = np.random.default_rng(0)
    items = [(float(np.float32(s)), int(d)) for s, d in zip(rng.normal(size=200), rng.integers(0, 1000, 200))]
    items += [(1.5, 7), (1.5, 3), (-0.0, 1), (0.0, 2), (-2.0, 9)]
    keyed = sorted(items, key=lambda x: -((_ord(x[0]) << 32) | (0xFFFFFFFF - x[1])))
    canon = sorted(items, key=lambda x: (-x[0], x[1]))
    # -0.0 and 0.0 compare equal as floats but order by sign bit in the key; exclude that pair from the check
    strip = lambda l: [x for x in l if x[0] != 0.0]
    assert strip(keyed) == strip(canon)


def test_lex_bound_inflation_covers_rounding():
    """The OR fast path of lex_score (bm25.cu) filters postings with the bound
        (approx(cd) + sum of upper bounds of the other present terms) * (1 + 2e-6) >= theta
    where approx(cd) = (idf*(K+1)) * fdividef(tf, tf + cache) uses an approximate reciprocal (<= 2 ulp) and a different
    association than the exact score idf * ((tf*(K+1)) / (tf + cache)), and the exact score is summed in QUERY order while
    the bound adds driver first.  Property: with the tightest admissible term bounds (ub == the term's exact contribution)
    and the approximate quotient pushed 2 ulp DOWN, the inflated bound still dominates the exact in-order f32 score."""
    f32 = np.float32
    rng = np.random.default_rng(11)
    k1p = f32(1.2) + f32(1.0)

    def down(x, n):
        for _ in range(n):
            x = np.nextafter(f32(x), f32(-np.inf))
        return f32(x)

    worst = 0.0
    for _ in range(20000):
        n = int(rng.integers(1, 5))
        idf = [f32(rng.uniform(0.05, 14.0)) for _ in range(n)]
        tf = [f32(rng.integers(1, 256)) for _ in range(n)]
        cache = [f32(rng.uniform(0.3, 4.0)) for _ in range(n)]
        present = [True] + [bool(rng.integers(0, 2)) for _ in range(n - 1)]
        drv = int(rng.integers(0, n))
        present[drv] = True
        contrib = [f32(idf[t] * f32(f32(tf[t] * k1p) / f32(tf[t] + cache[t]))) for t in range(n)]   # comp_of + term_score
        score = f32(0.0)
        for t in range(n):                                   # exact score: query order, from 0.0
            if present[t]:
                score = f32(score + contrib[t])
        didf_k = f32(idf[drv] * k1p)
        quot = down(f32(tf[drv] / f32(tf[drv] + cache[drv])), 2)      # fdividef: up to 2 ulp below the rounded quotient
        B = f32(didf_k * quot)
        for t in range(n):                                   # bound: driver first, then the other present terms
            if t != drv and present[t]:
                B = f32(B + contrib[t])
        assert f32(B * f32(1.000002)) >= score, (n, drv, float(B), float(score))
        worst = max(worst, float(score) / float(B) - 1.0)
    assert worst < 2e-6                                      # the slack actually needed stays well inside the inflation


def test_group_maximum_threshold_is_a_valid_lower_bound():
    """Threshold seeding of the tensor-core scans (vec_scan_tc.cu, sample mode): the k-th largest of the per-32-row-group maxima is
    never above the true k-th best score (k disjoint groups each hold a row at least that good), and for k << #groups it is
    close to the exact k-th of the sample."""
    rng = np.random.default_rng(12)
    for n_groups, k in ((1184, 10), (1184, 32), (64, 10), (16, 10), (8, 10)):
        scores = rng.normal(size=(n_groups, 32)).astype(np.float32)
        gmax = np.sort(scores.max(axis=1))[::-1]
        exact = np.sort(scores.ravel())[::-1]
        if n_groups >= k:
            seed = gmax[k - 1]
            assert seed <= exact[k - 1]
            # rank of the seed inside the sample: what the full scan pays for the looser bound
            rank = int((exact > seed).sum())
            assert rank >= k - 1
            if n_groups >= 64 * k // 10:
                assert rank <= 2 * k + 4
        # fewer groups than k: kth_from_groupmax returns "no threshold" (0), nothing to check


def test_filter_scan_margin_bounds_the_fp16_error():
    """Filter vector scan (vec_scan_tc.cu PREC_F16F + vec_refine.cu): with h() = round-to-fp16 of the power-of-two-scaled vectors,
    |a.b - h(a).h(b)| <= E_a |b| + H_a |b - h(b)| with the row maxima E_a = max|a - h(a)|, H_a = max|h(a)|; hence every exact top-k row has
    an approximate score >= (k-th best approximate) - 2 eps.  The kernel's f32 arithmetic restated in numpy."""
    rng = np.random.default_rng(21)
    f32 = np.float32
    for n, d, norm in ((4000, 768, True), (3000, 100, False), (2000, 32, False)):
        a = rng.normal(size=(n, d)).astype(np.float32) * (1.0 if norm else rng.uniform(0.1, 30.0, size=(n, 1)).astype(np.float32))
        if norm:
            a /= np.linalg.norm(a, axis=1, keepdims=True).astype(np.float32)
        b = rng.normal(size=(24, d)).astype(np.float32)
        b[3] = a[n // 2] + 0.05 * b[3]
        if norm:
            b /= np.linalg.norm(b, axis=1, keepdims=True).astype(np.float32)
        sa = f32(256.0) if norm else f32(2.0 ** (7 - int(np.floor(np.log2(np.abs(a[:1500]).max())))))   # Dot: from the first level
        h = lambda x: x.astype(np.float16).astype(np.float32)
        a_s = a * sa
        ah = h(a_s)
        assert np.isfinite(ah).all()
        Ea = f32(np.sqrt(((a_s - ah).astype(np.float64) ** 2).sum(1)).max()) * f32(1.00001)
        Ha = f32(np.sqrt((ah.astype(np.float64) ** 2).sum(1)).max()) * f32(1.00001)
        for j in range(b.shape[0]):
            sb = f32(2.0 ** (7 - int(np.floor(np.log2(np.abs(b[j]).max())))))
            b_s = b[j] * sb
            bh = h(b_s)
            exact = a_s.astype(np.float64) @ b_s.astype(np.float64)
            approx = (ah @ bh).astype(np.float64)                        # f32 accumulation like the tensor core (order differs: covered by the slack)
            nb = f32(np.linalg.norm(b_s)) * f32(1.00001); eb = f32(np.linalg.norm(b_s - bh)) * f32(1.00001)
            eps = (Ea * nb + Ha * eb + f32(d) * f32(2.0 ** -22) * Ha * nb) * f32(1.001)
            err = np.abs(exact - approx).max()
            assert err <= eps, (n, d, j, err, eps)
            for k in (1, 10, 16):
                kth = np.sort(approx)[::-1][k - 1]
                cand = set(np.nonzero(approx >= kth - 2.0 * float(eps))[0].tolist())
                top = set(np.argsort(-exact, kind="stable")[:k].tolist())
                assert top <= cand
                if norm and d == 768:
                    assert len(cand) <= k + 6, (k, len(cand))          # the bound is not wasteful: the candidate set fits the 32-entry list


def test_turboquant_oracle_against_a_hadamard_matrix():
    """orc_turboquant_i8 (the scalar TurboQuant::quantize_f32_i8, vector_similarity.rs:1929-1958): its butterfly FWHT equals the Sylvester
    Hadamard matrix / sqrt(dim) in f64, scale = max(||x|| / sqrt(dim) / 32, 1e-8), codes round(x / scale) clamped to +-127,
    norm = sum(code^2) * scale^2; the quantised dot estimates the f32 dot; an all-zero vector takes the 1e-8 floor."""
    from scipy.linalg import hadamard
    from oracle import oracle as O
    rng = np.random.default_rng(3)
    for d, dim in ((100, 128), (768, 1024), (64, 64), (5, 8)):
        mask = np.where(rng.random(dim) < 0.5, 1.0, -1.0).astype(np.float32)
        rows = (rng.normal(size=(6, d)) * 0.7).astype(np.float32)
        rows[5] = 0
        c, s, nrm = O.turboquant_rows_i8(rows, mask)
        x = np.zeros((6, dim)); x[:, :d] = rows; x *= mask
        y = x @ (hadamard(dim).astype(np.float64) / np.sqrt(dim)).T
        sc = np.maximum(np.linalg.norm(y, axis=1) / np.sqrt(dim) / 32, 1e-8)
        want = np.clip(np.round(y / sc[:, None]), -127, 127)
        assert np.abs(want - c).max() <= 1 and (want != c).mean() < 0.01          # f32 vs f64 rounding at .5 boundaries only
        assert np.allclose(s, sc, rtol=1e-5) and s[5] == np.float32(1e-8) and not c[5].any()
        assert np.allclose(nrm, (c.astype(np.int64) ** 2).sum(1) * s.astype(np.float64) ** 2, rtol=1e-5)
        est = (c[:5].astype(np.int32) @ c[0].astype(np.int32)) * s[:5] * s[0]
        ref = rows[:5] @ rows[0]
        assert np.abs(est - ref).max() < 0.05 * np.abs(ref).max() + 0.05
    # Cosine: normalize_f32 first
    c1, s1, _ = O.turboquant_rows_i8(rows[:2], mask, True)
    c2, s2, _ = O.turboquant_rows_i8(np.stack([O.normalize(rows[0]), O.normalize(rows[1])]), mask, False)
    assert (c1 == c2).all() and (s1 == s2).all()


def test_affine_sq_oracle_is_lossless_on_sift_like_data():
    """new_scale_norm_affine (vector_similarity.rs:1414-1463) on integer 0..255 data: once the running range has reached 255 the scale is 1 and
    the zero point -128, codes are x - 128 and -euclidean_i8_quantized_affine equals the exact negated squared distance; before that the state
    follows the reference's update rule (the stored maximum is the RASTERED range)."""
    from oracle import oracle as O
    rng = np.random.default_rng(8)
    rows = np.clip(np.abs(rng.normal(0, 45, (200, 128))).round(), 0, 255).astype(np.float32)
    rows[0] = np.clip(rows[0], 3, 90)                    # first vector: min 3, max 90 -> range raster(87) = 127, scale 127/255
    rows[1, 0] = 0; rows[1, 1] = 255
    c, s, nrm, zp, sq, st = O.quantize_affine_rows_i8(rows)
    assert s[0] == np.float32(127.0) / np.float32(255.0) and zp[0] == -128          # -128 - 3/scale = -134 -> clamped
    assert st == (0.0, 255.0) and (s[1:] == 1.0).all() and (zp[1:] == -128).all()
    assert (c[1:].astype(np.int32) == rows[1:].astype(np.int32) - 128).all()
    q = np.clip(rows[50] + rng.integers(-3, 4, 128), 0, 255).astype(np.float32)
    qc, qs, qn, qz, qsum, _ = O.quantize_affine_rows_i8(q[None], st, False)
    hits = O.search_vector_i8_affine(c[1:], s[1:], nrm[1:], zp[1:], sq[1:], qc[0], qs[0], qn[0], qz[0], qsum[0], 5)
    exact = sorted(((-float(((rows[1 + i] - q) ** 2).sum()), i) for i in range(199)), key=lambda t: (-t[0], t[1]))[:5]
    assert [(d, s_) for d, s_ in hits] == [(i, sc) for sc, i in exact]
    # raster_range: ranges above 1 widen to 2^m - 1
    r2 = np.array([[0, 1, 2, 40]], dtype=np.float32)
    _, s2, _, z2, _, st2 = O.quantize_affine_rows_i8(np.pad(r2, ((0, 0), (0, 4))))
    assert s2[0] == np.float32(63.0) / np.float32(255.0) and st2 == (0.0, 63.0)
