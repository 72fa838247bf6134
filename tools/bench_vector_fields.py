"""Field-filtered vector search on multi-vector documents, C2 size: 1 M x 768 f32 Cosine rows from 250 K docs (2 fields x 2 chunks per
doc), 256 queries per step, k = 10.  The same rows are added twice, with and without field ids, and four rows are printed:

  (a) no mask on the tagged index, beside the untagged index (tagging must cost nothing unmasked)
  (b) a mask passing 50 % of the rows (field 0 of 2)
  (c) a mask passing 5 % of the rows (a third field that every 10th doc carries instead of field 1)
  (d) (b) with the vb results requested (ssb_hit_ext): adds the best-row step that names each hit's field / chunk

Per row: queries/s over --steps timed steps (host clock around the synchronous call), the scan kernel time of the last step
(ssb_stats.dominant_kernel_ns), filter fallbacks and kernel launches per step, and a check of a sample of queries against a float64
restatement on the device.  The card name, power limit and max SM clock are read in the same run.  One JSON line per row.

    python tools/bench_vector_fields.py [--docs 250000] [--dims 768] [--steps 20] [--warmup 3] [--kernel 0]

Nothing is written to disk."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from seekstorm_b200 import Index, VectorSimilarity, synth  # noqa: E402
from seekstorm_b200._lib import SsbHitExt, SsbVecQuery, check, lib  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def layout(n_docs, rare_every=10):
    """per row (doc, field, chunk) in record order: doc d has rows (field 0, chunk 0), (0, 1), (f1, 0), (f1, 1), where f1 = 2 on every
    `rare_every`-th doc (the ~5 % field) and 1 elsewhere"""
    n = 4 * n_docs
    i = np.arange(n)
    doc = i // 4
    field = ((i // 2) % 2).astype(np.uint8)
    chunk = (i % 2).astype(np.uint32)
    field[(field == 1) & (doc % rare_every == 0)] = 2
    return doc, field, chunk


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=250000)
    ap.add_argument("--dims", type=int, default=768)
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel", type=int, default=0)
    ap.add_argument("--check", type=int, default=16, help="queries per row checked against the float64 restatement")
    a = ap.parse_args()
    dev = torch.device("cuda")
    n = 4 * a.docs
    doc, field, chunk = layout(a.docs)
    rows = synth.gen_vectors(n, a.dims, 71, "cuda")
    qs = synth.gen_vectors(a.queries, a.dims, 72, "cpu").numpy()
    per_level = 65536                                        # rows per level = 16384 docs x 4
    tagged = Index(0, vector_dims=a.dims, vector_similarity=VectorSimilarity.Cosine, vector_kernel=a.kernel)
    plain = Index(0, vector_dims=a.dims, vector_similarity=VectorSimilarity.Cosine, vector_kernel=a.kernel)
    tagged.reserve_vectors(n); plain.reserve_vectors(n)
    for lv, s in enumerate(range(0, n, per_level)):
        e = min(n, s + per_level)
        loc = (doc[s:e] - doc[s]).astype(np.uint16)
        tagged.add_vector_level(lv, rows[s:e], loc, field_ids=field[s:e], chunk_ids=chunk[s:e])
        plain.add_vector_level(lv, rows[s:e], loc)
    doc_id = ((np.arange(n) // per_level) << 16) | (doc - (np.arange(n) // per_level) * (per_level // 4))
    rn = torch.nn.functional.normalize(rows.double(), dim=1)
    qn = torch.nn.functional.normalize(torch.from_numpy(qs).to(dev).double(), dim=1)
    info = card()

    def run(ix, mask, ext):
        nq, k = a.queries, a.k
        vq = SsbVecQuery(qs.ctypes.data, nq, k, 0, 0, 0.0, 0, 0, 0.0)
        hits = np.zeros(nq * k, dtype=[("doc_id", "<u8"), ("score", "<f4"), ("pad", "<u4")])
        nh = np.zeros(nq, dtype=np.uint32)
        ex = (SsbHitExt * (nq * k))() if ext else None
        fm = np.full(nq, mask, dtype=np.uint32)
        def step():
            check(lib().ssb_search_vector_fields(ix._h, C.byref(vq), fm.ctypes.data if mask else None, hits.ctypes.data, nh.ctypes.data,
                                                 C.addressof(ex) if ext else None, None))
        for _ in range(a.warmup):
            step()
        st = ix.last_stats()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            step()
        dt = time.perf_counter() - t0
        st = ix.last_stats()
        return hits, nh, ex, a.steps * nq / dt, st

    def verify(hits, nh, ex, mask):
        bad = 0
        for q in range(0, a.queries, max(1, a.queries // a.check)):
            s = (rn @ qn[q]).float()
            if mask:
                ok = torch.from_numpy(((mask >> field.astype(np.int64)) & 1) == 1).to(dev)
                s = torch.where(ok, s, torch.full_like(s, -np.inf))
            # best row per doc: scatter max over the 4 rows of a doc
            sd = s.view(-1, 4).max(dim=1)
            top = torch.topk(sd.values, a.k)
            want = [int(doc_id[4 * int(d)]) for d in top.indices.cpu()]
            got = [int(hits[q * a.k + j]["doc_id"]) for j in range(int(nh[q]))]
            bad += got != want
            if ex is not None and got == want:
                for j, d in enumerate(top.indices.cpu().tolist()):
                    r = 4 * d + int(sd.indices[d])
                    bad += (ex[q * a.k + j].field_id, ex[q * a.k + j].chunk_id) != (int(field[r]), int(chunk[r]))
        return bad

    for name, ix, mask, ext in (("a_untagged", plain, 0, False), ("a_tagged_nomask", tagged, 0, False), ("b_mask50", tagged, 0b001, False),
                                ("c_mask5", tagged, 0b100, False), ("d_mask50_ext", tagged, 0b001, True)):
        hits, nh, ex, qps, st = run(ix, mask, ext)
        r = dict(row=name, rows=n, docs=a.docs, dims=a.dims, queries=a.queries, k=a.k, kernel=a.kernel, qps=round(qps, 1),
                 scan_ms=round(st["dominant_kernel_ns"] / 1e6, 4), filter_fallbacks_per_step=st["filter_fallbacks"],
                 launches_per_step=st["kernel_launches"], rows_passing=int(n if not mask else ((mask >> field.astype(np.int64)) & 1).sum()),
                 check_mismatches=verify(hits, nh, ex, mask), card=info)
        print(json.dumps(r), flush=True)
    tagged.close(); plain.close()


if __name__ == "__main__":
    main()
