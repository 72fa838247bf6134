"""Phrase queries on a two-field index (title + body), device-resident throughput.

Builds a corpus from a seed on the GPU: N docs (2 M by default) in 64K-doc levels, each doc a short title and a longer body of Zipf(1) tokens
over the bench's vocabulary, with the positions of every token (per posting one run per field, field 0 first).  Each step searches 1024
phrases of 2-3 frequent terms (ranks log-uniform in [1, 300]) with QueryType::Phrase; W warm-up steps, then K steps timed with CUDA events.
Prints queries/s per result type, the dominant kernel's time (lex_generic) from ssb_last_stats, and the card's name and power limit read in
the same run.  One JSON line on stdout; --out also writes it to a file.

    python tools/bench_phrase_multifield.py --docs 2000000 --steps 20 --warmup 3
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from seekstorm_b200 import Index, QueryType, ResultType, synth  # noqa: E402

LEVEL_DOCS = 65536
VOCAB = 1_000_000
FIELDS = ((8.0, 2, 64), (80.0, 8, 2000))      # (mean length, min, max) of the title and the body: lognormal, sigma 0.6
BOOSTS = (2.0, 1.0)
TOPK = 10


def gen_level(level_id, n_docs, seed, dev, cdf):
    """one level with per-field tfs [np, F], doc_len_bytes [F, n_docs] and field-major positions, all on `dev`"""
    g = torch.Generator(device=dev)
    g.manual_seed(seed * 1000003 + level_id)
    b4, dlc = synth._luts(dev)
    keys, lbytes = [], []
    for f, (mean, lo, hi) in enumerate(FIELDS):
        ln = torch.randn(n_docs, generator=g, device=dev, dtype=torch.float32) * 0.6 + math.log(mean)
        lens = torch.exp(ln).round().clamp_(lo, hi).to(torch.int64)
        lbytes.append(b4[lens])
        n_tok = int(lens.sum().item())
        terms = torch.searchsorted(cdf, torch.rand(n_tok, generator=g, device=dev, dtype=torch.float64)).clamp_(max=VOCAB - 1)
        docs = torch.repeat_interleave(torch.arange(n_docs, device=dev, dtype=torch.int64), lens)
        pos = torch.arange(n_tok, device=dev, dtype=torch.int64) - (torch.cumsum(lens, 0) - lens)[docs]
        keys.append((((terms * LEVEL_DOCS + docs) * 4 + f) << 16) | pos)       # term | doc | field | position: one sort orders them all
    key, _ = torch.sort(torch.cat(keys))
    del keys
    pk, inv, _ = torch.unique_consecutive(key >> 18, return_inverse=True, return_counts=True)
    fld = (key >> 16) & 3
    tfs = torch.zeros(pk.numel() * len(FIELDS), dtype=torch.int64, device=dev)
    tfs.scatter_add_(0, inv * len(FIELDS) + fld, torch.ones_like(fld))
    positions = (key & 0xFFFF).to(torch.int32).to(torch.int16)
    del key, inv, fld
    p_term = pk // LEVEL_DOCS
    term_ids, counts = torch.unique_consecutive(p_term, return_counts=True)
    offs = torch.zeros(term_ids.numel() + 1, dtype=torch.int64, device=dev)
    offs[1:] = torch.cumsum(counts, 0)
    doc_len_bytes = torch.stack(lbytes).contiguous()
    return dict(level_id=level_id, n_docs=n_docs, term_keys=synth.term_keys_torch(term_ids), posting_offsets=offs.to(torch.int32),
                doc_ids=(pk - p_term * LEVEL_DOCS).to(torch.int32).to(torch.int16), tfs=tfs.view(-1, len(FIELDS)).to(torch.int16).contiguous(),
                doc_len_bytes=doc_len_bytes, positions=positions, len_sum=int(dlc[doc_len_bytes.to(torch.int64)].sum().item()))


def gpu_name_and_power_limit(index):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:      # the numbers are still printed; the card is then reported as unknown
        return f"unknown ({e!r})", "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--docs", type=int, default=2_000_000)
    p.add_argument("--queries", type=int, default=1024, help="phrases per step")
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--seed", type=int, default=1106)
    p.add_argument("--out", default=None, help="also write the JSON result here")
    a = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_phrase_multifield: needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device())
    card, power = gpu_name_and_power_limit(dev.index)
    ix = Index(dev.index, max_batch=a.queries)
    ix.set_stream(torch.cuda.current_stream().cuda_stream)
    ix.set_field_boosts(BOOSTS)
    t0 = time.perf_counter()
    cdf = synth.zipf_cdf(VOCAB, dev)
    ls, n_pos, n_post = 0, 0, 0
    for li in range((a.docs + LEVEL_DOCS - 1) // LEVEL_DOCS):
        lv = gen_level(li, min(LEVEL_DOCS, a.docs - li * LEVEL_DOCS), a.seed, dev, cdf)
        ix.add_lexical_level(lv["level_id"], lv["n_docs"], lv["term_keys"], lv["posting_offsets"], lv["doc_ids"], lv["tfs"], lv["doc_len_bytes"],
                             lv["positions"])
        ls += lv["len_sum"]; n_pos += lv["positions"].numel(); n_post += lv["doc_ids"].numel()
        del lv
    ix.commit(a.docs, ls)
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    rng = np.random.default_rng(a.seed + 1000)
    phrases = [[int(x) for x in np.floor(np.exp(rng.uniform(0, np.log(300), int(rng.integers(2, 4)))))] for _ in range(a.queries)]
    qk = [[int(k) for k in synth.term_keys_np(np.array(ph, dtype=np.int64))] for ph in phrases]
    b, keep = ix._lex_batch(qk, QueryType.Phrase)
    out_keys = torch.zeros((len(qk), 32), dtype=torch.int64, device=dev)
    cnt = torch.zeros(len(qk), dtype=torch.int64, device=dev)
    res = {"metric": "phrase_multifield_qps", "card": card, "power_limit": power,
           "config": {"docs": a.docs, "fields": "title (lognormal mean 8) + body (lognormal mean 80), boosts 2.0 / 1.0", "vocab": VOCAB,
                      "positions": n_pos, "postings": n_post, "phrases_per_step": len(qk), "phrase_terms": "2-3, ranks log-uniform [1, 300]",
                      "steps": a.steps, "warmup": a.warmup, "index_build_s": round(build_s, 2)}}
    for name, rt in (("topk", ResultType.Topk), ("topkcount", ResultType.TopkCount)):
        def step():
            ix.search_lexical_keys(b, TOPK, rt, out_keys, cnt)
        for _ in range(a.warmup):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        step(); torch.cuda.synchronize()
        sv = ix.last_stats()
        res[name] = {"queries_per_s": round(len(qk) * a.steps / (ms / 1e3), 1), "ms_per_step": round(ms / a.steps, 3),
                     "lex_generic_ms": round(sv["dominant_kernel_ns"] / 1e6, 3), "postings_visited": sv.get("postings_visited")}
    res["matching_phrases"] = int((cnt > 0).sum().item())
    ix.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
