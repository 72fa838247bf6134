"""Multi-value string facets (StringSet16 / StringSet32) restated two ways.

The literal restatement follows the reference line by line: ingest into an insertion-ordered map of joined keys (index.rs:5763-5801),
string_set_to_single_term_id (index.rs:4282-4297), the resolution of FacetFilter::StringSet16 / 32 into combination ids
(search.rs:2643-2710) tested with `values.contains(id)` (is_facet_filter, add_result.rs:340-478), the per-combination bins of a shard
(add_result.rs:620-633) split over the stored members (search.rs:3615-3640), the index-wide split over the ingest counters
(index.rs:4531-4550), and the sort comparator on the first stored member (min_heap.rs:393-420, 900-925).

The numpy formulation works on what the library holds instead: the combination id column and the CSR of member ids, a filter as member
ids plus flagged combination ids, counts as one bincount over member occurrences."""
import numpy as np

COMBINATION = 1 << 63


# ---------------------------------------------------------------- the reference, restated
def ingest(docs, limit=65535):
    """facet.values after indexing `docs` (lists of strings): an insertion-ordered dict joined key -> (stored sorted list, doc count),
    and the id each doc's row holds.  `if facet.values.len() < u16::MAX` guards every write: past it the row keeps 0 (None here)."""
    values, ids = {}, []
    for lst in docs:
        if len(values) >= limit:
            ids.append(None)
            continue
        key = sorted(lst, key=lambda s: s.encode("utf-8"))          # Vec<String>::sort: byte-wise
        key_string = "_".join(key)
        if key_string not in values:
            values[key_string] = (key, 0)
        k, c = values[key_string]
        values[key_string] = (k, c + 1)
        ids.append(list(values).index(key_string))                  # get_index_of
    return values, ids


def single_term_ids(values):
    """string_set_to_single_term_id: member string -> the ids of the combinations whose stored list holds it"""
    out = {}
    for idx, (key_string, (members, _)) in enumerate(values.items()):
        for term in members:
            out.setdefault(term, set()).add(idx)
    return out


def resolve_filter(values, single, strings):
    """FacetFilter::StringSet16 / 32 -> FilterSparse::String16 / 32: per string its joined key's id, then every id holding it"""
    keys = list(values)
    out = []
    for v in strings:
        if v in values:                                             # facet.values.get_index_of(&[v].join("_"))
            out.append(keys.index(v))
        out.extend(sorted(single.get(v, ())))
    return out


def passes(ids, combination_ids):
    """is_facet_filter on FilterSparse::String16 / 32: the doc's id among the resolved ids"""
    s = set(combination_ids)
    return np.array([i in s for i in ids], dtype=bool)


def member_counts(values, bins):
    """search.rs:3615-3640: the counts of combination ids (bins: id -> count) added to each stored member, once per occurrence"""
    keys = list(values)
    out = {}
    for cid, c in bins.items():
        for term in values[keys[cid]][0]:
            out[term] = out.get(term, 0) + c
    return out


def index_member_counts(values):
    """index.rs:4531-4550: the ingest counters (docs per combination) split over the stored members"""
    out = {}
    for members, c in values.values():
        for term in members:
            out[term] = out.get(term, 0) + c
    return out


def top(counts, prefix="", length=10):
    """count descending, members whose string starts with prefix, at most length.  The reference breaks ties in hash-map order; the
    library takes the smaller member id, the smaller string, which this applies"""
    items = [(s, c) for s, c in counts.items() if c and s.startswith(prefix)]
    items.sort(key=lambda x: (-x[1], x[0].encode("utf-8")))
    return items[:length]


def first_member_cmp(values, id1, id2, descending):
    """min_heap.rs:393-420: the first stored members compared (descending: the larger string first); > 0: id1 ranks first.  The
    reference panics on an empty combination; the library sorts it below every string"""
    keys = list(values)
    a, b = values[keys[id1]][0], values[keys[id2]][0]
    ka = a[0].encode("utf-8") if a else None
    kb = b[0].encode("utf-8") if b else None
    if ka == kb:
        return 0
    less = ka is None or (kb is not None and ka < kb)
    return (-1 if less else 1) if descending else (1 if less else -1)


# ---------------------------------------------------------------- numpy over the library's layout
def csr(values):
    """(member strings in byte-wise order, offsets [n_sets + 1], member ids): ssb_set_facet_string_sets' arguments"""
    members = sorted({m.encode("utf-8") for lst, _ in values.values() for m in lst})
    pos = {m: i for i, m in enumerate(members)}
    offs, flat = [0], []
    for lst, _ in values.values():
        flat.extend(pos[m.encode("utf-8")] for m in lst)
        offs.append(len(flat))
    return [m.decode("utf-8") for m in members], np.array(offs, dtype=np.uint64), np.array(flat, dtype=np.uint32)


def combination_mask(offsets, member_ids, filter_values):
    """which combinations a member / flagged filter accepts: a flagged id, or a member in the list"""
    n_sets = len(offsets) - 1
    vals = np.asarray([int(v) for v in filter_values], dtype=np.uint64)
    flagged = (vals[(vals & np.uint64(COMBINATION)) != 0] & ~np.uint64(COMBINATION)).astype(np.int64)
    listed = vals[(vals & np.uint64(COMBINATION)) == 0].astype(np.int64)
    hit = np.isin(member_ids.astype(np.int64), listed)
    owner = np.repeat(np.arange(n_sets), np.diff(offsets.astype(np.int64)))
    ok = np.zeros(n_sets, dtype=bool)
    ok[owner[hit]] = True
    ok[flagged] = True
    return ok


def numpy_member_counts(offsets, member_ids, n_values, col, docs):
    """member id -> count over the rows `docs` of the combination column col"""
    per_set = np.bincount(col[docs].astype(np.int64), minlength=len(offsets) - 1)
    owner = np.repeat(np.arange(len(offsets) - 1), np.diff(offsets.astype(np.int64)))
    return np.bincount(member_ids.astype(np.int64), weights=per_set[owner], minlength=n_values).astype(np.int64)


def numpy_top(counts, lo=0, hi=None, length=10):
    """(member id, count) with count > 0 and id in [lo, hi): count descending, id ascending, at most length"""
    hi = len(counts) if hi is None else hi
    ids = np.nonzero(counts)[0]
    ids = ids[(ids >= lo) & (ids < hi)]
    order = np.lexsort((ids, -counts[ids]))
    return [(int(i), int(counts[i])) for i in ids[order][:length]]
