"""The empty query restated for the tests, never through the library's keys.

shard_route restates search_iterator_shard (iterator.rs:316-358) literally: the docs in id order, the delete set and is_facet_filter
(add_result.rs:95-338), the count of Count / TopkCount (Topk counts nothing), and add_topk with the empty query's comparator: the sort
criteria compared in their own types (helpers_sort.FacetRows), `_id` / `_score` ending the comparison (min_heap.rs:580-604), then the larger
doc id first (min_heap.rs:535-536, 1043-1044).  A leading `_score` orders by the doc id in its own direction, the index route's order
(iterator.rs:360-413) the library documents for it.  numpy_route is the same result by one np.lexsort over typed ranks."""
import functools
import heapq

import numpy as np

from seekstorm_b200 import _lib
from helpers_sort import _cmp, _cmp_value


def live_docs(levels, deleted=()):
    """the doc universe: level << 16 | 0 .. n_docs - 1 of every (level_id, n_docs), outside the delete set, ascending"""
    d = set(int(x) for x in deleted)
    return [(lv << 16) | i for lv, n in sorted(levels) for i in range(n) if ((lv << 16) | i) not in d]


def effective_criteria(criteria):
    """[(name, descending)] as the library orders them: a leading `_score` is `_id` in its direction"""
    if criteria and criteria[0][0] == "_score":
        return [("_id", criteria[0][1])]
    return list(criteria)


def compare(a, b, criteria, value):
    """> 0: doc a ranks before doc b.  value(name, doc): the typed value of a facet criterion (a Point criterion: the distance)"""
    for name, desc in effective_criteria(criteria):
        if name == "_id":
            o = _cmp(a, b)
            return o if desc else -o
        if name == "_score":                                     # every score is 0.0: equal, and the comparison ends
            break
        o = _cmp_value(value(name, a), value(name, b))
        if o:
            return o if desc else -o
    return _cmp(a, b)                                            # ties: the larger doc id first


def shard_route(docs, passes, k, result_type, criteria, value):
    """search_iterator_shard over `docs` (ascending): passes(doc) = not deleted and every filter accepts it.  -> (hit doc ids, count)"""
    key = functools.cmp_to_key(lambda a, b: compare(a, b, criteria, value))
    heap, count = [], 0
    for doc in docs:
        if not passes(doc):
            continue
        if result_type != _lib.RESULT_TOPK:
            count += 1
        if result_type == _lib.RESULT_COUNT or k == 0:
            continue
        if len(heap) < k:
            heapq.heappush(heap, key(doc))                       # add_topk: a min-heap of the k best
        elif compare(doc, heap[0].obj, criteria, value) > 0:
            heapq.heapreplace(heap, key(doc))
    return [h.obj for h in sorted(heap, reverse=True)], count


def numpy_route(docs, mask, k, criteria, ranks):
    """the same order by one np.lexsort: docs [n] int64, mask [n] bool (passes), ranks(name, docs) -> an int64 rank per doc in the
    criterion's order (ascending = smaller first).  -> the first k doc ids"""
    d = np.asarray(docs, dtype=np.int64)[np.asarray(mask, dtype=bool)]
    keys = []
    for name, desc in effective_criteria(criteria):
        if name == "_id":
            keys.append(-d if desc else d)
            break
        if name == "_score":
            break
        r = ranks(name, d)
        keys.append(-r if desc else r)
    order = np.lexsort([-d] + keys[::-1])
    return [int(x) for x in d[order[:k]]]


def value_fn(facets, points=None):
    """value(name, doc) over helpers_sort.FacetRows; points: name -> (per-doc distance array indexed by doc - first) for Point criteria"""
    points = points or {}

    def value(name, doc):
        if name in points:
            return float(points[name][doc - facets.first])
        return facets.value(name, doc)
    return value


def top_values(col, length, eligible=None):
    """get_index_string_facets_shard on one String facet column: the `length` ids with the most rows, count desc then id asc; eligible(id)
    restricts the ids before the cut (a prefix) -> [(id, count)]"""
    ids, cnt = np.unique(np.asarray(col, dtype=np.int64), return_counts=True)
    pairs = [(int(i), int(c)) for i, c in zip(ids, cnt) if eligible is None or eligible(int(i))]
    return sorted(pairs, key=lambda p: (-p[1], p[0]))[:length]
