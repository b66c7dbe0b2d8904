"""NumPy statement of the sorted scan, facet counts, aggregates and match scan of exact phrase queries
(sdbg_phrase_topk_by_column_batch / sdbg_phrase_facet_counts_batch / sdbg_phrase_aggregate_batch /
sdbg_phrase_scan_batch): the docs phrase_reference.match gives per segment (deletions, filter mask and exclusions
already applied), sorted, counted or aggregated per key exactly as sort_reference / facet_reference / agg_reference do
for the flat queries. Each segment's matching docs are handed to those references as the one list of a one-term OR, so
their order, NULL and key rules are reused as they are. The match scan's order is (segment, doc); a scored hit's score
is phrase_reference.score of its phrase frequency.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import agg_reference as ar
import facet_reference as fr
import phrase_reference as pr
import sort_reference as sr


def matches(seg_docs, phrase, rel=None, excl=(), deleted=None, masks=None):
    """Per segment (doc ids, phrase freqs) of the phrase's matches (phrase_reference.match)."""
    n = len(seg_docs)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return [pr.match(d, phrase, rel, excl, x, m) for d, x, m in zip(seg_docs, deleted, masks)]


def _as_one_term(seg_matches):
    """Per segment [the phrase's matching docs]: a one-term list set whose OR of term 0 is exactly the phrase query."""
    return [[ds] for ds, _ in seg_matches]


def sorted_hits(seg_matches, columns, descending=False, nulls_first=False, k=None):
    """sort_reference.sorted_hits of the phrase whose matches are seg_matches (from matches())."""
    return sr.sorted_hits(_as_one_term(seg_matches), "OR", [0], columns, descending, nulls_first, k)


def facet_counts(seg_matches, columns, key_min, key_span):
    """facet_reference.facet_counts of the phrase: (counts uint64[key_span], nulls)."""
    return fr.facet_counts(_as_one_term(seg_matches), "OR", [0], columns, key_min, key_span)


def aggregate(seg_matches, key_columns, val_columns, key_min=0, key_span=1):
    """agg_reference.aggregate of the phrase: (cells [key_span], NULL-key cell)."""
    return ar.aggregate(_as_one_term(seg_matches), "OR", [0], key_columns, val_columns, key_min, key_span)


def scan(seg_matches, seg_norms=None, c=None, offset=0, limit=None):
    """The match scan's page of the phrase: (segs uint32, docs uint32, scores float32) of the matches at ordinals
    [offset, offset + limit) in (segment, doc) order, and the total. c: the (c0, norm_const, norm_length) of
    phrase_reference.consts to score each hit as phrase_reference.score of its phrase frequency (None: scores 0).
    seg_norms: per segment the norms by row (doc - 1), or None for norm 1."""
    seg_norms = seg_norms or [None] * len(seg_matches)
    segs = np.concatenate([np.full(len(ds), si, np.uint32) for si, (ds, _) in enumerate(seg_matches)])
    docs = np.concatenate([ds for ds, _ in seg_matches]).astype(np.uint32)
    freqs = np.concatenate([fs for _, fs in seg_matches]).astype(np.uint32)
    total = len(docs)
    end = total if limit is None else min(total, offset + limit)
    sel = slice(min(offset, total), end)
    segs, docs, freqs = segs[sel], docs[sel], freqs[sel]
    scores = np.zeros(len(docs), np.float32)
    if c is not None:
        for i, (s, d, f) in enumerate(zip(segs, docs, freqs)):
            norms = seg_norms[s]
            scores[i] = pr.score(f, 1 if norms is None else norms[d - 1], *c)
    return (segs, docs, scores), total
