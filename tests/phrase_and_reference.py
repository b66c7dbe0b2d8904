"""NumPy statement of conjunctions of phrases, terms and negated phrases (sdbg_phrase_and_*_batch) over token-sequence
corpora (phrase_reference.py). A query is an AND of clauses; a clause is a phrase (terms, rel_pos or None, negated), a
one-slot clause a plain term. Doc d matches when every positive clause has phrase frequency > 0 in d, every negated
clause phrase frequency 0, d is not deleted, passes the mask and holds no excluded term. Its score is the float32 sum,
from 0, of bm25(phrase frequency, norm) over the positive clauses, each with its own (c0, norm_const, norm_length), in
ascending cost order within d's segment: a clause costs the smallest docs_count of its terms in that segment (the docs
holding the term, deleted ones included), ties in the query's clause order. Restated from the semantics (no reference
golden exists for phrases). The column passes hand each segment's matches to phrase_column_reference as they are.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import phrase_column_reference as pcr
import phrase_reference as pr


def docs_count(docs, term):
    """The docs of one segment (token sequences) that hold `term`."""
    return sum(1 for seq in docs if term in seq)


def cost_order(docs, clauses):
    """The clauses' indexes in one segment's cost order: ascending smallest docs_count of their terms, stable."""
    cost = [min(docs_count(docs, t) for t in terms) for terms, _, _ in clauses]
    return sorted(range(len(clauses)), key=lambda j: cost[j])


def match(docs, clauses, excl=(), deleted=None, mask=None):
    """(doc ids, per doc the phrase frequencies of every clause, in query order) of one segment's matches, by doc."""
    dels = set() if deleted is None else {int(d) for d in deleted}
    ex = {int(t) for t in excl}
    ds, fs = [], []
    for i, seq in enumerate(docs):
        d = i + 1
        if d in dels or (mask is not None and not mask[i]) or ex.intersection(seq):
            continue
        f = [pr.phrase_freq(seq, terms, rel) for terms, rel, _ in clauses]
        if all((x > 0) != neg for x, (_, _, neg) in zip(f, clauses)):
            ds.append(d)
            fs.append(f)
    return np.array(ds, np.uint32), fs


def matches(seg_docs, clauses, excl=(), deleted=None, masks=None):
    n = len(seg_docs)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return [match(d, clauses, excl, x, m) for d, x, m in zip(seg_docs, deleted, masks)]


def scores(docs, clauses, ds, fs, norms, consts):
    """float32 scores of one segment's matches: consts[j] is clause j's (c0, norm_const, norm_length), None when negated;
    norms by row (doc - 1), or None for norm 1."""
    order = [j for j in cost_order(docs, clauses) if not clauses[j][2]]
    out = np.zeros(len(ds), np.float32)
    for i, (d, f) in enumerate(zip(ds, fs)):
        s = np.float32(0)
        for j in order:
            s = np.float32(s + pr.score(f[j], 1 if norms is None else norms[d - 1], *consts[j]))
        out[i] = s
    return out


def topk(seg_docs, clauses, seg_matches, seg_norms, consts, k, threshold=np.float32(1.1754944e-38)):
    """The k best (score desc, segment asc, doc asc) of the matches scoring > threshold, as a structured array, and the
    match count."""
    rows, total = [], 0
    for si, (docs, (ds, fs), norms) in enumerate(zip(seg_docs, seg_matches, seg_norms)):
        total += len(ds)
        for d, s in zip(ds, scores(docs, clauses, ds, fs, norms, consts)):
            if s > np.float32(threshold):
                rows.append((np.float32(s), int(d), si))
    rows.sort(key=lambda r: (-r[0], r[2], r[1]))
    out = np.zeros(min(k, len(rows)), [("score", "<f4"), ("doc", "<u4"), ("seg", "<u4")])
    for i, r in enumerate(rows[:k]):
        out[i] = r
    return out, total


def count(seg_matches):
    return sum(len(ds) for ds, _ in seg_matches)


def sorted_hits(seg_matches, columns, descending=False, nulls_first=False, k=None):
    return pcr.sorted_hits(seg_matches, columns, descending, nulls_first, k)


def facet_counts(seg_matches, columns, key_min, key_span):
    return pcr.facet_counts(seg_matches, columns, key_min, key_span)


def aggregate(seg_matches, key_columns, val_columns, key_min=0, key_span=1):
    return pcr.aggregate(seg_matches, key_columns, val_columns, key_min, key_span)


def scan(seg_docs, clauses, seg_matches, seg_norms=None, consts=None, offset=0, limit=None):
    """The match scan's page: (segs uint32, docs uint32, scores float32) at ordinals [offset, offset + limit) in (segment,
    doc) order, and the total; consts None: scores 0."""
    seg_norms = seg_norms or [None] * len(seg_matches)
    segs = np.concatenate([np.full(len(ds), si, np.uint32) for si, (ds, _) in enumerate(seg_matches)])
    docs = np.concatenate([ds for ds, _ in seg_matches]).astype(np.uint32)
    if consts is None:
        sc = np.zeros(len(docs), np.float32)
    else:
        sc = np.concatenate([scores(d, clauses, ds, fs, nm, consts)
                             for d, (ds, fs), nm in zip(seg_docs, seg_matches, seg_norms)]).astype(np.float32)
    total = len(docs)
    end = total if limit is None else min(total, offset + limit)
    sel = slice(min(offset, total), end)
    return (segs[sel], docs[sel], sc[sel]), total
