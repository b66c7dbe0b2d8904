"""NumPy statement of conjunctions of OR groups of phrases and terms (sdbg_phrase_groups_*_batch) over token-sequence
corpora (phrase_reference.py). A query is an AND of groups; a group is (alternatives, negated), an alternative a phrase
(terms, rel_pos or None), a one-slot alternative a plain term. Doc d matches when every positive group has an
alternative with phrase frequency > 0 in d, no alternative of a negated group has, d is not deleted, passes the mask and
holds no excluded term. Its score is the float32 sum, from 0, of bm25(phrase frequency, norm) over the positive
alternatives with frequency > 0, each with its own (c0, norm_const, norm_length), in ascending cost order within d's
segment: an alternative costs the smallest docs_count of its terms in that segment (the docs holding the term, deleted
ones included), ties in the query's alternative order, flattened group by group. Restated from the semantics (no
reference golden exists for phrases; IResearch's Or of by_phrase / by_term children sums the children that match). The
column passes hand each segment's matches to phrase_column_reference as they are.

TEST INFRASTRUCTURE: imported by tests only."""
import numpy as np

import phrase_column_reference as pcr
import phrase_reference as pr


def docs_count(docs, term):
    """The docs of one segment (token sequences) that hold `term`."""
    return sum(1 for seq in docs if term in seq)


def flat(groups):
    """The query's alternatives flattened group by group, as (terms, rel_pos or None, negated)."""
    return [(list(terms), rel, neg) for alts, neg in groups for terms, rel in alts]


def cost_order(docs, groups):
    """The flattened alternatives' indexes in one segment's cost order: ascending smallest docs_count of their terms,
    stable."""
    alts = flat(groups)
    cost = [min(docs_count(docs, t) for t in terms) for terms, _, _ in alts]
    return sorted(range(len(alts)), key=lambda j: cost[j])


def match(docs, groups, excl=(), deleted=None, mask=None):
    """(doc ids, per doc the phrase frequencies of every alternative, flattened) of one segment's matches, by doc."""
    dels = set() if deleted is None else {int(d) for d in deleted}
    ex = {int(t) for t in excl}
    ds, fs = [], []
    for i, seq in enumerate(docs):
        d = i + 1
        if d in dels or (mask is not None and not mask[i]) or ex.intersection(seq):
            continue
        f, ok = [], True
        for alts, neg in groups:
            g = [pr.phrase_freq(seq, terms, rel) for terms, rel in alts]
            f += g
            ok = ok and (not any(g) if neg else any(g))
        if ok:
            ds.append(d)
            fs.append(f)
    return np.array(ds, np.uint32), fs


def matches(seg_docs, groups, excl=(), deleted=None, masks=None):
    n = len(seg_docs)
    deleted = deleted or [None] * n
    masks = masks or [None] * n
    return [match(d, groups, excl, x, m) for d, x, m in zip(seg_docs, deleted, masks)]


def scores(docs, groups, ds, fs, norms, consts):
    """float32 scores of one segment's matches: consts[j] is flattened alternative j's (c0, norm_const, norm_length),
    None when its group is negated; norms by row (doc - 1), or None for norm 1."""
    alts = flat(groups)
    order = [j for j in cost_order(docs, groups) if not alts[j][2]]
    out = np.zeros(len(ds), np.float32)
    for i, (d, f) in enumerate(zip(ds, fs)):
        s = np.float32(0)
        for j in order:
            if f[j] > 0:
                s = np.float32(s + pr.score(f[j], 1 if norms is None else norms[d - 1], *consts[j]))
        out[i] = s
    return out


def topk(seg_docs, groups, seg_matches, seg_norms, consts, k, threshold=np.float32(1.1754944e-38)):
    """The k best (score desc, segment asc, doc asc) of the matches scoring > threshold, as a structured array, and the
    match count."""
    rows, total = [], 0
    for si, (docs, (ds, fs), norms) in enumerate(zip(seg_docs, seg_matches, seg_norms)):
        total += len(ds)
        for d, s in zip(ds, scores(docs, groups, ds, fs, norms, consts)):
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


def scan(seg_docs, groups, seg_matches, seg_norms=None, consts=None, offset=0, limit=None):
    """The match scan's page: (segs uint32, docs uint32, scores float32) at ordinals [offset, offset + limit) in (segment,
    doc) order, and the total; consts None: scores 0."""
    seg_norms = seg_norms or [None] * len(seg_matches)
    segs = np.concatenate([np.full(len(ds), si, np.uint32) for si, (ds, _) in enumerate(seg_matches)])
    docs = np.concatenate([ds for ds, _ in seg_matches]).astype(np.uint32)
    if consts is None:
        sc = np.zeros(len(docs), np.float32)
    else:
        sc = np.concatenate([scores(d, groups, ds, fs, nm, consts)
                             for d, (ds, fs), nm in zip(seg_docs, seg_matches, seg_norms)]).astype(np.float32)
    total = len(docs)
    end = total if limit is None else min(total, offset + limit)
    sel = slice(min(offset, total), end)
    return (segs[sel], docs[sel], sc[sel]), total
