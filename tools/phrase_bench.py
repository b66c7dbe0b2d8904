"""Cost of the phrase check: exact phrase queries against the AND of the same terms, on a seeded token corpus.

The corpus: --docs docs (10 M by default) of 4..28 tokens each (uniform), tokens drawn from a Zipf(1.1) vocabulary of
--vocab terms, norms = doc lengths, one segment. Two batches of --queries phrases, windows of the corpus's own token
sequence (a window is picked with its frequency, so frequent adjacent pairs dominate): two-word phrases, and three- and
four-word phrases. For each batch it reports ms per step (CUDA events on the library's stream, L2 flushed before every step, after
warm-up) of
  phrase count (sdbg_phrase_count_batch)   against   AND count of the same terms (sdbg_match_count_batch)
  phrase top-1000 (sdbg_phrase_topk_batch) against   AND top-1000 (sdbg_bm25_topk_batch at pruning level 0)
and the matches of both. The AND is the phrase's candidate set, so the gap is the cost of checking positions. Then the
four passes of the phrases' matches, next to the phrase count, over two staged columns (an int64 column `ts` of uniform
values and an int32 column `cat` of 100 values):
  sorted LIMIT 1000 by ts (sdbg_phrase_topk_by_column_batch, pruning level 2 as shipped)
  facets GROUP BY cat (sdbg_phrase_facet_counts_batch)
  SUM / AVG(ts) GROUP BY cat (sdbg_phrase_aggregate_batch)
  the first scan page of 1000, unscored and scored (sdbg_phrase_scan_batch), and an unscored page of 1000 from the
  middle of each phrase's matches (a page deep in the result repeats the phrase check over the items before it).
A third batch, "phrase-and", times conjunctions of a phrase with a term (sdbg_phrase_and_*_batch): --queries
queries `"w1 w2" & t`, t a token drawn from the phrase's own doc, and the same with `& !"w3 w4"` added, w3 w4 a window
drawn as the phrases are. For each it reports the count, the top-1000 and the facets GROUP BY cat, next to the phrase
"w1 w2" alone and the AND of w1, w2 and t (and of w3, w4 not excluded: the AND of w1, w2, t is the candidate set).
A fourth batch, "phrase-groups", times phrases inside OR groups (sdbg_phrase_groups_*_batch), the shape synonym
expansion produces: --queries queries each of `("w1 w2" | s) & t`, `"w1 w2" | s` and `("w1 w2" | s) & t & !"w3 w4"`,
s a token of another doc, t a token of the phrase's doc (s, w1 and t distinct), next to `"w1 w2" & t` (phrase-and) and
`(w1 | s) & t` (the OR-group count, top-k and facets of sdbg_*_groups). The proxy candidates of `"w1 w2" | s` are the
docs of w1 or w2 (the cheaper) or s, wider than the phrase's own AND.
A fifth batch, "phrase-min", times minimum match counts over such groups (sdbg_phrase_groups_*_batch_min):
`2 of ("w1 w2" | s | t)`, `2 of ("w1 w2" | s | t) & u` and `2 of ("w1 w2" | s | "w3 w4")`, count, top-1000 and facets.
--batches picks the batches to run (comma-separated; all by default).
Prints one JSON line with the GPU name and power limit read in the same run.

    python tools/phrase_bench.py [--steps 5] [--warmup 2] [--docs 10000000] [--queries 4096] [--batches 2-word,phrase-and,phrase-groups,phrase-min]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import serenedb_b200 as sdb  # noqa: E402
from count_bench import gpu_info, timed  # noqa: E402


def corpus(n_docs, vocab, seed):
    # the sort key below packs (term, doc, position) into 64 bits: 29 bits of term, 30 of doc, 5 of position (< 32)
    if not 0 < n_docs < 1 << 30 or not 0 < vocab <= 1 << 29:
        raise SystemExit("--docs must be below 2^30 and --vocab at most 2^29")
    rng = np.random.default_rng(seed)
    lens = rng.integers(4, 29, n_docs).astype(np.int64)   # positions 0..27: 5 bits
    n_tok = int(lens.sum())
    terms = ((rng.zipf(1.1, n_tok) - 1) % vocab).astype(np.uint64)   # the tail past the vocabulary folds back onto it
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    doc = np.repeat(np.arange(1, n_docs + 1, dtype=np.uint64), lens)
    pos = np.arange(n_tok, dtype=np.uint64) - np.repeat(starts.astype(np.uint64), lens)
    # one sort by (term, doc, position) gives the postings and, per posting, its positions in order
    key = np.sort((terms << np.uint64(35)) | (doc << np.uint64(5)) | pos)
    t_of, d_of, p_of = key >> np.uint64(35), (key >> np.uint64(5)) & np.uint64((1 << 30) - 1), (key & np.uint64(31)).astype(np.uint32)
    td = key >> np.uint64(5)
    first = np.flatnonzero(np.concatenate([[True], td[1:] != td[:-1]]))
    freqs = np.diff(np.concatenate([first, [len(key)]])).astype(np.uint32)
    post_t, post_d = t_of[first].astype(np.int64), d_of[first].astype(np.uint32)
    w = sdb.PostingsWriter(n_docs, norms=lens.astype(np.uint32))
    tb = np.searchsorted(post_t, np.arange(vocab + 1))
    pb = np.searchsorted(t_of.astype(np.int64), np.arange(vocab + 1))
    for t in range(vocab):
        w.add_term(post_d[tb[t]:tb[t + 1]], freqs[tb[t]:tb[t + 1]])
    doc_bytes, metas = w.finish()
    return dict(n=n_docs, lens=lens, terms=terms, doc=doc, doc_bytes=doc_bytes, metas=metas, positions=p_of,
                term_pos_off=pb.astype(np.uint64), dwt=(tb[1:] - tb[:-1]))


def phrases(c, n, length, rng):
    """n phrases of `length` tokens, each a window of the corpus starting at a uniformly drawn token whose window stays in
    its doc: frequent word sequences are drawn in proportion to their frequency."""
    terms, doc = c["terms"], c["doc"]
    out = []
    while len(out) < n:
        i = rng.integers(0, len(terms) - length, n)
        ok = doc[i] == doc[i + length - 1]
        for j in i[ok][: n - len(out)]:
            out.append([int(x) for x in terms[j:j + length]])
    return out


def phrase_and_rows(c, reader, ctx, scorer, n, rng, steps, warmup):
    """The "phrase-and" batch: `"w1 w2" & t` and `"w1 w2" & t & !"w3 w4"` next to "w1 w2" and the AND of w1, w2, t."""
    terms, doc = c["terms"], c["doc"]
    ph, ts = [], []
    while len(ph) < n:
        i = int(rng.integers(0, len(terms) - 2))
        if doc[i] != doc[i + 1]:
            continue
        same = np.flatnonzero(doc[max(0, i - 28):i + 30] == doc[i]) + max(0, i - 28)
        ph.append([int(terms[i]), int(terms[i + 1])])
        ts.append(int(terms[int(same[int(rng.integers(0, len(same)))])]))
    neg = phrases(c, n, 2, rng)
    plain = [[p, [t]] for p, t in zip(ph, ts)]
    conj = [sorted(set(p + [t])) for p, t in zip(ph, ts)]
    pc = sdb.ExecutePhraseCountBatch(reader, ph)
    ac = sdb.ExecuteCountBatch(reader, conj, sdb.AND)
    qc = sdb.ExecutePhraseAndCountBatch(reader, plain)
    nc = sdb.ExecutePhraseAndCountBatch(reader, plain, exclude_phrases=[[x] for x in neg])
    _, _, qt = sdb.ExecutePhraseAndTopKBatch(reader, plain, scorer, 1000)
    fac = sdb.ExecutePhraseAndFacetCountsBatch(reader, plain, 2, 0, 100)
    if (not np.array_equal(qc, qt) or not np.array_equal(fac["counts"].sum(1), qc) or np.any(qc > pc) or np.any(qc > ac)
            or np.any(nc > qc)):
        raise SystemExit("phrase-and count / top-k / facet mismatch")
    r = {"phrase_matches": int(pc.sum()), "and_matches": int(ac.sum()), "phrase_and_matches": int(qc.sum()),
         "phrase_and_not_matches": int(nc.sum())}
    runs = (("phrase", lambda: sdb.ExecutePhraseCountBatch(reader, ph), lambda: sdb.ExecutePhraseTopKBatch(reader, ph, scorer, 1000),
             lambda: sdb.ExecutePhraseFacetCountsBatch(reader, ph, 2, 0, 100)),
            ("and", lambda: sdb.ExecuteCountBatch(reader, conj, sdb.AND), lambda: sdb.ExecuteTopKBatch(reader, conj, sdb.AND, scorer, 1000),
             lambda: sdb.ExecuteFacetCountsBatch(reader, conj, sdb.AND, 2, 0, 100)),
            ("phrase_and", lambda: sdb.ExecutePhraseAndCountBatch(reader, plain),
             lambda: sdb.ExecutePhraseAndTopKBatch(reader, plain, scorer, 1000),
             lambda: sdb.ExecutePhraseAndFacetCountsBatch(reader, plain, 2, 0, 100)),
            ("phrase_and_not", lambda: sdb.ExecutePhraseAndCountBatch(reader, plain, exclude_phrases=[[x] for x in neg]),
             lambda: sdb.ExecutePhraseAndTopKBatch(reader, plain, scorer, 1000, exclude_phrases=[[x] for x in neg]),
             lambda: sdb.ExecutePhraseAndFacetCountsBatch(reader, plain, 2, 0, 100, exclude_phrases=[[x] for x in neg])))
    for name, cnt, top, facets in runs:
        r[name + "_count_ms"] = timed(ctx, cnt, steps, warmup)
        r[name + "_top1000_ms"] = timed(ctx, top, steps, warmup)
        r[name + "_facets_ms"] = timed(ctx, facets, steps, warmup)
    return r


def phrase_groups_rows(c, reader, ctx, scorer, n, rng, steps, warmup):
    """The "phrase-groups" batch: `("w1 w2" | s) & t`, `"w1 w2" | s`, `("w1 w2" | s) & t & !"w3 w4"` next to `"w1 w2" & t`
    and `(w1 | s) & t`."""
    terms, doc = c["terms"], c["doc"]
    ph, ss, ts = [], [], []
    while len(ph) < n:
        i = int(rng.integers(0, len(terms) - 2))
        if doc[i] != doc[i + 1]:
            continue
        same = np.flatnonzero(doc[max(0, i - 28):i + 30] == doc[i]) + max(0, i - 28)
        t = int(terms[int(same[int(rng.integers(0, len(same)))])])
        s = int(terms[int(rng.integers(0, len(terms)))])
        if len({int(terms[i]), s, t}) < 3:
            continue
        ph.append([int(terms[i]), int(terms[i + 1])]); ss.append(s); ts.append(t)
    neg = [[x] for x in phrases(c, n, 2, rng)]
    and_t = [[[p], [[t]]] for p, t in zip(ph, ts)]
    or_t = [[[p, [s]], [[t]]] for p, s, t in zip(ph, ss, ts)]
    or_only = [[[p, [s]]] for p, s in zip(ph, ss)]
    grp = [[[p[0], s], [t]] for p, s, t in zip(ph, ss, ts)]
    pa = [[p, [t]] for p, t in zip(ph, ts)]
    counts = {"phrase_and": sdb.ExecutePhraseGroupsCountBatch(reader, and_t), "or_and_t": sdb.ExecutePhraseGroupsCountBatch(reader, or_t),
              "or": sdb.ExecutePhraseGroupsCountBatch(reader, or_only),
              "or_and_t_not": sdb.ExecutePhraseGroupsCountBatch(reader, or_t, exclude_phrases=neg),
              "groups": sdb.ExecuteCountGroupsBatch(reader, grp)}
    _, _, tt = sdb.ExecutePhraseGroupsTopKBatch(reader, or_t, scorer, 1000)
    fac = sdb.ExecutePhraseGroupsFacetCountsBatch(reader, or_t, 2, 0, 100)
    if (not np.array_equal(counts["phrase_and"], sdb.ExecutePhraseAndCountBatch(reader, pa)) or not np.array_equal(tt, counts["or_and_t"])
            or not np.array_equal(fac["counts"].sum(1), counts["or_and_t"]) or np.any(counts["or_and_t"] < counts["phrase_and"])
            or np.any(counts["or_and_t_not"] > counts["or_and_t"])):
        raise SystemExit("phrase-groups count / top-k / facet mismatch")
    r = {k + "_matches": int(v.sum()) for k, v in counts.items()}
    runs = (("phrase_and", lambda: sdb.ExecutePhraseAndCountBatch(reader, pa), lambda: sdb.ExecutePhraseAndTopKBatch(reader, pa, scorer, 1000),
             lambda: sdb.ExecutePhraseAndFacetCountsBatch(reader, pa, 2, 0, 100)),
            ("groups", lambda: sdb.ExecuteCountGroupsBatch(reader, grp), lambda: sdb.ExecuteTopKGroupsBatch(reader, grp, scorer, 1000),
             lambda: sdb.ExecuteFacetCountsGroupsBatch(reader, grp, 2, 0, 100)))
    runs += tuple((name, (lambda q=q, x=x: sdb.ExecutePhraseGroupsCountBatch(reader, q, exclude_phrases=x)),
                   (lambda q=q, x=x: sdb.ExecutePhraseGroupsTopKBatch(reader, q, scorer, 1000, exclude_phrases=x)),
                   (lambda q=q, x=x: sdb.ExecutePhraseGroupsFacetCountsBatch(reader, q, 2, 0, 100, exclude_phrases=x)))
                  for name, q, x in (("or_and_t", or_t, None), ("or", or_only, None), ("or_and_t_not", or_t, neg)))
    for name, cnt, top, facets in runs:
        r[name + "_count_ms"] = timed(ctx, cnt, steps, warmup)
        r[name + "_top1000_ms"] = timed(ctx, top, steps, warmup)
        r[name + "_facets_ms"] = timed(ctx, facets, steps, warmup)
    return r


def phrase_min_rows(c, reader, ctx, scorer, n, rng, steps, warmup):
    """The "phrase-min" batch: `2 of ("w1 w2" | s | t)`, `2 of ("w1 w2" | s | t) & u` and `2 of ("w1 w2" | s | "w3 w4")`
    (sdbg_phrase_groups_*_batch_min): s, t and u occur near the phrase in its doc, so the minimums are met often."""
    terms, doc = c["terms"], c["doc"]
    ph, near = [], []
    while len(ph) < n:
        i = int(rng.integers(0, len(terms) - 2))
        if doc[i] != doc[i + 1]:
            continue
        same = np.flatnonzero(doc[max(0, i - 28):i + 30] == doc[i]) + max(0, i - 28)
        s, t, u = (int(terms[int(same[int(rng.integers(0, len(same)))])]) for _ in range(3))
        if len({int(terms[i]), int(terms[i + 1]), s, t, u}) < 5:
            continue
        ph.append([int(terms[i]), int(terms[i + 1])]); near.append((s, t, u))
    w34 = phrases(c, n, 2, rng)
    two = [[[p, [s], [t]]] for p, (s, t, _) in zip(ph, near)]
    two_u = [[[p, [s], [t]], [[u]]] for p, (s, t, u) in zip(ph, near)]
    two_ph = [[[p, [s], q]] for p, (s, _, _), q in zip(ph, near, w34)]
    r = {}
    for name, q, m in (("two", two, [[2]] * n), ("two_and_u", two_u, [[2, 1]] * n), ("two_phrases", two_ph, [[2]] * n)):
        cnt = sdb.ExecutePhraseGroupsCountBatch(reader, q, min_match=m)
        one = sdb.ExecutePhraseGroupsCountBatch(reader, q)
        _, _, tt = sdb.ExecutePhraseGroupsTopKBatch(reader, q, scorer, 1000, min_match=m)
        fac = sdb.ExecutePhraseGroupsFacetCountsBatch(reader, q, 2, 0, 100, min_match=m)
        if not np.array_equal(tt, cnt) or not np.array_equal(fac["counts"].sum(1), cnt) or np.any(cnt > one):
            raise SystemExit("phrase-min count / top-k / facet mismatch")
        r[name + "_matches"] = int(cnt.sum())
        r[name + "_count_ms"] = timed(ctx, lambda: sdb.ExecutePhraseGroupsCountBatch(reader, q, min_match=m), steps, warmup)
        r[name + "_top1000_ms"] = timed(ctx, lambda: sdb.ExecutePhraseGroupsTopKBatch(reader, q, scorer, 1000, min_match=m), steps,
                                        warmup)
        r[name + "_facets_ms"] = timed(ctx, lambda: sdb.ExecutePhraseGroupsFacetCountsBatch(reader, q, 2, 0, 100, min_match=m), steps,
                                       warmup)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--batches", default="2-word,3/4-word,phrase-and,phrase-groups,phrase-min")
    a = ap.parse_args()
    want = set(a.batches.split(","))
    c = corpus(a.docs, a.vocab, 7)
    ctx = sdb.Context(0)
    seg = sdb.Segment(ctx, c["n"])
    seg.stage_postings(c["doc_bytes"], c["metas"])
    seg.stage_norms(c["lens"].astype(np.uint8), 1)
    seg.stage_positions(c["positions"], c["term_pos_off"])
    crng = np.random.default_rng(13)
    seg.stage_column(1, crng.integers(0, 1 << 40, c["n"]).astype(np.int64))   # ts
    seg.stage_column(2, crng.integers(0, 100, c["n"]).astype(np.int32))       # cat
    reader = sdb.IndexReader([seg], c["n"], int(c["lens"].sum()), c["dwt"])
    scorer = sdb.BM25()
    rng = np.random.default_rng(11)
    out = {"gpu": gpu_info(), "docs": c["n"], "tokens": int(c["lens"].sum()), "queries": a.queries, "batches": {}}
    ctx.set_wand(0)
    for name, qs in (("2-word", phrases(c, a.queries, 2, rng)),
                     ("3/4-word", phrases(c, a.queries // 2, 3, rng) + phrases(c, a.queries - a.queries // 2, 4, rng))):
        if name not in want:
            continue
        conj = [sorted(set(q)) for q in qs]
        pc = sdb.ExecutePhraseCountBatch(reader, qs)
        ac = sdb.ExecuteCountBatch(reader, conj, sdb.AND)
        _, _, pt = sdb.ExecutePhraseTopKBatch(reader, qs, scorer, 1000)
        if not np.array_equal(pc, pt) or np.any(pc > ac):
            raise SystemExit("phrase count / top-k total mismatch")
        r = {"phrase_matches": int(pc.sum()), "and_matches": int(ac.sum())}
        r["phrase_count_ms"] = timed(ctx, lambda: sdb.ExecutePhraseCountBatch(reader, qs), a.steps, a.warmup)
        r["and_count_ms"] = timed(ctx, lambda: sdb.ExecuteCountBatch(reader, conj, sdb.AND), a.steps, a.warmup)
        r["phrase_top1000_ms"] = timed(ctx, lambda: sdb.ExecutePhraseTopKBatch(reader, qs, scorer, 1000), a.steps, a.warmup)
        r["and_top1000_ms"] = timed(ctx, lambda: sdb.ExecuteTopKBatch(reader, conj, sdb.AND, scorer, 1000), a.steps, a.warmup)
        # the four passes over the same phrases; each is checked against the count before it is timed
        ctx.set_wand(2)
        srt = sdb.ExecutePhraseTopKByColumnBatch(reader, qs, 1, 1000)
        fac = sdb.ExecutePhraseFacetCountsBatch(reader, qs, 2, 0, 100)
        agg = sdb.ExecutePhraseMatchAggregatesBatch(reader, qs, 1, 2, 0, 100)
        scan = sdb.ExecutePhraseMatchScanBatch(reader, qs, None, 1000)
        mid = np.ascontiguousarray(pc // 2, dtype=np.uint64)
        if (not np.array_equal(srt["n_out"], np.minimum(pc, 1000)) or not np.array_equal(fac["counts"].sum(1), pc)
                or not np.array_equal(agg["count"].sum(1), pc) or [t for _, t in scan] != pc.tolist()):
            raise SystemExit("phrase pass / count mismatch")
        r["phrase_sorted1000_ms"] = timed(ctx, lambda: sdb.ExecutePhraseTopKByColumnBatch(reader, qs, 1, 1000), a.steps, a.warmup)
        ctx.set_wand(0)
        r["phrase_facets_ms"] = timed(ctx, lambda: sdb.ExecutePhraseFacetCountsBatch(reader, qs, 2, 0, 100), a.steps, a.warmup)
        r["phrase_sum_avg_ms"] = timed(ctx, lambda: sdb.ExecutePhraseMatchAggregatesBatch(reader, qs, 1, 2, 0, 100), a.steps,
                                       a.warmup)
        r["phrase_scan1000_ms"] = timed(ctx, lambda: sdb.ExecutePhraseMatchScanBatch(reader, qs, None, 1000), a.steps, a.warmup)
        r["phrase_scan1000_scored_ms"] = timed(ctx, lambda: sdb.ExecutePhraseMatchScanBatch(reader, qs, scorer, 1000), a.steps,
                                               a.warmup)
        r["phrase_scan1000_mid_ms"] = timed(ctx, lambda: sdb.ExecutePhraseMatchScanBatch(reader, qs, None, 1000, mid), a.steps,
                                            a.warmup)
        out["batches"][name] = r
    if "phrase-and" in want:
        out["batches"]["phrase-and"] = phrase_and_rows(c, reader, ctx, scorer, a.queries, np.random.default_rng(17), a.steps, a.warmup)
    if "phrase-groups" in want:
        out["batches"]["phrase-groups"] = phrase_groups_rows(c, reader, ctx, scorer, a.queries, np.random.default_rng(19), a.steps,
                                                             a.warmup)
    if "phrase-min" in want:
        out["batches"]["phrase-min"] = phrase_min_rows(c, reader, ctx, scorer, a.queries, np.random.default_rng(23), a.steps, a.warmup)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
