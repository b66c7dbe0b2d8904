"""Every block encoding of the posting format through the kernels that serve queries, not only through the decoder:
bit-packed docs of width 2..31 and freqs of width 2..31, bitsets, all-same gaps and freqs of 8 / 16 / 32 bits, raw and
StreamVByte tails, single-doc terms, blocks larger than the 512-byte prefetch slot, and norm columns of none / 1 / 2 /
4 bytes. Built from explicit lists, so the expected doc ids and freqs are known without decoding. Results are compared
bit for bit with the oracle's exhaustive evaluation; decoded scores with a NumPy float32 statement of bm25()."""
import numpy as np
import pytest

import orc
import serenedb_b200 as sdb
from gpu_util import assert_hits_equal, ctx, oracle_terms, to_gpu
from shape_corpora import NORM_WIDTHS, bm25_f32, shape_segment

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=NORM_WIDTHS, ids=lambda w: f"norms{w or 0}")
def seg(request):
    oseg, norms, lists = shape_segment(request.param)
    g = to_gpu(oseg)
    ttf = int(norms.astype(np.uint64).sum()) if norms is not None else oseg.n_docs
    reader = sdb.IndexReader([g], oseg.n_docs, ttf, [len(d) for _, d, _ in lists])
    names = {name: t for t, (name, _, _) in enumerate(lists)}
    shapes = [t for t, (name, _, _) in enumerate(lists) if not name.endswith("+lead")]
    cache = {}

    def expect(kind, tis, k, mode=1):
        key = (kind, tuple(tis), k, mode)
        if key not in cache:
            cache[key] = orc.bm25_topk([oseg], kind, oracle_terms(reader, sdb.BM25(), tis), k, mode=mode)
        return cache[key]
    yield dict(oseg=oseg, g=g, norms=norms, lists=lists, reader=reader, names=names, shapes=shapes, expect=expect,
               width=request.param)
    ctx().set_wand(0)


def _queries(s):
    """Single terms, each shape ANDed with (and, as a lead-mode pair, ORed with) its shorter companion, and 2..4-term
    disjunctions across shapes."""
    rng = np.random.default_rng(7)
    sh = s["shapes"]
    q = [("OR", [t], 10) for t in sh]
    q += [("AND", [t, t + 1], 20) for t in sh if len(s["lists"][t][1]) > 1]
    q += [("OR", [t, t + 1], 10) for t in sh if len(s["lists"][t][1]) >= 40]
    for _ in range(24):
        tis = sorted(int(x) for x in rng.choice(sh, size=int(rng.integers(2, 5)), replace=False))
        q.append(("OR", tis, int(rng.choice([1, 10, 100]))))
    return q


def test_decode_score_every_shape(seg):
    scorer = sdb.BM25()
    for t, (name, docs, freqs) in enumerate(seg["lists"]):
        st = seg["reader"].stats(scorer, t)
        c0 = scorer.num(st)
        d, f, s = seg["g"].decode_score_term(t, c0, st.norm_const, st.norm_length)
        assert np.array_equal(d, docs), name
        assert np.array_equal(f, freqs), name
        norms = seg["norms"][docs - 1] if seg["norms"] is not None else np.ones(len(docs), np.uint32)
        exp = bm25_f32(freqs, norms, c0, st.norm_const, st.norm_length)
        assert np.array_equal(s.view(np.uint32), exp.view(np.uint32)), name


@pytest.mark.parametrize("wand", [0, 1, 2])
def test_topk_every_shape(seg, wand):
    ctx().set_wand(wand)
    scorer = sdb.BM25()
    for kind, tis, k in _queries(seg):
        hits, total = sdb.ExecuteTopK(seg["reader"], tis, sdb.AND if kind == "AND" else sdb.OR, scorer, k)
        oh, ototal, _ = seg["expect"](kind, tis, k)
        assert_hits_equal(hits, oh)
        if wand == 0 or kind == "AND":
            assert total == ototal, (kind, [seg["lists"][t][0] for t in tis])
        else:
            assert total <= ototal


@pytest.mark.parametrize("env", [{"SDBG_STREAM": "0"}], ids=["legacy"])
def test_topk_kernel_variants(seg, env, monkeypatch):
    """The legacy window kernel: same results."""
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    scorer = sdb.BM25()
    for wand in (0, 2):
        ctx().set_wand(wand)
        for kind, tis, k in _queries(seg):
            hits, total = sdb.ExecuteTopK(seg["reader"], tis, sdb.AND if kind == "AND" else sdb.OR, scorer, k)
            oh, ototal, _ = seg["expect"](kind, tis, k)
            assert_hits_equal(hits, oh)
            assert total == ototal if (wand == 0 or kind == "AND") else total <= ototal


def test_stream_scored_docs_every_shape(seg):
    if seg["width"] is None:
        pytest.skip("the oracle's dense evaluation of a 2^30-doc segment needs 5 GB of host memory")
    scorer = sdb.BM25()
    qs = [("OR", [t]) for t in seg["shapes"]] + [("AND", [t, t + 1]) for t in seg["shapes"][::3]]
    qs += [("OR", q) for q in ([seg["shapes"][i] for i in (0, 10, 20)], [seg["shapes"][i] for i in (5, 31, 40, 45)])]
    for kind, tis in qs:
        docs, scores = sdb.StreamScoredDocs(seg["reader"], 0, tis, sdb.AND if kind == "AND" else sdb.OR, scorer)
        oh, ototal, _ = seg["expect"](kind, tis, seg["oseg"].n_docs, mode=0)
        order = np.argsort(oh["doc"], kind="stable")
        assert len(docs) == ototal == len(oh), (kind, tis)
        assert np.array_equal(docs, oh["doc"][order])
        assert np.array_equal(scores.view(np.uint32), oh["score"][order].view(np.uint32))


def test_filter_and_deleted_docs(seg):
    """Hybrid filter plus a DocumentMask over the shapes: probes and streamed lists both skip deleted and filtered docs."""
    if seg["width"] != 2:
        pytest.skip("one norm width is enough for the per-doc checks")
    n = seg["oseg"].n_docs
    rng = np.random.default_rng(3)
    col = (np.arange(1, n + 1, dtype=np.int64) * 2654435761 % 1000).astype(np.int32)
    seg["oseg"].add_column(4, col)
    seg["g"].stage_column(4, col)
    every = np.unique(np.concatenate([d for _, d, _ in seg["lists"]]))
    deleted = every[rng.random(len(every)) < 0.2].astype(np.uint32)
    seg["oseg"].set_docs_mask(deleted)
    seg["g"].stage_docs_mask(deleted)
    scorer = sdb.BM25()
    try:
        for wand in (0, 2):
            ctx().set_wand(wand)
            for kind, tis, k in _queries(seg)[::2]:
                hits, total = sdb.ExecuteTopK(seg["reader"], tis, sdb.AND if kind == "AND" else sdb.OR, scorer, k,
                                              filt=sdb.pred(4, "BETWEEN", 100, 700))
                oh, ototal, _ = orc.bm25_topk([seg["oseg"]], kind, oracle_terms(seg["reader"], scorer, tis), k,
                                              filt=orc.make_pred(4, "BETWEEN", 100, 700), mode=1)
                assert_hits_equal(hits, oh)
                assert total == ototal if (wand == 0 or kind == "AND") else total <= ototal
                assert not np.isin(hits["doc"], deleted).any()
    finally:
        seg["oseg"].set_docs_mask([])
        seg["g"].stage_docs_mask(None)
