"""The GPU value-stream decoders byte for byte: every decoded value of every row, read back through the public C-ABI
with  GROUP BY rowid, bit_or(x1) ... bit_or(x7)  (one row per group, so bit_or is the value; a NULL row has count 0),
against the values that were inserted and the oracle's own decode of the same image (liblz4, libzstd, the pglz
restatement).  Each corpus (tests/decoder_corpus.py) runs through every staging path (cg_shard_stage, cg_scan_relation
from pageable pages, the DMA path), every LZ4 decoder form (eight lanes per stream, a lane per stream with one or several
streams per warp, the 32-stream lockstep form, the choice by launch size) and both zstd forms, on the default kernel
family and on the interpretive kernels."""
import numpy as np
import pytest

import decoder_corpus as dc
from gpu_harness import cg  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

NUM2 = 2 | (2 << 8)          # numeric(p, 2)


# decoder form -> cg_set_option values
FORMS = {
    "lz4 groups": dict(lz4_lanes=0),
    "lz4 lanes": dict(lz4_lanes=1, lz4_lane_warps=64),
    "lz4 lanes, several per warp": dict(lz4_lanes=1, lz4_lane_warps=1),
    "lz4 lanes lockstep": dict(lz4_lanes=1, lz4_lane_warps=0),
    "auto, zstd serial": dict(lz4_lanes=2, zstd_coop=0),
    "auto": dict(lz4_lanes=2, zstd_coop=1),
}
DEFAULTS = dict(lz4_lanes=-1, lz4_lane_warps=64, zstd_coop=-1)


@pytest.fixture
def form(cg, request):
    for k, v in FORMS[request.param].items():
        cg.set_option(k, v)
    yield request.param
    for k, v in DEFAULTS.items():
        cg.set_option(k, v)


class Rel:
    """a relation image, its column layout, and what every row must read back as: (values, nulls) per column"""

    def __init__(self, cg, name, pages, stripes, nodes, attlens, vals, nulls, limit, type_classes=None):
        self.name, self.attlens, self.vals, self.nulls = name, attlens, vals, nulls
        self.image = (pages, stripes, nodes, limit)
        self.rel = cg.Relation.from_image(pages, stripes, nodes, attlens, type_classes)


def _check_oracle_agrees(oracle, r, type_classes=None):
    pages, stripes, nodes, limit = r.image
    got, gotn = oracle.Table.attach(pages, stripes, nodes, r.attlens, type_classes, chunk_row_limit=limit).decode_all()
    for c in range(len(r.attlens)):
        assert np.array_equal(gotn[c], r.nulls[c]), (r.name, c)
        assert np.array_equal(np.where(gotn[c] == 1, 0, got[c]), np.where(r.nulls[c] == 1, 0, r.vals[c])), (r.name, c)


def _codec_rel(cg, oracle, name, kind, level, inserts, chunk, seed, first_rowid=0):
    t, vals, nulls = dc.codec_table(oracle, kind, level, inserts, chunk, seed, first_rowid)
    r = Rel(cg, name, t.pages(), t.stripes_array(), t.nodes_array(), dc.ATTLENS, vals, nulls, chunk)
    _check_oracle_agrees(oracle, r)
    return r


def _stream_rel(cg, oracle, name, chunks, attlen):
    pages, stripes, nodes, limit, rows = dc.image_with_streams(oracle, chunks, attlen)
    vals, nulls = [], []
    for kind, stream, raw in chunks:
        v, m = dc.expected_values(oracle.codec_decompress(kind, stream, raw) if kind else stream, attlen, max(raw // attlen, 1))
        vals.append(v)
        nulls.append(m)
    n = sum(rows)
    r = Rel(cg, name, pages, stripes, nodes, [8, attlen], [np.arange(n), np.concatenate(vals)],
            [np.zeros(n, np.uint8), np.concatenate(nulls)], limit)
    _check_oracle_agrees(oracle, r)
    return r


@pytest.fixture(scope="module")
def corpus(cg, oracle):
    if not (oracle.lib().orc_have_lz4() and oracle.lib().orc_have_zstd()):
        pytest.skip("liblz4 / libzstd missing")
    rels = []
    codecs = [("lz4", dc.COMP_LZ4, 0), ("pglz", dc.COMP_PGLZ, 0)] + [(f"zstd {l}", dc.COMP_ZSTD, l) for l in (1, 3, 9, 19)]
    for i, (name, kind, level) in enumerate(codecs):
        rels.append(_codec_rel(cg, oracle, f"{name} small chunks", kind, level, dc.SMALL_INSERTS, 2064, seed=i))
    for i, (name, kind, level) in enumerate(codecs[:3] + codecs[-1:]):
        rels.append(_codec_rel(cg, oracle, f"{name} 100000-row chunks", kind, level, [112_345], 100_000, seed=10 + i))
    rels.append(_codec_rel(cg, oracle, "lz4 3500 streams", dc.COMP_LZ4, 0, [7000], 16, seed=20))
    t, vals, nulls = dc.codec_table(oracle, dc.COMP_NONE, 0, [300, 2064, 1000, 17, 5000, 64], 2064, seed=21)
    pages, stripes, nodes = dc.recompress(oracle, t, [dc.COMP_LZ4, dc.COMP_PGLZ, dc.COMP_ZSTD, dc.COMP_NONE, dc.COMP_ZSTD, dc.COMP_LZ4])
    rels.append(Rel(cg, "mixed codecs", pages, stripes, nodes, dc.ATTLENS, vals, nulls, 2064))
    _check_oracle_agrees(oracle, rels[-1])
    for name, attlen, kind, cases in dc.HAND_RELATIONS:
        rels.append(_stream_rel(cg, oracle, f"hand {name}", dc.hand_relation_chunks(kind, cases), attlen))
    return rels


def _run(cg, rel, agg, path, want_stats=True):
    if path == "shard":
        sh = cg.Shard(rel)
        agg.scan_shard(sh, want_stats)
        sh.free()
    elif path == "dma":
        rel.register()
        try:
            agg.scan_relation(rel, want_stats)
        finally:
            rel.unregister()
    else:
        agg.scan_relation(rel, want_stats)


def _partial(cg, r, kmin=None, kmax=None, rows=None):
    d = dc.readback_desc(cg, r.attlens)
    k0, k1, _, n = cg.relation_bounds(r.rel, d)
    return cg.GpuColumnarAgg(d, r.rel.column_descs(), k0 if kmin is None else kmin, k1 if kmax is None else kmax,
                             max(n if rows is None else rows, 1))


def _check_readback(agg, attlens, vals, nulls, what):
    """the partial's groups against the expected rows: the key set is exactly the rowids, and per column the non-NULL
    count and the value (integers compared in their own width)"""
    f = agg.fetch()
    assert not f["key_nulls"].any(), what
    order = np.argsort(f["keys"], kind="stable")
    assert np.array_equal(f["keys"][order], vals[0]), what
    for a, w in enumerate(attlens[1:]):
        c = a + 1
        cnt = f["count"][order, a]
        assert np.array_equal(cnt == 0, nulls[c] == 1), (what, c, "NULLs")
        assert cnt.max(initial=0) <= 1, (what, c)
        if w < 0:
            lo, hi = f["sum_lo"][order, a].view(np.int64), f["sum_hi"][order, a]
            assert np.array_equal(hi, np.where(lo < 0, -1, 0)), (what, c)
            got = lo
        else:
            got = f["minmax"][order, a]
        live = nulls[c] == 0
        g, e = got[live], vals[c][live]
        if 0 < w < 8:
            mask = (1 << (8 * w)) - 1
            g, e = g & mask, e & mask
        bad = np.nonzero(g != e)[0]
        assert bad.size == 0, (what, c, f"{bad.size} wrong values, first at row {int(np.nonzero(live)[0][bad[0]])}")


def readback(cg, r, path, what):
    """one scan per kernel family: the default choice and the interpretive kernels"""
    for family in ("default", "general"):
        cg.set_option("force_general", 1 if family == "general" else 0)
        try:
            agg = _partial(cg, r)
            _run(cg, r.rel, agg, path)
            _check_readback(agg, r.attlens, r.vals, r.nulls, (what, r.name, family))
            agg.free()
        finally:
            cg.set_option("force_general", 0)


PATHS = ["shard", "pageable", "dma"]


@pytest.mark.parametrize("path", PATHS)
def test_readback_is_exact_on_uncompressed_relations(cg, oracle, path):
    """the readback on its own terms: a NONE-compressed relation reads back as the inserted arrays, NULLs included, for
    widths 1, 2, 4 and 8 at their extremes"""
    n = 20_000
    rng = np.random.default_rng(1)
    vals = [np.arange(n)] + [rng.integers(-2**(8 * w - 1), 2**(8 * w - 1) - 1, n, endpoint=True) for w in dc.ATTLENS[1:]]
    for c, w in enumerate(dc.ATTLENS[1:], 1):
        vals[c][:4] = [-2**(8 * w - 1), 2**(8 * w - 1) - 1, 0, -1]
    nulls = [np.zeros(n, np.uint8)] + [(rng.random(n) < p).astype(np.uint8) for p in (0, 0.1, 0.5, 0, 0.2, 0.01, 0.9)]
    nulls[3][2000:4000] = 1
    t = oracle.Table(dc.ATTLENS, stripe_row_limit=9000, chunk_row_limit=1000)
    t.insert(vals, nulls)
    r = Rel(cg, "uncompressed", t.pages(), t.stripes_array(), t.nodes_array(), dc.ATTLENS, vals, nulls, 1000)
    _check_oracle_agrees(oracle, r)
    readback(cg, r, path, "none")


@pytest.mark.parametrize("form", list(FORMS), indirect=True)
@pytest.mark.parametrize("path", PATHS)
def test_decoded_bytes_are_exact(cg, corpus, path, form):
    for r in corpus:
        readback(cg, r, path, form)


@pytest.mark.parametrize("form", ["lz4 groups", "lz4 lanes", "auto, zstd serial"], indirect=True)
@pytest.mark.parametrize("path", PATHS)
def test_malformed_streams_are_refused(cg, oracle, corpus, path, form):
    """each malformed stream is refused (CG_ECORRUPT) by a bounds check of the decoder, on every path; a clean relation
    scanned next still reads back exactly"""
    from citus_b200 import capi
    clean = next(r for r in corpus if r.name == "hand lz4")
    good = dc.Lz4Block().seq(b"0123456789", 10, 300).end(b"abcdefghijkl")
    for name, kind, stream, raw, _ in dc.MALFORMED:
        pages, stripes, nodes, limit, rows = dc.image_with_streams(oracle, [(dc.COMP_LZ4, good[0], len(good[1])), (kind, stream, raw)])
        bad = cg.Relation.from_image(pages, stripes, nodes, [8, 1])
        agg = cg.GpuColumnarAgg(dc.readback_desc(cg, [8, 1]), bad.column_descs(), 0, sum(rows) - 1, sum(rows))
        with pytest.raises(capi.CitusGpuError) as e:
            _run(cg, bad, agg, path)
            agg.fetch()
        assert e.value.code == capi.CG_ECORRUPT, (name, e.value)
        agg.free()
    readback(cg, clean, path, form)


def _varlena_rel(cg, oracle, first_rowid):
    rng = np.random.default_rng(5)
    n = 12_000
    vals = [np.arange(first_rowid, first_rowid + n), rng.integers(-10**12, 10**12, n)]
    nulls = [np.zeros(n, np.uint8), (rng.random(n) < 0.1).astype(np.uint8)]
    t = oracle.Table([8, -1], [0, NUM2], stripe_row_limit=5000, chunk_row_limit=1000, compression=dc.COMP_LZ4)
    t.insert(vals, nulls)
    r = Rel(cg, "varlena numeric lz4", t.pages(), t.stripes_array(), t.nodes_array(), [8, -1], vals, nulls, 1000, [0, NUM2])
    _check_oracle_agrees(oracle, r, [0, NUM2])
    return r


def test_back_to_back_scans_decode_every_byte(cg, oracle, corpus):
    """DMA path: compressed scans issued one after another without synchronising -- more of them than the three side
    streams the decoders rotate over, zstd on the compute stream -- each into its own partial, then each read back; then
    the same relations accumulated into one partial"""
    same = []
    first = 0
    for i, (name, kind) in enumerate((("lz4", dc.COMP_LZ4), ("pglz", dc.COMP_PGLZ), ("zstd", dc.COMP_ZSTD))):
        same.append(_codec_rel(cg, oracle, f"{name} b2b", kind, 3 if kind == dc.COMP_ZSTD else 0, [4000, 2000, 9000], 2064, 30 + i, first))
        first += 15_000
    t, vals, nulls = dc.codec_table(oracle, dc.COMP_NONE, 0, [3000, 3000, 3000, 3000], 2064, seed=40, first_rowid=first)
    pages, stripes, nodes = dc.recompress(oracle, t, [dc.COMP_ZSTD, dc.COMP_LZ4, dc.COMP_PGLZ, dc.COMP_NONE])
    same.append(Rel(cg, "mixed b2b", pages, stripes, nodes, dc.ATTLENS, vals, nulls, 2064))
    _check_oracle_agrees(oracle, same[-1])
    first += 12_000
    rels = same + [_varlena_rel(cg, oracle, first)]
    for r in rels:
        r.rel.register()
    try:
        aggs = [_partial(cg, r) for r in rels]
        for r, agg in zip(rels, aggs):
            agg.scan_relation(r.rel, want_stats=False)
        for r, agg in zip(rels, aggs):
            _check_readback(agg, r.attlens, r.vals, r.nulls, ("back to back", r.name))
            agg.free()
        # one partial over all the same-schema relations, rowids disjoint
        agg = _partial(cg, same[0], 0, first - 1, first)
        for r in same:
            agg.scan_relation(r.rel, want_stats=False)
        vals = [np.concatenate([r.vals[c] for r in same]) for c in range(len(dc.ATTLENS))]
        nulls = [np.concatenate([r.nulls[c] for r in same]) for c in range(len(dc.ATTLENS))]
        _check_readback(agg, dc.ATTLENS, vals, nulls, "accumulated")
        agg.free()
    finally:
        for r in rels:
            r.rel.unregister()
