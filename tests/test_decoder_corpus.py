"""CPU checks of the decoder corpus (tests/decoder_corpus.py) that tests/test_gpu_decoders.py feeds to the GPU decoders:
every hand-assembled stream decodes, through liblz4 / libzstd / the pglz restatement, to the bytes computed while it
was assembled, and every malformed one is refused by them; the images that carry the streams are valid relations for
the library and decode, through the oracle's reader, to exactly those bytes; the readback query generates valid sm_90a
code.  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import decoder_corpus as dc


@pytest.fixture(scope="module")
def cg():
    from citus_b200 import build
    build.build()
    from citus_b200 import capi, columnar
    capi.lib()
    return columnar


def _have(oracle, kind):
    return {dc.COMP_LZ4: oracle.lib().orc_have_lz4, dc.COMP_ZSTD: oracle.lib().orc_have_zstd}.get(kind, lambda: 1)()


def test_hand_assembled_streams_agree_with_the_codecs(oracle):
    """the expected bytes of every hand stream were computed by copying bytes while the stream was assembled; the codec
    the reference calls (DecompressBuffer) must produce the same bytes"""
    seen = 0
    for name, _, kind, cases in dc.HAND_RELATIONS:
        if not _have(oracle, kind):
            pytest.skip("codec library missing")
        for case, (stream, want) in cases.items():
            assert oracle.codec_decompress(kind, stream, len(want)) == want, (name, case)
            seen += 1
    assert seen == sum(len(c) for _, _, _, c in dc.HAND_RELATIONS) >= 100
    # the shapes the GPU decoders branch on are really there
    assert any(len(w) > 65_535 for s, w in dc.HAND_LZ4.values())
    assert dc.HAND_LZ4["empty block"] == (b"\0", b"")
    assert any(len(s) == 9 + 3 + 131_072 for s, _ in dc.HAND_ZSTD_LARGE.values())       # one raw block of 128 KB


def test_xxh64_known_answers():
    """the content checksum of the hand frames: XXH64 with seed 0 (reference values of the xxHash test vectors)"""
    assert dc.xxh64(b"") == 0xEF46DB3751D8E999
    assert dc.xxh64(b"a") == 0xD24EC4F1A98C6E5B
    assert dc.xxh64(b"abc") == 0x44BC2CF5AD770999
    assert dc.xxh64(b"Nobody inspects the spammish repetition") == 0xFBCEA83C8A378BF1


def test_malformed_streams_are_refused_by_the_codecs(oracle):
    for name, kind, stream, raw, _ in dc.MALFORMED:
        if not _have(oracle, kind):
            continue
        if name == "lz4 offset 0":
            continue        # liblz4 copies whatever its output buffer held; the GPU decoders refuse it (a corrupt stream)
        with pytest.raises(oracle.OracleError):
            oracle.codec_decompress(kind, stream, raw)


def _library_checks(cg, rel, rows, limit):
    """validate_relation (behind every entry point), the chunk mask and the bounds of the readback query"""
    from citus_b200 import capi
    d = dc.readback_desc(cg, [rel.view.columns[i].attlen for i in range(rel.natts)])
    for s in range(rel.view.nstripes):
        mask = np.zeros(rel.view.stripes[s].chunk_count, np.uint8)
        f = C.c_int64(-1)
        capi.check(capi.lib().cg_selected_chunk_mask(C.byref(rel.view), s, C.byref(d), mask.ctypes.data, C.byref(f)))
        assert mask.all() and f.value == 0
    kmin, kmax, _, n = cg.relation_bounds(rel, d)
    assert (kmin, kmax, n) == (0, rows - 1, rows)


def test_images_with_streams_decode_to_the_streams(cg, oracle):
    """every hand relation: a valid image for the library, and the oracle's reader (DecompressBuffer per chunk) decodes
    the x column to the expected bytes, NULL rows where a chunk holds fewer values than rows"""
    for name, attlen, kind, cases in dc.HAND_RELATIONS:
        if not _have(oracle, kind):
            continue
        chunks = dc.hand_relation_chunks(kind, cases)
        pages, stripes, nodes, limit, rows = dc.image_with_streams(oracle, chunks, attlen)
        rel = cg.Relation.from_image(pages, stripes, nodes, [8, attlen])
        _library_checks(cg, rel, sum(rows), limit)
        vals, nulls = oracle.Table.attach(pages, stripes, nodes, [8, attlen], chunk_row_limit=limit).decode_all()
        assert np.array_equal(vals[0], np.arange(sum(rows))) and not nulls[0].any()
        at = 0
        for (k, stream, raw), r in zip(chunks, rows):
            want = oracle.codec_decompress(k, stream, raw) if k else stream
            v, m = dc.expected_values(want, attlen, r)
            assert np.array_equal(vals[1][at:at + r], v) and np.array_equal(nulls[1][at:at + r], m), (name, k, raw)
            at += r
        assert {n.compression_type for n in oracle.Table.attach(pages, stripes, nodes, [8, attlen]).nodes()} >= {0, kind}


def test_malformed_images_are_refused_by_the_oracle(cg, oracle):
    for name, kind, stream, raw, _ in dc.MALFORMED:
        if not _have(oracle, kind) or name == "lz4 offset 0":
            continue
        pages, stripes, nodes, limit, rows = dc.image_with_streams(oracle, [(kind, stream, raw)])
        _library_checks(cg, cg.Relation.from_image(pages, stripes, nodes, [8, 1]), sum(rows), limit)
        with pytest.raises(oracle.OracleError):
            oracle.Table.attach(pages, stripes, nodes, [8, 1], chunk_row_limit=limit).decode_all()


def _check_decodes_to(oracle, pages, stripes, nodes, limit, vals, nulls):
    got, gotn = oracle.Table.attach(pages, stripes, nodes, dc.ATTLENS, chunk_row_limit=limit).decode_all()
    for c in range(len(dc.ATTLENS)):
        assert np.array_equal(gotn[c], nulls[c]), c
        assert np.array_equal(np.where(nulls[c] == 1, 0, got[c]), np.where(nulls[c] == 1, 0, vals[c])), c


def test_codec_written_relations_decode_to_the_inserted_values(cg, oracle):
    """the oracle's writer with each codec: its reader gives back what was inserted; pglz stores the incompressible
    column raw next to the compressed ones; the many-chunk relation has more than 16 streams per SM of a 132-SM H100 in
    one stage, so "auto" picks the eight-lanes-per-stream LZ4 kernel there"""
    for kind, level in ((dc.COMP_LZ4, 0), (dc.COMP_PGLZ, 0), (dc.COMP_ZSTD, 1), (dc.COMP_ZSTD, 19)):
        if not _have(oracle, kind):
            continue
        t, vals, nulls = dc.codec_table(oracle, kind, level, dc.SMALL_INSERTS, 2064, seed=kind)
        kinds = {n.compression_type for n in t.nodes()}
        assert kind in kinds and (kind != dc.COMP_PGLZ or dc.COMP_NONE in kinds)
        assert any(n.decompressed_size == 0 and n.row_count > 0 for n in t.nodes())     # the all-NULL chunk
        _check_decodes_to(oracle, t.pages(), t.stripes_array(), t.nodes_array(), 2064, vals, nulls)
        rel = cg.Relation.from_image(t.pages(), t.stripes_array(), t.nodes_array(), dc.ATTLENS)
        _library_checks(cg, rel, sum(dc.SMALL_INSERTS), 2064)
    if oracle.lib().orc_have_lz4():
        t, vals, nulls = dc.codec_table(oracle, dc.COMP_LZ4, 0, [7000], 16, seed=9)
        assert sum(n.compression_type == dc.COMP_LZ4 for n in t.nodes()) > 132 * 16
        _check_decodes_to(oracle, t.pages(), t.stripes_array(), t.nodes_array(), 16, vals, nulls)


def test_recompressed_relation_mixes_every_codec(cg, oracle):
    """ALTER TABLE ... SET (compression ...) between inserts: stripes of LZ4, pglz, zstd and raw streams in one relation"""
    if not (oracle.lib().orc_have_lz4() and oracle.lib().orc_have_zstd()):
        pytest.skip("codec library missing")
    t, vals, nulls = dc.codec_table(oracle, dc.COMP_NONE, 0, [300, 2064, 1000, 17, 5000, 64], 2064, seed=3)
    kinds = [dc.COMP_LZ4, dc.COMP_PGLZ, dc.COMP_ZSTD, dc.COMP_NONE, dc.COMP_ZSTD, dc.COMP_LZ4]
    pages, stripes, nodes = dc.recompress(oracle, t, kinds)
    att = oracle.Table.attach(pages, stripes, nodes, dc.ATTLENS, chunk_row_limit=2064)
    assert {n.compression_type for n in att.nodes()} == {0, 1, 2, 3}
    _check_decodes_to(oracle, pages, stripes, nodes, 2064, vals, nulls)
    _library_checks(cg, cg.Relation.from_image(pages, stripes, nodes, dc.ATTLENS), sum([300, 2064, 1000, 17, 5000, 64]), 2064)


def test_readback_query_generates_valid_code(cg):
    """GROUP BY rowid, bit_or(x1) ... bit_or(x7) over the corpus's column layouts, direct-indexed over 10^6 keys, and
    sum over a numeric column: the generated kernels compile for sm_90a"""
    from citus_b200 import capi
    for lens in (dc.ATTLENS, [8, 1], [8, 4], [8, -1]):
        d = dc.readback_desc(cg, lens)
        cols = (capi.CgColumnDesc * len(lens))()
        for i, l in enumerate(lens):
            cols[i].attlen, cols[i].type_class = l, (2 | (2 << 8) if l < 0 else 0)
        kind = C.c_int32(-1)
        buf = C.create_string_buffer(1 << 19)
        rc = capi.lib().cg_jit_compile_check(C.byref(d), cols, len(lens), 0, 999_999, 10**6, C.byref(kind), buf, len(buf))
        assert rc == 0, capi.lib().cg_last_error().decode()
        assert kind.value == 2 and buf.value
