"""CPU checks of tests/foreign_streams.py: the module imports, every case labelled "shaped" decodes in the oracle, the LZ labels agree with
the model of what lzi_parse_kernel takes, and the one-stage block records decode like the stage itself."""
import numpy as np

import foreign_streams as fs


def test_shaped_lz_cases_decode_and_odd_ones_leave_the_parse(oracle):
    cases = fs.lz_cases()
    assert sum(label == "shaped" for _, _, label in cases) >= 30 and sum(label == "odd" for _, _, label in cases) >= 10
    for name, s, label in cases:
        try:
            d = oracle.transform_inverse(fs.T_LZ, s, 40 << 20, fill=0)
        except oracle.OracleError:
            d = None
        if label == "shaped":
            assert d is not None and fs.lz_parallel_shape(s), name
        elif label == "odd":
            assert d is None or not fs.lz_parallel_shape(s), name


def test_lz_writer_matches_the_oracle_forward_layout(oracle):
    """a parse written by hand decodes to what it describes"""
    lit = np.frombuffer(b"abcdefgh", np.uint8)
    s = fs.lz_stream([(lit, ("d", 12, 8, 1)), (lit[:2], ("r0", 5, 0, 0)), (np.frombuffer(b"0123456789ABCDEF", np.uint8), None)])
    want = b"abcdefgh" + b"abcdefghabcd" + b"ab" + b"ghabc" + b"0123456789ABCDEF"
    assert bytes(oracle.transform_inverse(fs.T_LZ, s, 200)) == want


def test_zrlt_repro_is_the_forward_of_a_long_run(oracle):
    x = np.concatenate([np.ones(8170, np.uint8), np.zeros((1 << 23) - 1, np.uint8)])
    assert np.array_equal(oracle.transform_forward(fs.T_ZRLT, x)[0], fs.zrlt_repro())
    assert np.array_equal(oracle.transform_inverse(fs.T_ZRLT, fs.zrlt_repro(), len(x)), x)


def test_generators_are_seeded(oracle):
    a, b = fs.zrlt_cases(), fs.zrlt_cases()
    assert all(x[0] == y[0] and np.array_equal(x[1], y[1]) for x, y in zip(a, b))
    m = fs.mutations([(n, s) for n, s, _ in fs.lz_cases()[:20]], 50, seed=1)
    assert all(x[0] == y[0] and np.array_equal(x[1], y[1]) for x, y in zip(m, fs.mutations([(n, s) for n, s, _ in fs.lz_cases()[:20]], 50, seed=1)))
    assert len(fs.mm_cases()) > 1000 and len(fs.alias_cases()) > 100 and len(fs.text_cases(oracle)) > 100


def test_block_record_decodes_like_the_stage(oracle):
    for name, s in fs.mm_cases()[:300:7] + [(n, s) for n, s, _ in fs.alias_cases()[:60]]:
        t = fs.T_MM if name.startswith(("m", "ff", "esc", "all")) else fs.T_PACK
        p, bits = fs.block_record(s)
        room = (1 << 16) + 4096
        try:
            want = oracle.transform_inverse(t, s, room, fill=0)
        except oracle.OracleError:
            want = None
        try:
            got = oracle.decode_block(p, bits, t << 42, 0, 0, 1 << 16)
        except oracle.OracleError:
            got = None
        assert (want is None) == (got is None) and (want is None or np.array_equal(want, got)), name
