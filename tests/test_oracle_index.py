"""CPU check of the index model (tests/index_oracle.py) against the oracle: at -l 0 .. 5, checksums 0 / 32 / 64, headered and headerless,
the model's record positions and header fields are the stream's, its reads are slices of the oracle's decode, a damaged block fails the
requests on it with the code of decoding it alone, and the blob it states is self-consistent."""
import struct

import numpy as np
import pytest

import headerless_oracle as ho
import index_oracle as io_
import range_oracle as ro

LEVELS = [("NONE", "NONE"), ("PACK+LZ", "NONE"), ("DNA+LZ", "HUFFMAN"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")]
BS = 1024


@pytest.mark.parametrize("ck", [0, 32, 64])
@pytest.mark.parametrize("level", range(6))
def test_model_reads_are_slices_of_the_decode(oracle, level, ck):
    tr, en = LEVELS[level]
    rng = np.random.default_rng(level * 3 + ck)
    n = 7 * BS - 100
    x = np.frombuffer(bytes(rng.choice(np.frombuffer(b"abcdefgh \n", np.uint8), n)), np.uint8)
    t48, et = oracle.parse_transform(tr), oracle.parse_entropy(en)
    for headerless in (False, True):
        if headerless:
            s = ho.compress(oracle, x, tr, en, BS, ck)
            m = io_.build(oracle, s, {"transform48": t48, "entropy": et, "block_size": BS, "checksum_bits": ck, "output_size": -1})
            assert m["header_bits"] == 0 and m["input_size"] == 0
        else:
            s = oracle.compress(x, tr, en, block_size=BS, checksum_bits=ck, input_size=n)
            m = io_.build(oracle, s)
            assert m["input_size"] == n and m["header_bits"] == ro.header_bits(s)
        assert (m["transform48"], m["entropy"], m["block_size"], m["checksum_bits"], m["nblocks"], m["size"]) == (t48, et, BS, ck, 7, -1)
        reqs = [(0, n), (5, 0), (BS - 1, 2), (n - 3, 10), (n, 1), (1 << 40, 5), (2 * BS, 3 * BS)] + [(int(o), int(k)) for o, k in
                                                                                              zip(rng.integers(0, n, 20), rng.integers(0, 3000, 20))]
        assert m["size"] == -1
        for (o, k), got in zip(reqs, io_.read(oracle, s, m, reqs)):
            assert got == ("ok", x[o: o + k].tobytes())
        assert m["size"] == n
        # the blob: fixed fields, the records, and a hash that covers them
        b = io_.blob(m)
        assert len(b) == 104 + 16 * 7 and struct.unpack_from("<Q", b, 48)[0] == 7 and struct.unpack_from("<q", b, 56)[0] == n
        assert [struct.unpack_from("<Q", b, 96 + 8 * i)[0] for i in range(14)] == [p for p, _ in m["recs"]] + [k for _, k in m["recs"]]
        assert struct.unpack_from("<Q", b, len(b) - 8)[0] == io_.xxh64(b[:-8])
        # damage in block 3: the requests on it fail with the code of decoding it alone, the others are untouched
        if not headerless:
            for kind in ["header"] + (["checksum"] if ck else []):
                bad = ro.corrupt(s, m["recs"][3], kind)
                mb = io_.build(oracle, bad)
                alone = ro.outcome(ro.decompress_range, oracle, bad, 4, 5)
                assert alone[0] == "err"
                for (o, k), got in zip(reqs, io_.read(oracle, bad, mb, reqs)):
                    k = min(k, n - o) if o < n else 0
                    if k and o // BS <= 3 <= (o + k - 1) // BS:
                        assert got == alone
                    else:
                        assert got == ("ok", x[o: o + k].tobytes())


def test_empty_stream_and_bad_streams(oracle):
    s = oracle.compress(np.zeros(0, np.uint8), "NONE", "NONE", block_size=BS)
    m = io_.build(oracle, s)
    assert (m["nblocks"], m["size"]) == (0, 0) and io_.read(oracle, s, m, [(0, 5), (0, 0)]) == [("ok", b""), ("ok", b"")]
    assert len(io_.blob(m)) == 104
    x = np.arange(3000, dtype=np.uint32).astype(np.uint8)
    s = oracle.compress(x, "LZ", "HUFFMAN", block_size=BS)
    with pytest.raises(Exception) as e:
        io_.build(oracle, s[:-1])
    assert e.value.code == 13
