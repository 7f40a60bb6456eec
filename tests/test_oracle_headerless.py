"""CPU checks of the headerless stream model (tests/headerless_oracle.py) the GPU tests compare against: the headerless stream is the
oracle's stream without its header bits, block by block; an empty input gives the end marker alone; the headerless reader round-trips;
and the parameter check returns validateHeaderless's codes."""
import math

import numpy as np
import pytest

import headerless_oracle as hlo
import range_oracle as ro

BS = 1024
CHAINS = [("NONE", "NONE"), ("BWT+RANK+ZRLT", "ANS0"), ("BWTS+MTFT+ZRLT", "ANS1"), ("LZ", "RANGE"), ("LZX", "HUFFMAN"), ("ROLZ", "NONE")]
SIZES = [0, 1, 1023, 4 * BS, 4 * BS + 377]


def _data(n, seed=7):
    """Compressible bytes: words from a small vocabulary with some noise."""
    rng = np.random.default_rng(seed + n)
    words = [b"alpha ", b"beta ", b"gamma ", b"delta\n", b"kanzi ", b"block ", b"\x00\x01\x02\x03"]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(len(words)))] if rng.random() < 0.9 else bytes(rng.integers(0, 256, 3, dtype=np.uint8))
    return np.frombuffer(bytes(out[:n]), np.uint8)


@pytest.mark.parametrize("transform,entropy", CHAINS)
@pytest.mark.parametrize("checksum", [0, 32, 64])
@pytest.mark.parametrize("hint", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_headerless_is_the_stream_without_its_header(oracle, transform, entropy, checksum, hint, n):
    data = _data(n)
    s = oracle.compress(data, transform, entropy, BS, checksum, input_size=n if hint else 0)
    hb = ro.header_bits(s)
    assert hb == 160 + (16 if hint and 0 < n < 1 << 16 else 0)
    total = hlo.end_bit(s, hb)
    assert (total + 7) // 8 == len(s)
    hl = hlo.records(oracle, data, transform, entropy, BS, checksum)
    assert len(hl) == math.ceil((total - hb) / 8)
    assert np.array_equal(np.unpackbits(hl)[: total - hb], np.unpackbits(np.frombuffer(bytes(s), np.uint8))[hb:total])
    assert np.array_equal(hl, hlo.compress(oracle, data, transform, entropy, BS, checksum, input_size=n if hint else 0))


@pytest.mark.parametrize("transform,entropy", CHAINS[:3])
def test_empty_input_is_the_end_marker(oracle, transform, entropy):
    assert bytes(hlo.records(oracle, b"", transform, entropy, BS)) == b"\x00"
    assert bytes(hlo.compress(oracle, b"", transform, entropy, BS, 32, input_size=5)) == b"\x00"


@pytest.mark.parametrize("transform,entropy", CHAINS)
@pytest.mark.parametrize("checksum", [0, 32, 64])
@pytest.mark.parametrize("n", SIZES)
def test_headerless_roundtrip(oracle, transform, entropy, checksum, n):
    data = _data(n, seed=11)
    hl = hlo.compress(oracle, data, transform, entropy, BS, checksum)
    assert bytes(hlo.decompress(oracle, hl, transform, entropy, BS, checksum)) == bytes(data)
    nblocks = -(-n // BS)
    if nblocks >= 3:
        part = hlo.decompress(oracle, hl, transform, entropy, BS, checksum, from_block=2, to_block=nblocks)
        assert bytes(part) == bytes(data[BS: (nblocks - 1) * BS])


def test_headerless_truncated_and_corrupt(oracle):
    data = _data(4 * BS + 377)
    hl = hlo.compress(oracle, data, "BWT+RANK+ZRLT", "ANS0", BS, 32)
    assert ro.outcome(hlo.decompress, oracle, hl[:-3], "BWT+RANK+ZRLT", "ANS0", BS, 32) == ("err", 13)
    recs = ro.walk(hl, 0)
    st, code = ro.outcome(hlo.decompress, oracle, ro.corrupt(hl, recs[1], "checksum"), "BWT+RANK+ZRLT", "ANS0", BS, 32)
    assert (st, code) == ("err", 19)


T_BWT, T_SNAPPY, T_SRT = 1 << 42, 4 << 42, 13 << 42


@pytest.mark.parametrize("args,code", [
    ((T_BWT, 5, BS, 0, 6), 0),
    ((T_SRT, 6, 1 << 30, 64, 6), 0),       # a kanzi chain and codec: valid here; the GPU answers CREATE_CODEC for them
    ((T_BWT, 5, BS, 0, 7), 18),            # bsVersion > 6 (:1184-1187)
    ((T_BWT, 5, BS, 0, 5), 16),            # older versions: not read by the GPU decoders
    ((T_BWT, 3, BS, 0, 6), 18),            # PAQ: no entropy.GetType name
    ((T_BWT, 10, BS, 0, 6), 18),
    ((T_SNAPPY, 5, BS, 0, 6), 18),         # SNAPPY: no transform.GetType name
    ((20 << 42, 5, BS, 0, 6), 18),
    ((1 << 48, 5, BS, 0, 6), 18),
    ((T_BWT, 5, 1023, 0, 6), 18),          # block size outside [1024, 1 GiB] (:1236-1239): INVALID_PARAM, not BLOCK_SIZE
    ((T_BWT, 5, (1 << 30) + 16, 0, 6), 18),
    ((T_BWT, 5, 1025, 0, 6), 0),           # the reference does not ask for a multiple of 16 here
    ((T_BWT, 5, BS, 16, 6), 18),           # checksum not 0 / 32 / 64 (:1254-1256)
])
def test_validate_headerless_codes(args, code):
    assert hlo.validate(*args) == code
