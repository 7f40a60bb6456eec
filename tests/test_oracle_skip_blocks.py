"""CPU checks of kanzi's skipBlocks option (kanzi c --skip) as the tests state it (tests/skip_oracle.py): the Python statement of
encodingTask.encode's decision pins the oracle's (oracle/kzo_block.cpp encode_block) on magic numbers, block lengths and entropies on both
sides of INCOMPRESSIBLE_THRESHOLD; the skip streams decode back to their input at every level; and with the option off the stream model
is the oracle's stream byte for byte."""
import bz2
import ctypes as C
import gzip
import lzma

import numpy as np
import pytest

import skip_oracle as so

BS = 4096
LEVELS = [("NONE", "NONE"), ("LZX", "NONE"), ("DNA+LZ", "HUFFMAN"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")]  # -l 0 .. -l 5 (app/BlockCompressor.go)


def _text(n, seed=0):
    rng = np.random.default_rng(seed)
    words = [b"alpha ", b"beta ", b"gamma ", b"delta\n", b"kanzi ", b"block ", b"stored ", b"raw "]
    out = bytearray()
    while len(out) < n:
        out += words[int(rng.integers(len(words)))]
    return np.frombuffer(bytes(out[:n]), np.uint8)


def _led(head, n=2000, seed=1):
    """compressible text led by the given bytes"""
    return np.concatenate([np.frombuffer(head, np.uint8), _text(n - len(head), seed)])


def _oracle_stores(oracle, block):
    """the oracle's decision: the mode byte of its NONE & NONE record with skip_blocks carries COPY_BLOCK_MASK"""
    payload, _ = oracle.encode_block(block, 0, 0, 0, skip_blocks=True)
    return bool(payload[0] & 0x80)


def _check(oracle, block, want):
    assert so.stored(block) == want, so.reason(block)
    assert _oracle_stores(oracle, block) == want


COMPRESSED_HEADS = [k.to_bytes(4, "big") for k in (so.JPG, so.GIF, so.PNG, so.LZMA, so.ZSTD, so.BROTLI, so.CAB, so.ZIP, so.FLAC, so.XZ, so.KNZ, so.RAR)] + [
    so.BZIP2.to_bytes(3, "big") + b"9", so.ID3.to_bytes(3, "big") + b"\x04", so.GZIP.to_bytes(2, "big") + b"\x08\x00"]


@pytest.mark.parametrize("head", COMPRESSED_HEADS, ids=lambda h: h.hex())
def test_every_compressed_magic_is_stored(oracle, head):
    block = _led(head)
    assert so.block_entropy(block) < so.INCOMPRESSIBLE_THRESHOLD  # stored for its magic number alone
    assert so.reason(block) == "magic"
    _check(oracle, block, True)


def test_jpeg_app0_only(oracle):
    """GetMagicType returns the key itself for FFD8FFEx, and IsDataCompressed knows only FFD8FFE0"""
    _check(oracle, _led(b"\xff\xd8\xff\xe0"), True)
    for x in range(0xE1, 0xF0):
        _check(oracle, _led(b"\xff\xd8\xff" + bytes([x])), False)


@pytest.mark.parametrize("head", [b"%PDF", b"\x7fELF", b"RIFF", b"BM\x36\x00", b"MZ\x90\x00", b"\xfe\xed\xfa\xce", b"P5\x0a3"], ids=lambda h: h.hex())
def test_other_magic_numbers_are_not_stored(oracle, head):
    """recognised formats outside IsDataCompressed: PDF, ELF, RIFF, BMP, MZ, Mach-O, PGM"""
    assert so.magic_type(_led(head)) != 0
    _check(oracle, _led(head), False)


def test_block_lengths_15_and_16(oracle):
    rng = np.random.default_rng(3)
    r15, r16 = rng.integers(0, 256, 15, dtype=np.uint8), rng.integers(0, 256, 16, dtype=np.uint8)
    assert so.reason(r15) == "small"
    payload, _ = oracle.encode_block(r15, 0, 0, 0, skip_blocks=False)
    assert payload[0] & 0x80  # stored with the option off too
    _check(oracle, r15, True)
    assert so.block_entropy(np.arange(16, dtype=np.uint8)) == 512  # the most 16 bytes can give
    _check(oracle, np.arange(16, dtype=np.uint8), False)
    _check(oracle, np.concatenate([np.frombuffer(b"\x1f\x8b", np.uint8), r16[2:]]), True)
    _check(oracle, np.frombuffer(b"\x1f\x8b" + bytes(13), np.uint8), True)


def test_constant_and_uniform_blocks(oracle):
    rng = np.random.default_rng(4)
    for n in (16, 1000, 4096, 1 << 16):
        _check(oracle, np.full(n, 0x41, np.uint8), False)
    for n in (4096, 1 << 16, 1 << 20):
        u = rng.integers(0, 256, n, dtype=np.uint8)
        assert so.reason(u) == "entropy"
        _check(oracle, u, True)


@pytest.mark.parametrize("n", [1 << 12, 1 << 16])
def test_entropy_972_and_973(oracle, n):
    lo, hi = so.entropy_block(972, n, seed=5), so.entropy_block(973, n, seed=6)
    assert oracle.lib().kzo_entropy1024(lo.ctypes.data, lo.size) == 972
    assert oracle.lib().kzo_entropy1024(hi.ctypes.data, hi.size) == 973
    _check(oracle, lo, False)
    _check(oracle, hi, True)


def test_entropy_matches_the_oracle(oracle):
    rng = np.random.default_rng(7)
    for n in (16, 17, 255, 256, 257, 4095, 65537, 1 << 20):
        for alpha in (0.3, 1.0, 3.0):
            x = np.minimum(rng.zipf(1 + alpha, n) - 1, 255).astype(np.uint8)
            assert so.block_entropy(x) == oracle.lib().kzo_entropy1024(x.ctypes.data, C.c_size_t(n)), (n, alpha)


def corpus(seed=0):
    """BS-byte blocks: text, uniform random, stdlib gzip / bz2 / xz members, text led by a PNG signature and by FFD8FFE1, the 972 / 973
    blocks, then a short last block"""
    rng = np.random.default_rng(seed)
    t = _text(64 * BS, seed).tobytes()
    blocks = [_text(BS, seed + 1), rng.integers(0, 256, BS, dtype=np.uint8)]
    for member in (gzip.compress(t, mtime=0), bz2.compress(t), lzma.compress(t, format=lzma.FORMAT_XZ)):
        blocks.append(np.frombuffer((member * (BS // len(member) + 1))[:BS], np.uint8))
    blocks += [_led(b"\x89PNG", BS, seed + 2), _led(b"\xff\xd8\xff\xe1", BS, seed + 3), so.entropy_block(972, BS, seed + 4),
               so.entropy_block(973, BS, seed + 5), _text(BS, seed + 6)]
    return blocks


@pytest.mark.parametrize("tail", [15, 16, 1000])
def test_corpus_decisions(oracle, tail):
    blocks = corpus() + [np.frombuffer(b"\x1f\x8b" + bytes(i & 0xFF for i in range(tail - 2)), np.uint8)]
    got = [so.reason(b) for b in blocks]
    assert got == [None, "entropy", "magic", "magic", "magic", "magic", None, None, "entropy", None, "small" if tail == 15 else "magic"]
    for b, r in zip(blocks, got):
        assert _oracle_stores(oracle, b) == (r is not None)


@pytest.mark.parametrize("transform,entropy", LEVELS)
@pytest.mark.parametrize("checksum", [0, 32])
def test_skip_streams_roundtrip(oracle, transform, entropy, checksum):
    x = np.concatenate(corpus(seed=checksum) + [np.arange(16, dtype=np.uint8)])
    s = so.compress(oracle, x, transform, entropy, BS, checksum, input_size=x.size)
    assert np.array_equal(oracle.decompress(s, x.size + 64), x)
    off = so.compress(oracle, x, transform, entropy, BS, checksum, input_size=x.size, skip=False)
    assert np.array_equal(off, oracle.compress(x, transform, entropy, BS, checksum, input_size=x.size))
    assert not np.array_equal(s, off)


def test_none_none_differs_in_the_mode_byte(oracle):
    """a stored block carries COPY_BLOCK_MASK, a plain NONE & NONE block does not"""
    u = np.random.default_rng(8).integers(0, 256, BS, dtype=np.uint8)
    on, _ = oracle.encode_block(u, 0, 0, 0, skip_blocks=True)
    off, _ = oracle.encode_block(u, 0, 0, 0, skip_blocks=False)
    assert on[0] & 0x80 and not off[0] & 0x80
    assert np.array_equal(on[1:], off[1:]) and on[0] & 0x7F == off[0] & 0x7F
    s_on = so.compress(oracle, u, "NONE", "NONE", BS)
    s_off = so.compress(oracle, u, "NONE", "NONE", BS, skip=False)
    assert s_on.size == s_off.size and not np.array_equal(s_on, s_off)
