"""GPU tests of writes into a compressed stream (kz_write_ranges[_device], StreamIndex.write_many / write / append / write_many_device):
the new stream src[:keep] + tail is byte for byte what compress gives for the new data, on the level chains -l 0 .. 5 with checksums
0 / 32 / 64, headered (input-size hint 0 and not) and headerless, skip blocks off and on; the updated index is the rebuilt one apart from
the size, reads through it and a decompress of the new stream give the new data; host and device variants agree; successive appends equal
one compress; the work a call does (kz_profile); the errors; and, for -l 3 and -l 5, the oracle's compress of the new data."""
import struct

import numpy as np
import pytest

import index_oracle as io_

pytestmark = pytest.mark.gpu

LEVELS = [("NONE", "NONE"), ("LZX", "NONE"), ("DNA+LZ", "HUFFMAN"), ("TEXT+UTF+PACK+MM+LZX", "HUFFMAN"), ("TEXT+UTF+EXE+PACK+MM+ROLZ", "NONE"),
          ("TEXT+UTF+BWT+RANK+ZRLT", "ANS0")]
# (checksum bits, header: "hint" / "zero" / "none", skip blocks)
MODES = [(0, "hint", False), (32, "zero", True), (64, "none", False)]
BS = 1024


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def to_dev(torch, a, extra=64):
    d = torch.zeros(len(a) + extra, dtype=torch.uint8, device="cuda")
    if len(a):
        d[: len(a)] = torch.from_numpy(np.ascontiguousarray(a, np.uint8)).cuda()
    return d


def apply(x, writes):
    """pwrite model: writes in order, a gap reads as zeros, WRITE_APPEND is the current end."""
    y = bytearray(x.tobytes())
    for o, d in writes:
        d = bytes(d)
        if not d:
            continue
        o = len(y) if o == (1 << 64) - 1 else o
        if o > len(y):
            y += bytes(o - len(y))
        y[o:o + len(d)] = d
    return np.frombuffer(bytes(y), np.uint8)


class Setup:
    def __init__(self, kz, gpu, chain, ck, header, skip, bs=BS):
        self.kz, self.gpu, self.tr, self.en, self.ck, self.header, self.skip, self.bs = kz, gpu, chain[0], chain[1], ck, header, skip, bs
        self.hl = None
        if header == "none":
            self.hl = {"transform": kz.transform_type(self.tr), "entropy": kz.entropy_type(self.en), "block_size": bs, "checksum_bits": ck}

    def hint(self, x):
        return len(x) if self.header == "hint" else 0

    def compress(self, y, hint):
        return self.gpu.compress(y, self.tr, self.en, block_size=self.bs, checksum_bits=self.ck, input_size=hint, headerless=self.header == "none",
                                 skip_blocks=self.skip)


def blob_but_size(ix):
    b = ix.save()
    return b[:56] + b[64:-8]


def check_write(kz, gpu, torch, st, x, writes, device=True):
    """Writes into the stream of x; checks the new stream, the updated index, reads and decompress; the device variant against the host one.
    Returns (keep, new stream, host index)."""
    hint = st.hint(x)
    s = st.compress(x, hint)
    y = apply(x, writes)
    gpu.set_skip_blocks(st.skip)
    try:
        ix = gpu.index(s, headerless=st.hl)
        keep, tail = ix.write_many(s, writes)
        written = ix.save()  # before the reads below learn the size
        new = np.concatenate([s[:keep], np.frombuffer(tail, np.uint8)])
        want = st.compress(y, hint)
        assert new.tobytes() == want.tobytes()
        if not [w for w in writes if len(w[1])]:
            assert keep == len(s) and tail == b""
        rebuilt = gpu.index(new, headerless=st.hl)
        assert blob_but_size(ix) == blob_but_size(rebuilt)
        assert ix.size in (-1, len(y))
        if len(y):
            assert ix.read(new, 0, len(y) + 10) == y.tobytes()
        assert gpu.decompress(new, len(y) + 64, headerless=st.hl).tobytes() == y.tobytes()
        if device:
            ixd = gpu.index(s, headerless=st.hl)
            bufs = [np.frombuffer(bytes(d), np.uint8) for _, d in writes]
            data = np.concatenate(bufs) if bufs else np.zeros(0, np.uint8)
            ln = [b.size for b in bufs]
            doff = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64) if ln else []
            d_src, d_data = to_dev(torch, s), to_dev(torch, data)
            cap = len(s) + sum(n // st.bs + 2 for n in ln) * kz.load_library().kz_max_block_output(st.bs) + 16 + len(y)
            d_dst = torch.zeros(cap, dtype=torch.uint8, device="cuda")
            kd, nd = ixd.write_many_device(d_src, len(s), [w[0] for w in writes], ln, d_data, doff, d_dst, cap)
            assert kd == keep and d_dst[:nd].cpu().numpy().tobytes() == tail
            assert ixd.save() == written
        return keep, new, ix
    finally:
        gpu.set_skip_blocks(False)


def scenarios(rng, n, bs):
    blob = lambda k: rng.integers(0, 256, k, dtype=np.uint8).tobytes()  # noqa: E731
    text = lambda k: (b"the quick brown fox " * (k // 20 + 1))[:k]  # noqa: E731
    A = (1 << 64) - 1
    return [
        [(2 * bs + 100, text(300))],                                   # inside one block
        [(bs - 50, blob(200))],                                        # across two blocks
        [(bs, text(bs))],                                              # a whole block
        [(10, text(40)), (20, blob(10)), (5, text(100))],              # overlapping batch, later wins
        [(n + 3 * bs + 7, text(33))],                                  # a zero gap
        [(A, text(500)), (A, blob(bs + 3))],                           # appends
        [(100, b""), (n + 5, b"")],                                    # no-op
        [(0, text(n + 10))],                                           # everything
    ]


@pytest.mark.parametrize("mode", MODES, ids=["ck%d-%s-skip%d" % m for m in MODES])
@pytest.mark.parametrize("level", range(len(LEVELS)))
def test_writes_match_compress(kz, gpu, synth, torch, level, mode):
    ck, header, skip = mode
    st = Setup(kz, gpu, LEVELS[level], ck, header, skip)
    rng = np.random.default_rng(level * 10 + ck)
    n = 5 * BS - 300
    x = np.ascontiguousarray(synth.markov_text(n, seed=level + 1)[:n], np.uint8)
    for writes in scenarios(rng, n, BS):
        check_write(kz, gpu, torch, st, x, writes)
    # an empty stream, and a stream with a full last block
    check_write(kz, gpu, torch, st, np.zeros(0, np.uint8), [((1 << 64) - 1, b"hello " * 300)])
    check_write(kz, gpu, torch, st, x[: 3 * BS], [((1 << 64) - 1, b"tail" * 100)])


def test_unknown_size_and_loaded_index(kz, gpu, synth, torch):
    st = Setup(kz, gpu, LEVELS[2], 32, "hint", False)
    n = 6 * BS - 77
    x = np.ascontiguousarray(synth.markov_text(n, seed=3)[:n], np.uint8)
    s = st.compress(x, n)
    for writes in ([(100, b"abc")], [((1 << 64) - 1, b"xyz" * 50)], [(5 * BS, b"q" * BS), ((1 << 64) - 1, b"r" * 10)]):
        ix = kz.StreamIndex.load(gpu.index(s).save(), gpu)
        assert ix.size == -1
        keep, tail = ix.write_many(s, writes)
        y = apply(x, writes)
        assert s[:keep].tobytes() + tail == st.compress(y, n).tobytes()
        assert ix.size in (-1, len(y))


def test_successive_appends(kz, gpu, synth, torch):
    st = Setup(kz, gpu, LEVELS[2], 32, "zero", False)
    rng = np.random.default_rng(9)
    x = np.zeros(0, np.uint8)
    s = st.compress(x, 0)
    ix = gpu.index(s)
    for _ in range(50):
        p = synth.markov_text(int(rng.integers(0, 3000)) + 1, seed=int(rng.integers(1 << 30)))
        keep, tail = ix.append(s, p)
        s = np.concatenate([s[:keep], np.frombuffer(tail, np.uint8)])
        x = np.concatenate([x, p])
    assert s.tobytes() == st.compress(x, 0).tobytes()
    assert ix.size == len(x) and blob_but_size(ix) == blob_but_size(gpu.index(s))


def test_work(kz, gpu, synth):
    st = Setup(kz, gpu, LEVELS[3], 0, "hint", False, bs=4096)
    n = 8 * 4096
    x = np.ascontiguousarray(synth.markov_text(n, seed=2)[:n], np.uint8)
    s = st.compress(x, n)

    def work(writes):
        ix = gpu.index(s)
        ix.read(s, n - 1, 1)  # the size is known
        gpu.profile(True)
        gpu.profile_reset()
        try:
            ix.write_many(s, writes)
            return gpu.stage_bytes("write:decoded")[1], gpu.stage_bytes("write:encoded")[1]
        finally:
            gpu.profile(False)

    assert work([(3 * 4096 + 1000, b"w" * 2048)]) == (1, 1)
    assert work([(2 * 4096, b"w" * 4096)]) == (0, 1)
    assert work([((1 << 64) - 1, b"w" * 100)]) == (0, 1)


@pytest.mark.parametrize("level", [3, 5])
def test_oracle_parity(kz, gpu, oracle, synth, torch, level):
    tr, en = LEVELS[level]
    n = 4 * BS - 100
    x = np.ascontiguousarray(synth.markov_text(n, seed=11)[:n], np.uint8)
    s = oracle.compress(x, tr, en, block_size=BS, checksum_bits=32, input_size=n)
    ix = gpu.index(s)
    writes = [(BS + 17, b"oracle parity " * 20), ((1 << 64) - 1, b"appended " * 30)]
    keep, tail = ix.write_many(s, writes)
    y = apply(x, writes)
    assert s[:keep].tobytes() + tail == oracle.compress(y, tr, en, block_size=BS, checksum_bits=32, input_size=n).tobytes()


def test_errors(kz, gpu, synth, torch):
    st = Setup(kz, gpu, LEVELS[0], 32, "hint", False)
    n = 6 * BS
    x = np.ascontiguousarray(synth.markov_text(n, seed=4)[:n], np.uint8)
    s = st.compress(x, n)
    ix = gpu.index(s)
    # a stale index
    s2 = s.copy()
    s2[3] ^= 1
    with pytest.raises(kz.KanziError) as e:
        ix.write(s2, 10, b"x")
    assert e.value.code == 18
    # a damaged record in a block that must be decoded: the CRC code, index and bytes unchanged
    bad = s.copy()
    bad[(ix_start(ix, 2) + 200) // 8] ^= 0x10
    ixb = gpu.index(bad)
    before, copy = ixb.save(), bad.copy()
    with pytest.raises(kz.KanziError) as e:
        ixb.write(bad, 2 * BS + 5, b"zz")
    assert e.value.code == 19 and ixb.save() == before and (bad == copy).all()
    # a damaged record nobody decodes is moved as it is, not reported
    keep, tail = ixb.write(bad, 0, b"head")
    new = np.concatenate([bad[:keep], np.frombuffer(tail, np.uint8)])
    with pytest.raises(kz.KanziError):
        gpu.decompress(new, n + 64)
    # a short cap names the capacity, which then suffices
    ixd = gpu.index(s)
    d_src, d_data = to_dev(torch, s), to_dev(torch, np.frombuffer(b"capacity", np.uint8))
    d_dst = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    with pytest.raises(kz.KanziError) as e:
        ixd.write_many_device(d_src, len(s), [BS + 1], [8], d_data, [0], d_dst, 16)
    need = e.value.needed
    assert e.value.code == 12 and need > 16
    keep, nd = ixd.write_many_device(d_src, len(s), [BS + 1], [8], d_data, [0], d_dst, need)
    assert s[:keep].tobytes() + d_dst[:nd].cpu().numpy().tobytes() == st.compress(apply(x, [(BS + 1, b"capacity")]), n).tobytes()
    # an open session
    ix = gpu.index(s)
    r = gpu.stream_reader(batch_blocks=2)
    try:
        with pytest.raises(kz.KanziError) as e:
            ix.write(s, 0, b"x")
        assert e.value.code == 18
    finally:
        r.close()
    # a loaded index naming a chain the GPU path lacks (SRT)
    b = bytearray(gpu.index(s).save())
    b[8:16] = struct.pack("<Q", kz.transform_type("SRT"))
    b[-8:] = struct.pack("<Q", io_.xxh64(bytes(b[:-8])))
    with pytest.raises(kz.KanziError) as e:
        kz.StreamIndex.load(bytes(b), gpu).write(s, 0, b"x")
    assert e.value.code == 14


def ix_start(ix, b):
    """the first payload bit of record b, from the blob"""
    blob = ix.save()
    return struct.unpack_from("<Q", blob, 96 + 8 * b)[0]
