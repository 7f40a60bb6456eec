"""GPU tests of writes into many compressed streams in one call (kz_write_ranges_streams[_device], Context.write_streams /
write_streams_device). Every slot must get what StreamIndex.write_many gives on a second index of the same stream: keep, tail, status and
the saved index, on the level chains -l 0 .. 5 with checksums 0 / 32 / 64, hint, zero-hint and headerless headers, skip blocks off and on,
empty streams, full last blocks, fresh, known-size and loaded indexes, under interleaved write batches. Also: the oracle's compress of the
edited data at -l 3 / -l 5, slot-level failures confined to their slot, call-level refusals that write nothing, the work (launches that do
not grow with the slots, write:* counters equal to the single calls' sums, a one-slot call equal to kz_write_ranges), and slots no write
names. Blocks of 1 KiB and 4 KiB keep the file short."""
import struct

import numpy as np
import pytest

import index_oracle as io_
from test_gpu_write_ranges import LEVELS, MODES, Setup, apply, scenarios, to_dev

pytestmark = pytest.mark.gpu

A = (1 << 64) - 1
BS = 1024


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def make_index(kz, gpu, st, s, kind):
    """fresh (size unknown), known (the last block read once) or loaded (from a saved blob)"""
    ix = gpu.index(s, headerless=st.hl)
    if kind == "known" and ix.info["nblocks"]:
        ix.read(s, ix.info["nblocks"] * st.bs - 1, 1)
    if kind == "loaded":
        ix = kz.StreamIndex.load(ix.save(), gpu)
    return ix


def single(kz, ix, s, writes):
    """what write_many gives: (keep, tail, status)"""
    try:
        keep, tail = ix.write_many(s, writes)
        return keep, tail, 0
    except kz.KanziError as e:
        return len(s), b"", -e.code


def interleave(rng, per_slot):
    """one write list over all slots, each slot's writes in their order"""
    left = [list(w) for w in per_slot]
    out = []
    while any(left):
        s = int(rng.choice([i for i, w in enumerate(left) if w]))
        out.append((s, *left[s].pop(0)))
    return out


def device_layout(torch, streams, caps):
    """streams at 16-byte aligned offsets with 64 bytes behind each, and 16-byte aligned output windows"""
    so, pos = [], 0
    for x in streams:
        so.append(pos)
        pos += (len(x) + 64 + 15) // 16 * 16
    src = np.zeros(max(pos, 16), np.uint8)
    for o, x in zip(so, streams):
        src[o:o + len(x)] = x
    do, pos = [], 0
    for c in caps:
        do.append(pos)
        pos += (int(c) + 15) // 16 * 16
    return to_dev(torch, src), so, do, max(pos, 16)


def run_device(kz, gpu, torch, streams, indexes, writes, caps, guard=0, wrapper=False):
    """kz_write_ranges_streams_device over host lists -> (rc, keep, out_n, status, tails, d_dst, dst_off); wrapper: through
    Context.write_streams_device instead of the raw ABI (rc is then None)"""
    d_src, so, do, total = device_layout(torch, streams, caps)
    bufs = [np.frombuffer(bytes(w[2]), np.uint8) for w in writes]
    data = np.concatenate(bufs) if bufs else np.zeros(0, np.uint8)
    ln = np.array([b.size for b in bufs], np.uint64)
    doff = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64) if len(ln) else np.zeros(0, np.uint64)
    d_data = to_dev(torch, data)
    d_dst = torch.full((total + 64,), guard, dtype=torch.uint8, device="cuda")
    lib = kz.load_library()
    ix = gpu._index_slots(indexes)
    arr = lambda v, t=np.uint64: np.ascontiguousarray(v, t)  # noqa: E731
    so_, sl_, off_, ws_, do_, cap_ = arr(so), arr([len(x) for x in streams]), arr([w[1] for w in writes]), arr([w[0] for w in writes], np.uint32), \
        arr(do), arr(caps)
    keep, out_n, status = np.zeros(len(streams), np.uint64), np.zeros(len(streams), np.uint64), np.zeros(len(streams), np.int32)
    p = lambda a: a.ctypes.data if a.size else None  # noqa: E731
    if wrapper:
        rc = None
        keep, out_n, status = gpu.write_streams_device(d_src, so, [len(x) for x in streams], indexes, [w[0] for w in writes], [w[1] for w in writes],
                                                       ln, d_data, doff, d_dst, do, caps)
    else:
        rc = lib.kz_write_ranges_streams_device(gpu.h, len(streams), __import__("ctypes").addressof(ix), d_src.data_ptr(), p(so_), p(sl_), len(writes), p(ws_),
                                                p(off_), p(ln), d_data.data_ptr(), p(doff), d_dst.data_ptr(), p(do_), p(cap_), p(keep), p(out_n),
                                                p(status))
    host = d_dst.cpu().numpy()
    tails = [host[do[s]: do[s] + int(out_n[s])].tobytes() if not status[s] else b"" for s in range(len(streams))]
    return rc, keep, out_n, status, tails, host, do


def cap_of(kz, st, s, writes):
    ln = [len(w[1]) for w in writes if len(w[1])]
    return len(s) + sum(n // st.bs + 2 for n in ln) * kz.load_library().kz_max_block_output(st.bs) + 16


def build_slots(kz, gpu, synth, rng, skip, bs):
    """(Setup, x, stream, index kind) over every level and mode of this skip setting"""
    slots = []
    for level in range(len(LEVELS)):
        for ck, header, sk in MODES:
            if sk != skip:
                continue
            st = Setup(kz, gpu, LEVELS[level], ck, header, sk, bs)
            for kind, n in (("fresh", int(rng.integers(2 * bs, 5 * bs))), ("known", 3 * bs), ("loaded", int(rng.integers(bs, 4 * bs)))):
                x = np.ascontiguousarray(synth.markov_text(n, seed=int(rng.integers(1 << 20)))[:n], np.uint8)
                slots.append((st, x, st.compress(x, st.hint(x)), kind))
            if level in (0, 5):
                x = np.zeros(0, np.uint8)
                slots.append((st, x, st.compress(x, st.hint(x)), "fresh"))
    return slots


@pytest.mark.parametrize("skip", [False, True])
def test_equivalence(kz, gpu, synth, torch, skip):
    rng = np.random.default_rng(7 + skip)
    slots = build_slots(kz, gpu, synth, rng, skip, BS)
    per = []
    for st, x, s, kind in slots:
        sc = scenarios(rng, len(x), BS)
        pick = rng.choice(len(sc), 2, replace=False)
        per.append(sc[pick[0]] + sc[pick[1]] if len(x) else [(A, b"hello " * 300), (A, b"")])
    writes = interleave(rng, per)
    gpu.set_skip_blocks(skip)
    try:
        ia = [make_index(kz, gpu, st, s, kind) for st, x, s, kind in slots]
        ib = [make_index(kz, gpu, st, s, kind) for st, x, s, kind in slots]
        ic = [make_index(kz, gpu, st, s, kind) for st, x, s, kind in slots]
        keeps, tails, status = gpu.write_streams([s for _, _, s, _ in slots], ia, writes)
        for k, (st, x, s, kind) in enumerate(slots):
            want = single(kz, ib[k], s, per[k])
            assert (keeps[k], tails[k], status[k]) == want, (k, st.tr, st.ck, st.header, kind)
            assert ia[k].save() == ib[k].save()
            assert status[k] == 0
            new = np.concatenate([s[:keeps[k]], np.frombuffer(tails[k], np.uint8)])
            y = apply(x, per[k])
            assert gpu.decompress(new, len(y) + 64, headerless=st.hl).tobytes() == y.tobytes()
        # the device variant gives the same slots
        caps = [cap_of(kz, st, s, per[k]) + 64 for k, (st, x, s, kind) in enumerate(slots)]
        rc, kd, nd, sd, td, _, _ = run_device(kz, gpu, torch, [s for _, _, s, _ in slots], ic, writes, caps)
        assert rc == 0 and list(sd) == status and list(kd) == keeps and td == tails
        assert all(ic[k].save() == ia[k].save() for k in range(len(slots)))
        # and so does Context.write_streams_device, the public wrapper of the same call
        iw = [make_index(kz, gpu, st, s, kind) for st, x, s, kind in slots]
        _, kw, nw, sw, tw, _, _ = run_device(kz, gpu, torch, [s for _, _, s, _ in slots], iw, writes, caps, wrapper=True)
        assert list(sw) == list(sd) and list(kw) == list(kd) and list(nw) == list(nd) and tw == td
        assert all(iw[k].save() == ia[k].save() for k in range(len(slots)))
    finally:
        gpu.set_skip_blocks(False)


@pytest.mark.parametrize("level", [3, 5])
def test_oracle_parity(kz, gpu, oracle, synth, level):
    tr, en = LEVELS[level]
    rng = np.random.default_rng(level)
    xs, ss, per = [], [], []
    for k in range(4):
        n = int(rng.integers(2 * BS, 5 * BS))
        x = np.ascontiguousarray(synth.markov_text(n, seed=20 + k)[:n], np.uint8)
        xs.append(x)
        ss.append(oracle.compress(x, tr, en, block_size=BS, checksum_bits=32, input_size=n))
        per.append([(int(rng.integers(0, n)), b"oracle parity %d " % k * 10), (A, b"appended " * (k + 1) * 20)])
    ix = [gpu.index(s) for s in ss]
    keeps, tails, status = gpu.write_streams(ss, ix, interleave(rng, per))
    for k in range(4):
        assert status[k] == 0
        y = apply(xs[k], per[k])
        want = oracle.compress(y, tr, en, block_size=BS, checksum_bits=32, input_size=len(xs[k]))
        assert ss[k][:keeps[k]].tobytes() + tails[k] == want.tobytes()


def ix_start(ix, b):
    return struct.unpack_from("<Q", ix.save(), 96 + 8 * b)[0]


def test_isolation(kz, gpu, synth, torch):
    st = Setup(kz, gpu, LEVELS[2], 32, "hint", False)
    n = 6 * BS
    streams, xs = [], []
    for k in range(6):
        x = np.ascontiguousarray(synth.markov_text(n, seed=40 + k)[:n], np.uint8)
        xs.append(x)
        streams.append(st.compress(x, n))
    # slot 1: stale (a byte of its stream changed after indexing); slot 2: a loaded index naming SRT; slot 3: a damaged record that must be
    # decoded; slot 4: a short dst_cap; slots 0 and 5 are good
    stale = streams[1].copy()
    stale[3] ^= 1
    b = bytearray(gpu.index(streams[2]).save())
    b[8:16] = struct.pack("<Q", kz.transform_type("SRT"))
    b[-8:] = struct.pack("<Q", io_.xxh64(bytes(b[:-8])))
    bad = streams[3].copy()
    bad[(ix_start(gpu.index(bad), 2) + 200) // 8] ^= 0x10
    srcs = [streams[0], stale, streams[2], bad, streams[4], streams[5]]
    per = [[(2 * BS + 5, b"zz" * 10)] for _ in range(6)]
    writes = interleave(np.random.default_rng(3), per)

    def indexes():
        return [gpu.index(streams[0]), gpu.index(streams[1]), kz.StreamIndex.load(bytes(b), gpu), gpu.index(bad), gpu.index(streams[4]),
                gpu.index(streams[5])]

    ia, ib = indexes(), indexes()
    before = [x.save() for x in ia]
    caps = [cap_of(kz, st, s, p) for s, p in zip(srcs, per)]
    caps[4] = 16
    rc, keep, out_n, status, tails, host, do = run_device(kz, gpu, torch, srcs, ia, writes, caps, guard=0xAB)
    want = [single(kz, ib[k], srcs[k], per[k]) for k in range(6)]
    for k in (1, 2, 3, 4):  # a failed slot's window keeps the guard bytes
        assert (host[do[k]: do[k] + caps[k]] == 0xAB).all(), k
    assert status[0] == 0 and status[1] == -18 and status[2] == -14 and status[3] < 0 and status[4] == -12 and status[5] == 0
    assert rc == -18  # the first failing slot's code
    for k in (1, 2, 3):
        assert want[k][2] == status[k] and ia[k].save() == before[k] and keep[k] == len(srcs[k]) and out_n[k] == 0
    for k in (0, 5):
        assert (keep[k], tails[k], 0) == want[k] and ia[k].save() == ib[k].save()
    assert ia[4].save() == before[4] and out_n[4] > 16
    # the short-cap slot alone, with the capacity it named
    caps2 = [0, 0, 0, 0, int(out_n[4]), 0]
    rc, keep2, out2, st2, tails2, _, _ = run_device(kz, gpu, torch, srcs, [None, None, None, None, ia[4], None],
                                                    [w for w in writes if w[0] == 4], caps2)
    assert rc == 0 and st2[4] == 0 and (keep2[4], tails2[4], 0) == want[4] and ia[4].save() == ib[4].save()
    # the host variant retries it itself
    ic = indexes()
    keeps, tails, status = gpu.write_streams(srcs, ic, writes)
    assert status == [0, -18, -14, int(want[3][2]), 0, 0] and tails[4] == want[4][1]


def test_call_level_refusals(kz, gpu, synth, torch):
    st = Setup(kz, gpu, LEVELS[1], 0, "hint", False)
    n = 3 * BS
    streams = [st.compress(np.ascontiguousarray(synth.markov_text(n, seed=60 + k)[:n], np.uint8), n) for k in range(3)]
    per = [[(100, b"abc")], [(A, b"def" * 50)], [(BS + 1, b"g" * 10)]]
    writes = interleave(np.random.default_rng(1), per)
    caps = [cap_of(kz, st, s, p) for s, p in zip(streams, per)]

    def refused(indexes, ws, caps=caps, srcs=streams):
        blobs = [x.save() for x in indexes if x is not None]
        rc, keep, out_n, status, _, host, _ = run_device(kz, gpu, torch, srcs, indexes, ws, caps, guard=0xAB)
        assert rc < 0 and (status == rc).all() and (out_n == 0).all()
        assert (host == 0xAB).all()  # nothing written, guards included
        assert [x.save() for x in indexes if x is not None] == blobs
        return rc

    ix = [gpu.index(s) for s in streams]
    assert refused(ix, writes + [(3, 0, b"x")]) == -18                 # w_stream past nstreams
    assert refused([ix[0], ix[0], ix[2]], writes) == -18               # one index in two written slots
    # device misalignment: a stream at an offset that is not a multiple of 16
    lib = kz.load_library()
    d_src = to_dev(torch, np.concatenate([np.zeros(8, np.uint8), streams[0]]))
    d_data = to_dev(torch, np.frombuffer(b"abc", np.uint8))
    d_dst = torch.full((4096,), 0xAB, dtype=torch.uint8, device="cuda")
    keep, out_n, status = np.zeros(1, np.uint64), np.zeros(1, np.uint64), np.zeros(1, np.int32)
    u = lambda v, t=np.uint64: np.array(v, t)  # noqa: E731
    args = [u([8]), u([len(streams[0])]), u([0], np.uint32), u([100]), u([3]), u([0]), u([0]), u([4000])]
    slots = gpu._index_slots([ix[0]])
    blob = ix[0].save()
    rc = lib.kz_write_ranges_streams_device(gpu.h, 1, __import__("ctypes").addressof(slots), d_src.data_ptr(), args[0].ctypes.data, args[1].ctypes.data,
                                            1, args[2].ctypes.data, args[3].ctypes.data, args[4].ctypes.data, d_data.data_ptr(), args[5].ctypes.data,
                                            d_dst.data_ptr(), args[6].ctypes.data, args[7].ctypes.data, keep.ctypes.data, out_n.ctypes.data,
                                            status.ctypes.data)
    assert rc == -18 and status[0] == -18 and (d_dst.cpu().numpy() == 0xAB).all() and ix[0].save() == blob
    # overlapping output windows: the run_device layout with slot 1's window moved onto slot 0's

    def overlapping():
        d_srcx, so, do, total = device_layout(torch, streams, caps)
        do[1] = do[0] + 16
        dd = torch.full((total + 64,), 0xAB, dtype=torch.uint8, device="cuda")
        bufs = [np.frombuffer(w[2], np.uint8) for w in writes]
        data = np.concatenate(bufs)
        ln = u([b.size for b in bufs])
        doff = np.concatenate([[0], np.cumsum(ln)[:-1]]).astype(np.uint64)
        dat = to_dev(torch, data)
        k, o, s_ = np.zeros(3, np.uint64), np.zeros(3, np.uint64), np.zeros(3, np.int32)
        a = [u(so), u([len(x) for x in streams]), u([w[0] for w in writes], np.uint32), u([w[1] for w in writes]), ln, doff, u(do), u(caps)]
        sl = gpu._index_slots(ix)
        blobs = [x.save() for x in ix]
        rc = lib.kz_write_ranges_streams_device(gpu.h, 3, __import__("ctypes").addressof(sl), d_srcx.data_ptr(), a[0].ctypes.data, a[1].ctypes.data,
                                                len(writes), a[2].ctypes.data, a[3].ctypes.data, a[4].ctypes.data, dat.data_ptr(), a[5].ctypes.data,
                                                dd.data_ptr(), a[6].ctypes.data, a[7].ctypes.data, k.ctypes.data, o.ctypes.data, s_.ctypes.data)
        assert rc == -18 and (s_ == -18).all() and (dd.cpu().numpy() == 0xAB).all() and [x.save() for x in ix] == blobs

    overlapping()
    # an open session, both variants
    r = gpu.stream_reader(batch_blocks=2)
    try:
        assert refused(ix, writes) == -18
        blobs = [x.save() for x in ix]
        keeps, tails, status = gpu.write_streams(streams, ix, writes)
        assert status == [-18] * 3 and tails == [b""] * 3 and [x.save() for x in ix] == blobs
    finally:
        r.close()


def test_work(kz, gpu, synth, torch):
    # a chain whose stages launch once per batch: transforms that run in sub-batches of a fixed number of blocks (TEXT, UTF, LZ, ...)
    # add launches per sub-batch on every batched path
    st = Setup(kz, gpu, ("NONE", "HUFFMAN"), 32, "hint", False, bs=4096)
    n = 3 * 4096 - 500
    x = np.ascontiguousarray(synth.markov_text(n, seed=5)[:n], np.uint8)
    s = st.compress(x, n)
    slot_writes = [(4096 + 10, b"w" * 100), (A, b"a" * 700)]  # a fresh index must learn its size for the append

    def launches(copies, device):
        ix = [gpu.index(s) for _ in range(copies)]
        writes = [(k, o, d) for k in range(copies) for o, d in slot_writes]
        gpu.launch_count(reset=True)
        if device:
            caps = [cap_of(kz, st, s, slot_writes)] * copies
            rc, *_ = run_device(kz, gpu, torch, [s] * copies, ix, writes, caps)
            assert rc == 0
        else:
            assert gpu.write_streams([s] * copies, ix, writes)[2] == [0] * copies
        return gpu.launch_count()

    for device in (False, True):
        assert launches(3, device) == launches(300, device)
    # write:decoded and write:encoded equal the sums of the single calls, slots that learn their size included

    def counters(fn):
        gpu.profile(True)
        gpu.profile_reset()
        try:
            fn()
            return gpu.stage_bytes("write:decoded")[1:], gpu.stage_bytes("write:encoded")[1:]
        finally:
            gpu.profile(False)

    kinds = ["fresh", "known", "loaded", "fresh"]
    per = [slot_writes, [(100, b"q" * 5000)], [(A, b"z" * 10)], [(8000, b"m" * 3)]]
    sums = [0, 0, 0, 0]
    for k, kind in enumerate(kinds):
        ix = make_index(kz, gpu, st, s, kind)
        (db, dn), (eb, en) = counters(lambda: ix.write_many(s, per[k]))
        sums = [sums[0] + db, sums[1] + dn, sums[2] + eb, sums[3] + en]
    ix = [make_index(kz, gpu, st, s, kind) for kind in kinds]
    (db, dn), (eb, en) = counters(lambda: gpu.write_streams([s] * 4, ix, interleave(np.random.default_rng(2), per)))
    assert [db, dn, eb, en] == sums and sums[0] > 0
    # a one-slot call makes the launches and write:* counters of kz_write_ranges[_device]
    for kind in ("fresh", "known"):
        a, b2 = make_index(kz, gpu, st, s, kind), make_index(kz, gpu, st, s, kind)
        gpu.launch_count(reset=True)
        ca = counters(lambda: a.write_many(s, slot_writes))
        la = gpu.launch_count(reset=True)
        cb = counters(lambda: gpu.write_streams([s], [b2], [(0, o, d) for o, d in slot_writes]))
        lb = gpu.launch_count(reset=True)
        assert (la, ca) == (lb, cb) and a.save() == b2.save()
        a, b2 = make_index(kz, gpu, st, s, kind), make_index(kz, gpu, st, s, kind)
        d_src = to_dev(torch, s)
        data = np.frombuffer(b"".join(d for _, d in slot_writes), np.uint8)
        d_data = to_dev(torch, data)
        cap = cap_of(kz, st, s, slot_writes)
        d_dst = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        ln = [len(d) for _, d in slot_writes]
        gpu.launch_count(reset=True)
        ca = counters(lambda: a.write_many_device(d_src, len(s), [o for o, _ in slot_writes], ln, d_data, [0, ln[0]], d_dst, cap))
        la = gpu.launch_count(reset=True)
        cb = counters(lambda: run_device(kz, gpu, torch, [s], [b2], [(0, o, d) for o, d in slot_writes], [cap]))
        lb = gpu.launch_count(reset=True)
        assert (la, ca) == (lb, cb) and a.save() == b2.save()


def test_unnamed_slots(kz, gpu, synth, torch):
    st = Setup(kz, gpu, LEVELS[0], 0, "hint", False)
    n = 2 * BS + 10
    x = np.ascontiguousarray(synth.markov_text(n, seed=8)[:n], np.uint8)
    s = st.compress(x, n)
    garbage = np.random.default_rng(0).integers(0, 256, 500, dtype=np.uint8)
    ix = gpu.index(s)
    other = gpu.index(s)
    blob = other.save()
    # slot 0: garbage with no index; slot 1: written; slot 2: only a zero-length write, with an index
    keeps, tails, status = gpu.write_streams([garbage, s, s], [None, ix, other], [(1, 5, b"hi"), (2, 7, b""), (0, 0, b"")])
    assert status == [0, 0, 0] and keeps[0] == len(garbage) and tails[0] == b"" and keeps[2] == len(s) and tails[2] == b""
    assert other.save() == blob
    assert s[:keeps[1]].tobytes() + tails[1] == st.compress(apply(x, [(5, b"hi")]), n).tobytes()
    rc, keep, out_n, st_, tails_d, _, _ = run_device(kz, gpu, torch, [garbage, s, s], [None, gpu.index(s), other], [(1, 5, b"hi"), (2, 7, b"")],
                                                    [0, cap_of(kz, st, s, [(5, b"hi")]), 0])
    assert rc == 0 and list(st_) == [0, 0, 0] and keep[0] == len(garbage) and out_n[0] == 0 and out_n[2] == 0 and tails_d[1] == tails[1]
    # a call that names no slot checks no buffer: misaligned device buffers and offsets are not read, so not refused
    d_src = to_dev(torch, np.concatenate([np.zeros(8, np.uint8), s]))
    d_dst = torch.full((256,), 0xAB, dtype=torch.uint8, device="cuda")
    keep, out_n, st_ = gpu.write_streams_device(d_src.data_ptr() + 1, [8], [len(s)], [None], [0], [5], [0], d_src.data_ptr(), [0],
                                                d_dst.data_ptr() + 1, [3], [100])
    assert list(st_) == [0] and list(keep) == [len(s)] and list(out_n) == [0] and (d_dst.cpu().numpy() == 0xAB).all()


@pytest.mark.parametrize("level", [0, 2])
def test_learned_last_block_under_a_write(kz, gpu, synth, level):
    """An index that does not know the size decodes the old last block first; a write into that block must win over its old bytes, in
    kz_write_ranges as in a many-slot call (the old bytes and the write once raced in one copy launch)."""
    st = Setup(kz, gpu, LEVELS[level], 32, "zero", False)
    n = 2028
    x = np.ascontiguousarray(synth.markov_text(n, seed=70 + level)[:n], np.uint8)
    s = st.compress(x, 0)
    for writes in ([(974, b"W" * 200), (2148, b"V" * 300)], [(1024 + 5, b"U" * 900), (2100, b"T" * 10)]):
        y = apply(x, writes)
        want = st.compress(y, 0).tobytes()
        ix = gpu.index(s)
        assert ix.size == -1
        keep, tail = ix.write_many(s, writes)
        assert s[:keep].tobytes() + tail == want
        keeps, tails, status = gpu.write_streams([s, s], [gpu.index(s), gpu.index(s)], [(0, o, d) for o, d in writes] + [(1, o, d) for o, d in writes])
        assert status == [0, 0] and all(s[:k].tobytes() + t == want for k, t in zip(keeps, tails))
