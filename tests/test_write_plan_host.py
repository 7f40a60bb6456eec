"""CPU check of the write plan (kanzi-go_b200/csrc/kz_write_plan.h) under g++ with ASan / UBSan: plan_writes and splice_records against a
brute-force Python model that paints every decoded byte with its source (the old data, a write, or a zero gap). Random batches of
overlapping, repeated, zero-length and past-the-end writes, KZ_WRITE_APPEND chains, empty streams, full and partial last blocks, and a
size known or unknown: the re-encoded and decoded blocks, the pieces that tile every re-encoded block exactly once, the cut bit, the
segments behind it, the passes within the budget, and the record table of the new stream. With the size unknown, a plan that does not
ask for it must be what every possible size gives."""
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "write_plan_host.cpp")
HDRS = [os.path.join(ROOT, "kanzi-go_b200", "csrc", h) for h in ("kz_write_plan.h", "kz_read_plan.h", "kz_stream_plan.h")]
EXE = os.path.join(ROOT, "tests", "host", "_build", "write_plan_host")
APPEND = (1 << 64) - 1
OK, NEED_SIZE, TOO_LARGE = 0, 1, 2
OLD, WRITE, ZERO = 0, 1, 2
CARRY, NEW, MOVED, END = 0, 1, 2, 3


@pytest.fixture(scope="module")
def exe():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or max(os.path.getmtime(f) for f in [SRC] + HDRS) > os.path.getmtime(EXE):
        r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-o", EXE, SRC],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def read_block_cost(bs):
    slot = (bs + max(512, bs >> 4) + 64 + 15) & ~15
    return 3 * slot


class Stream:
    """A synthetic index: nb records of random prefix and payload lengths behind a header of hb bits."""

    def __init__(self, rng, nb, bs, size, hb):
        self.nb, self.bs, self.size, self.hb = nb, bs, size, hb
        self.start, self.bits = [], []
        pos = hb
        for _ in range(nb):
            self.start.append(pos + rng.randint(8, 39))
            self.bits.append(rng.randint(1, 300))
            pos = self.start[-1] + self.bits[-1]

    def prefix_bit(self, b):
        return self.hb if b == 0 else self.start[b - 1] + self.bits[b - 1]


def run(exe, cases):
    lines = []
    for st, writes, enc_cost, budget in cases:
        head = [st.nb, st.bs, st.size, st.hb, len(writes), enc_cost, budget]
        lines.append(" ".join(map(str, head + st.start + st.bits + [w[0] for w in writes] + [w[1] for w in writes])))
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return [list(map(int, ln.split())) for ln in r.stdout.splitlines()]


def parse(v):
    status, new_size, known, nblocks, n, cut, npasses, nsegs, npieces = v[:9]
    i = 9
    p = {"status": status, "new_size": new_size, "known": known, "nblocks": nblocks, "cut": cut}

    def take(k):
        nonlocal i
        out = v[i:i + k]
        i += k
        return out

    p["enc"], p["enc_len"], p["decode"] = take(n), take(n), take(n)
    p["piece_of"] = take(n + 1) if n else []
    p["pieces"] = [tuple(take(5)) for _ in range(npieces)]
    p["first"] = take(npasses + 1) if n else []
    p["segs"] = [tuple(take(5)) for _ in range(nsegs)]
    if status == OK:
        p["total"], p["stream_bytes"], p["size"] = take(3)
    p["rest"] = v[i:]
    return p


def paint(st, s, writes):
    """The source of every byte after the writes, the old size being s: ("O", pos), ("W", i, k) or ("Z",)."""
    data = [("O", p) for p in range(s)]
    for i, (o, n) in enumerate(writes):
        if n == 0:
            continue
        o = len(data) if o == APPEND else o
        if o > len(data):
            data += [("Z",)] * (o - len(data))
        if o + n > len(data):
            data += [None] * (o + n - len(data))
        for k in range(n):
            data[o + k] = ("W", i, k)
    return data


def model_layout(st, s, writes):
    data = paint(st, s, writes)
    bs = st.bs
    nblocks = (len(data) + bs - 1) // bs
    enc, enc_len, decode, pieces = [], [], [], []
    for b in range(nblocks):
        blk = data[b * bs:(b + 1) * bs]
        if all(t[0] == "O" for t in blk) and b < st.nb and (b + 1 < st.nb or len(blk) == s - b * bs):
            continue
        enc.append(b)
        enc_len.append(len(blk))
        decode.append(int(any(t[0] == "O" for t in blk)))
        ps = []
        for at, t in enumerate(blk):
            kind = {"O": OLD, "W": WRITE, "Z": ZERO}[t[0]]
            w, frm = (t[1], t[2]) if kind == WRITE else (0, 0)
            if ps and ps[-1][0] == kind and ps[-1][3] == w and ps[-1][1] + ps[-1][2] == at and (kind != WRITE or ps[-1][4] + ps[-1][2] == frm):
                ps[-1][2] += 1
            else:
                ps.append([kind, at, 1, w, frm])
        pieces.append([tuple(x) for x in ps])
    return len(data), nblocks, enc, enc_len, decode, pieces


def needs_size(st, writes):
    if st.size >= 0:
        return False
    lo, hi = (st.nb - 1) * st.bs, st.nb * st.bs
    reach, ivs = 0, []
    for o, n in writes:
        if n == 0:
            continue
        if o == APPEND and reach < hi:
            return True
        o = max(hi, reach) if o == APPEND else o
        reach = max(reach, o + n)
        ivs.append((o, o + n))
    if reach <= lo:
        return False
    cov = set()
    for a, e in ivs:
        cov.update(range(max(a, lo), min(e, hi)))
    return len(cov) < hi - lo


def check(st, writes, enc_cost, budget, p):
    bs, nb = st.bs, st.nb
    if needs_size(st, writes):
        assert p["status"] == NEED_SIZE
        return
    assert p["status"] == OK
    lo, hi = (nb - 1) * bs, nb * bs
    known = st.size >= 0
    if known:
        sizes = [st.size]
    else:
        sizes = list(range(lo + 1, hi + 1))
    results = [model_layout(st, s, writes) for s in sizes]
    reach = max([0] + [(o + n) for o, n in writes if n and o != APPEND])
    size_known = known or reach > lo
    assert p["known"] == int(size_known)
    for new_size, nblocks, enc, enc_len, decode, pieces in results:
        if size_known:
            assert p["new_size"] == new_size and p["nblocks"] == nblocks
        else:
            assert p["nblocks"] == nb
        assert p["enc"] == enc and p["enc_len"] == enc_len and p["decode"] == decode
        got = [p["pieces"][p["piece_of"][j]:p["piece_of"][j + 1]] for j in range(len(enc))]
        assert got == pieces
    enc = p["enc"]
    if not enc:
        assert p["segs"] == [] and p["cut"] == 0
        return
    # pieces tile each block: ascending, adjacent, summing to its length
    for j in range(len(enc)):
        ps = p["pieces"][p["piece_of"][j]:p["piece_of"][j + 1]]
        at = 0
        for kind, a, n, w, frm in ps:
            assert a == at and n >= 1
            at += n
        assert at == p["enc_len"][j]
    # the cut and the segments
    k0 = min(enc[0], nb)
    assert p["cut"] == st.prefix_bit(k0)
    segs, j, b = [], 0, enc[0]
    if p["cut"] % 8:
        segs.append((CARRY, 0, 0, p["cut"] & ~7, p["cut"] % 8))
    while b < p["nblocks"]:
        if j < len(enc) and enc[j] == b:
            e = j
            while e + 1 < len(enc) and enc[e + 1] == enc[e] + 1:
                e += 1
            segs.append((NEW, j, e - j + 1, 0, 0))
            b, j = enc[e] + 1, e + 1
        else:
            e = min(enc[j], nb) if j < len(enc) else nb
            segs.append((MOVED, b, e - b, st.prefix_bit(b), st.prefix_bit(e) - st.prefix_bit(b)))
            b = e
    segs.append((END, 0, 0, 0, 0))
    assert p["segs"] == segs
    # passes: consecutive, within the budget unless one block
    cost = read_block_cost(bs) + enc_cost
    per = max(1, budget // cost)
    assert p["first"] == list(range(0, len(enc), per)) + [len(enc)]
    # the spliced record table: old records before the cut stay, then every segment in order
    starts, bits = list(st.start[:k0]), list(st.bits[:k0])
    pos = p["cut"]
    for kind, first, count, bit, nbits in segs:
        if kind == NEW:
            for jj in range(first, first + count):
                pre, pay = 9 + jj % 4, 64 + 13 * jj
                starts.append(pos + pre)
                bits.append(pay)
                pos += pre + pay
        elif kind == MOVED:
            for bb in range(first, first + count):
                starts.append(st.start[bb] - bit + pos)
                bits.append(st.bits[bb])
            pos += nbits
        elif kind == END:
            pos += 8
    nbl = p["nblocks"]
    assert p["total"] == pos and p["stream_bytes"] == (pos + 7) // 8
    assert p["size"] == (p["new_size"] if size_known else st.size)
    rest = p["rest"]
    assert rest[:nbl] == starts and rest[nbl:2 * nbl] == bits and len(rest) == 2 * nbl


def parse_all(outs):
    return [parse(v) for v in outs]


def random_case(rng):
    bs = rng.choice([4, 8, 16])
    nb = rng.choice([0, 0, 1, 2, 3, 5])
    hb = rng.choice([0, 160, 176, 208, 3])
    if nb == 0:
        size = 0
    elif rng.random() < 0.4:
        size = -1
    else:
        size = rng.randint((nb - 1) * bs + 1, nb * bs)
    st = Stream(rng, nb, bs, size, hb)
    total = nb * bs + 2 * bs
    writes = []
    for _ in range(rng.randint(0, 7)):
        r = rng.random()
        if r < 0.15:
            writes.append((APPEND, rng.randint(0, 2 * bs)))
        elif r < 0.25:
            writes.append((rng.randint(0, total), 0))
        elif r < 0.35:
            writes.append((rng.randint(0, max(0, nb - 1)) * bs, bs))  # a whole block
        else:
            o = rng.randint(0, total)
            writes.append((o, rng.randint(1, 2 * bs)))
    if writes and rng.random() < 0.2:
        writes.append(writes[rng.randrange(len(writes))])  # a repeated write
    enc_cost = rng.choice([0, 1000, 50000])
    budget = rng.choice([1 << 30, 1, 20000, 60000])
    return st, writes, enc_cost, budget


def test_random_batches(exe):
    rng = random.Random(1234)
    cases = [random_case(rng) for _ in range(3000)]
    for case, p in zip(cases, parse_all(run(exe, cases))):
        check(*case, p)


def test_named_cases(exe):
    rng = random.Random(7)
    bs = 16
    full = Stream(rng, 3, bs, 48, 160)
    part = Stream(rng, 3, bs, 40, 160)
    unknown = Stream(rng, 3, bs, -1, 160)
    empty = Stream(rng, 0, bs, 0, 160)
    hl_empty = Stream(rng, 0, bs, 0, 0)
    cases = [
        (full, [(20, 4)], 0, 1 << 30),                    # inside one block
        (full, [(10, 20)], 0, 1 << 30),                   # across two blocks
        (full, [(16, 16)], 0, 1 << 30),                   # a whole block: nothing decoded
        (full, [(APPEND, 5)], 0, 1 << 30),                # append behind a full last block: nothing decoded, cut at the end marker
        (part, [(APPEND, 5)], 0, 1 << 30),                # append into a partial last block
        (part, [(APPEND, 5), (APPEND, 30), (APPEND, 1)], 0, 1 << 30),  # an append chain
        (part, [(100, 3)], 0, 1 << 30),                   # a gap of zeros over several blocks
        (full, [(5, 0), (200, 0)], 0, 1 << 30),           # zero-length writes change nothing
        (full, [], 0, 1 << 30),
        (unknown, [(3, 4)], 0, 1 << 30),                  # before the last block: the size stays unknown
        (unknown, [(APPEND, 4)], 0, 1 << 30),             # needs the size
        (unknown, [(33, 2)], 0, 1 << 30),                 # into the last block, partly: needs the size
        (unknown, [(32, 16), (APPEND, 4)], 0, 1 << 30),   # covers the last block, then appends: no size needed
        (unknown, [(32, 10), (40, 20)], 0, 1 << 30),      # covered by two writes together
        (empty, [(APPEND, 40)], 0, 1 << 30),              # into an empty stream
        (empty, [(7, 3)], 0, 1 << 30),                    # into an empty stream behind a gap
        (hl_empty, [(0, 17)], 0, 1 << 30),
        (full, [(0, 48), (1, 1), (0, 48)], 0, 1 << 30),   # later writes win
        (full, [(0, 100)], 10**9, 1),                     # one block per pass
        (full, [(0, 100)], 0, 3 * read_block_cost(bs)),   # three blocks per pass
    ]
    outs = parse_all(run(exe, cases))
    for case, p in zip(cases, outs):
        check(*case, p)
    assert outs[2]["decode"] == [0] and outs[3]["decode"] == [0] and outs[3]["cut"] == full.prefix_bit(3)
    assert outs[0]["decode"] == [1] and outs[0]["enc"] == [1]
    assert outs[7]["enc"] == [] and outs[8]["enc"] == []
    assert outs[9]["known"] == 0 and outs[9]["size"] == -1
    assert outs[10]["status"] == NEED_SIZE and outs[11]["status"] == NEED_SIZE
    assert outs[12]["status"] == OK and outs[12]["new_size"] == 52 and outs[12]["decode"] == [0, 0]
    assert outs[13]["status"] == OK and outs[13]["new_size"] == 60


def test_too_large(exe):
    rng = random.Random(3)
    st = Stream(rng, 2, 1024, 2048, 160)
    cases = [
        (st, [(1 << 62, 1)], 0, 1 << 30),                # past 2^62
        (st, [((1 << 64) - 2, 1)], 0, 1 << 30),          # offset + length overflows
        (st, [(APPEND, (1 << 64) - 100)], 0, 1 << 30),
    ]
    for p in parse_all(run(exe, cases)):
        assert p["status"] == TOO_LARGE
