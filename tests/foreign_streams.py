"""TEST INFRASTRUCTURE ONLY. Stage streams that no encoder here writes, for the data-parallel inverses of LZ / LZX (kz_lz_inv.cu), ZRLT
(kz_zrlt.cu), MM (kz_fsd.cu), PACK / DNA (kz_alias.cu) and TEXT (kz_text_par.cu). A kanzi stream may come from another writer (kanzi C++
or Java, another kanzi-go version, other parse heuristics), so the inverses must decode every stream the reference decodes and reject
every stream it rejects. The oracle's inverse says which is which; these generators only make the shapes where a scan-based kernel is
likely to part from the reference's one-pass loop.

Every case is (name, stream, label): label "shaped" marks streams an encoder could have written (the oracle must accept them at a
generous cap), "odd" marks streams the parallel LZ parse must hand to its serial kernel, None marks anything else. Everything is
seeded: the same lists every run.
"""
import importlib

import numpy as np

synth = importlib.import_module("kanzi-go_b200.synth")

MIB = 1 << 20
ZTILE = 8192  # bytes per tile of zrlt_inverse_kernel
T_LZ, T_LZX, T_ZRLT, T_MM, T_PACK, T_DNA, T_TEXT = 3, 16, 6, 15, 18, 19, 10
TRANSFORMS = {"LZ": T_LZ, "LZX": T_LZX, "ZRLT": T_ZRLT, "MM": T_MM, "PACK": T_PACK, "DNA": T_DNA, "TEXT": T_TEXT}


def _u8(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint8))


def _cat(*parts):
    return _u8(np.concatenate([_u8(p) for p in parts])) if parts else np.zeros(0, np.uint8)


# ---- LZ / LZX: a writer of the v6 layout LZXCodec.inverseV6 reads (LZCodec.go:621-778) ---------------------------------------------

def emit_length(x):
    """emitLengthLZ (LZCodec.go:193-213): 1, 3 or 4 bytes"""
    if x < 254:
        return [x]
    if x < 65536 + 254:
        x -= 254
        return [254, x >> 8, x & 255]
    x -= 255
    assert x < 1 << 24
    return [255, (x >> 16) & 255, (x >> 8) & 255, x & 255]


def lz_stream(items, min_match=4, wide=False):
    """items: [(literals, match)], match None (a token with literals only) or (kind, m_len, dist, nb): kind "d" writes dist in nb bytes
    (1, 2 or 3, whatever its value), "r0" / "r1" reuse a repeat distance (dist and nb ignored). -> the stream: the 13-byte head (token,
    distance and length section offsets, flags: bit 0 = 24-bit distances, bits 1..3 = min_match - 2), then the literal, token, distance
    and match-length sections."""
    lit, tok, dst, mln = [], [], [], []
    for literals, match in items:
        literals = _u8(literals)
        L = len(literals)
        if L >= 7:
            lit.append(_u8(emit_length(L - 7)))
            code = 7
        else:
            code = L
        lit.append(literals)
        t = code << 5
        if match is not None:
            kind, m_len, dist, nb = match
            ml = m_len - min_match
            assert ml >= 0
            if kind == "d":
                t |= {1: 0x08, 2: 0x10, 3: 0x18}[nb]
                dst.extend([(dist >> (8 * (nb - 1 - i))) & 255 for i in range(nb)])
                if ml >= 7:
                    mln.extend(emit_length(ml - 7))
                    ml = 7
            else:
                t |= 0x04 if kind == "r1" else 0
                if ml >= 3:
                    mln.extend(emit_length(ml - 3))
                    ml = 3
            t |= ml
        tok.append(t)
    lit = _cat(*lit) if lit else np.zeros(0, np.uint8)
    head = np.zeros(13, np.uint8)
    head[0:4] = np.frombuffer(np.uint32(13 + len(lit)).tobytes(), np.uint8)
    head[4:8] = np.frombuffer(np.uint32(len(tok)).tobytes(), np.uint8)
    head[8:12] = np.frombuffer(np.uint32(len(dst)).tobytes(), np.uint8)
    head[12] = (1 if wide else 0) | ((min_match - 2) << 1)
    return _cat(head, lit, _u8(tok), _u8(dst), _u8(mln))


def _nb(dist):
    return 1 if dist < 256 else (2 if dist < 65536 else 3)


def random_parse(rng, ntok, min_match=4, wide=False, final=16, rep_share=0.4, forced_nb=None, long_every=0):
    """a valid parse of ntok tokens: literal runs of 0 .. 300 bytes (the first and last ones non-empty), explicit distances inside the
    output (written in forced_nb bytes when given), rep0 / rep1 tokens once two distances exist, match lengths min_match .. +300; the
    last token carries `final` literals only. long_every > 0: every such token gets a match with the 4-byte length extension."""
    max_dist = (1 << 24) - 2 if wide else (1 << 16) - 2
    items, out, reps = [], 0, []
    for k in range(ntok - 1):
        r = rng.random()
        L = int(rng.integers(1, 7)) if r < 0.4 else (0 if r < 0.7 else int(rng.integers(7, 300)))
        if k == 0:
            L = max(L, 1)
        out += L
        m_len = min_match + (int(rng.integers(0, 10)) if rng.random() < 0.8 else int(rng.integers(10, 300)))
        if long_every and k % long_every == long_every - 1:
            m_len = min_match + 65790 + int(rng.integers(0, 2000))
        if len(reps) >= 2 and rng.random() < rep_share:
            kind = "r0" if rng.random() < 0.5 else "r1"
            match = (kind, m_len, 0, 0)
            d = reps[-1] if kind == "r0" else reps[-2]
            reps.append(d)
        else:
            d = int(rng.integers(1, min(out, max_dist, (1 << 8 * forced_nb) - 1 if forced_nb else max_dist) + 1))
            match = ("d", m_len, d, forced_nb or _nb(d))
            reps.append(d)
        items.append((rng.integers(0, 256, L), match))
        out += m_len
    items.append((rng.integers(0, 256, final), None))
    return items


def lz_cases():
    """[(name, stream, label)] for T_LZ / T_LZX (the inverses are the same)"""
    rng = np.random.default_rng(1001)
    out = []

    def add(name, items, label, **kw):
        out.append((name, lz_stream(items, **kw), label))

    for mm in range(2, 10):
        for wide in (False, True):
            add("minmatch%d_wide%d" % (mm, wide), random_parse(rng, 300, min_match=mm, wide=wide), "shaped", min_match=mm, wide=wide)
    for nb in (1, 2, 3):
        add("dist_in_%d_bytes" % nb, random_parse(rng, 400, forced_nb=nb), "shaped")
    big = rng.integers(0, 256, 70000)
    for d, label in ((65534, "shaped"), (65535, "odd")):  # MAX_DISTANCE1 = 65534 under the 16-bit flag
        add("dist%d_16bit" % d, [(big, ("d", 20, d, 3)), (rng.integers(0, 256, 20), None)], label)
    add("dist65535_24bit", [(big, ("d", 20, 65535, 3)), (rng.integers(0, 256, 20), None)], "shaped", wide=True)
    add("reps_mixed_2000", random_parse(rng, 2000, rep_share=0.8), "shaped")
    for d in range(1, 17):  # overlapping copies with the 4-byte match extension
        add("overlap_dist%d" % d, [(rng.integers(0, 256, d), ("d", 4 + 65790 + 7 * d, d, 1)), (rng.integers(0, 256, 16), None)], "shaped")
    add("run_1mib_dist1", [(rng.integers(0, 256, 1), ("d", MIB, 1, 1)), (rng.integers(0, 256, 16), None)], "shaped")
    add("long_matches_every_3rd", random_parse(rng, 200, long_every=3), "shaped")
    for L in (6, 7, 260, 261, 65796, 65797, (1 << 24) + 100):
        add("literals%d" % L, [(rng.integers(0, 256, L), ("d", 8, 1, 1)), (rng.integers(0, 256, 16), None)], "shaped")
    ext = [(rng.integers(0, 256, 300 + k), ("d", 4 + 7 + 300 + k, 1 + k, 1)) for k in range(100)]  # > 32 extensions in a round
    add("extended_100", ext + [(rng.integers(0, 256, 16), None)], "shaped")
    for ntok in (1, 31, 32, 33, 1000, 5000):
        add("tokens%d" % ntok, random_parse(rng, ntok), "shaped")
    add("tokens60000", random_parse(rng, 60000, final=5000), "shaped")
    # the shapes the parallel parse hands to the serial kernel
    # final literal runs of 1, 13 and 14 bytes behind runs of 3 and 30 (the 30 carries a length byte, which moves the break)
    for first in (3, 30):
        for final in (1, 13, 14):
            add("final_literals_%d_after_%d" % (final, first), [(rng.integers(0, 256, first), ("d", 6, 1, 1)), (rng.integers(0, 256, final), None)],
                None)
    add("lit_hits_src_end_early", [(rng.integers(0, 256, 3), ("d", 6, 1, 1)), (rng.integers(0, 256, 5), ("d", 6, 1, 1)),
                                   (rng.integers(0, 256, 9), None)], "odd")
    add("last_token_no_literals", [(rng.integers(0, 256, 30), ("d", 6, 1, 1)), (np.zeros(0), ("d", 6, 2, 1))], "odd")
    # the break at the only literal run after the first match, then two more tokens that the reference never reads
    add("tokens_left_over", [(rng.integers(0, 256, 40), ("d", 6, 1, 1)), (rng.integers(0, 256, 20), None), (np.zeros(0), ("d", 6, 1, 1)),
                             (np.zeros(0), ("d", 6, 1, 1))], "odd")
    add("dist0", [(rng.integers(0, 256, 30), ("d", 6, 0, 1)), (rng.integers(0, 256, 16), None)], "odd")
    add("dist_past_start", [(rng.integers(0, 256, 30), ("d", 6, 31, 1)), (rng.integers(0, 256, 16), None)], "odd")
    add("rep_before_any_distance", [(rng.integers(0, 256, 30), ("r0", 6, 0, 0)), (rng.integers(0, 256, 16), None)], "odd")
    items = random_parse(rng, 50)
    for k in range(1, 4):  # the last run ends k bytes before the token section: src_idx != tk_idx at the end
        t = lz_stream(items[:-1] + [(np.zeros(20 - k), None)])
        tk = int(np.frombuffer(t[0:4].tobytes(), np.uint32)[0])
        t = _cat(t[:tk], np.zeros(k), t[tk:])
        t[0:4] = np.frombuffer(np.uint32(tk + k).tobytes(), np.uint8)
        out.append(("unused_literal_bytes_%d" % k, t, "odd"))
    base = lz_stream(random_parse(rng, 60))
    for k, (a, b, c, label) in enumerate(((5, 0, 0, None), (0, 1 << 20, 0, "odd"), (0, 0, 1 << 20, "odd"), (len(base), 0, 0, "odd"),
                                          (0xFFFFFFF0, 0, 0, "odd"), (0, 0, -1, None), (0, -1, 0, None))):
        s = base.copy()  # sections that overlap or point past the end
        v = np.frombuffer(s[0:12].tobytes(), np.uint32).astype(np.int64)
        v[0] = (v[0] - a) if a < 1000 else a
        v[1] += b
        v[2] += c
        s[0:12] = np.frombuffer((v & 0xFFFFFFFF).astype(np.uint32).tobytes(), np.uint8)
        out.append(("sections_%d" % k, s, label))
    out.append(("head_only_13", _cat(np.zeros(12), [8]), None))
    out.append(("short_12", np.zeros(12, np.uint8), None))
    return out


def lz_parallel_shape(s):
    """True when lzi_parse_kernel keeps a stream the reference accepts: a token section of at least one token, every literal run but
    the last ending before the reference's break (tk_idx - 13), the last token carrying literals that end on the token section, and no
    distance 0 (the reference accepts one and copies destination bytes it never wrote; the parse leaves that to the serial kernel)"""
    s = _u8(s)
    n = len(s)
    if n < 13:
        return False
    tk0, tk_n, m_n = (int(v) for v in np.frombuffer(s[:12].tobytes(), np.uint32))
    if tk0 > n or tk0 + tk_n > n or tk0 + tk_n + m_n > n or tk0 < 13 or tk_n == 0:
        return False
    src_end, pos, m_pos = tk0 - 13, 13, tk0 + tk_n
    for k in range(tk_n):
        tok, last = int(s[tk0 + k]), k == tk_n - 1
        f = tok & 0x18
        if not last and f:
            nb = f >> 3
            if m_pos + nb > n or not any(s[m_pos: m_pos + nb]):
                return False
            m_pos += nb
        if tok >= 32:
            L = tok >> 5
            if tok >= 0xE0:
                if pos >= n:
                    return False
                v, nb = int(s[pos]), 1
                if v >= 254:
                    nb = 3 if v == 254 else 4
                    if pos + nb > n:
                        return False
                    v += (int(s[pos + 1]) << 8) + int(s[pos + 2]) if v == 254 else (int(s[pos + 1]) << 16) + (int(s[pos + 2]) << 8) + int(s[pos + 3])
                L = 7 + v
                pos += nb
            pos += L
            if pos > n or (not last and pos >= src_end):
                return False
        if last:
            return tok >= 32 and pos == tk0
    return False


# ---- ZRLT (ZRLT.go:146-225): every byte string is a stream ---------------------------------------------------------------------------

def zrlt_random(n, rng, p_digit=0.35, p_ff=0.1):
    u = rng.random(n)
    x = rng.integers(2, 0xFE, n).astype(np.uint8)
    x[u < p_digit] = (rng.random(int(np.count_nonzero(u < p_digit))) < 0.5).astype(np.uint8)
    ff = (u >= p_digit) & (u < p_digit + p_ff)
    x[ff] = 0xFF
    fe = (u >= p_digit + p_ff) & (u < p_digit + p_ff + 0.03)
    x[fe] = 0xFE
    return x


def zrlt_repro():
    """a 23-digit group across the first tile boundary: 8,170 bytes of 1, then 2^23 - 1 zeros; kanzi allows that in any block above
    8 MiB. The ZRLT forward of that data gives this stream back."""
    return _cat(np.full(8170, 2), np.zeros(23))


def zrlt_cases():
    """[(name, stream, cap or None)]: None = the cap sweep around the oracle's output length"""
    rng = np.random.default_rng(2002)
    out = []
    for n in (1, 2, 3, 15, 16, 17, 1000, ZTILE - 1, ZTILE, ZTILE + 1, 3 * ZTILE + 5, 200000):
        out.append(("random_n%d" % n, zrlt_random(n, rng), None))
    out.append(("random_ff_heavy", zrlt_random(100000, rng, 0.2, 0.5), None))
    out.append(("random_digits_heavy", zrlt_random(50000, rng, 0.6, 0.1), None))
    out.append(("random_4mib", zrlt_random(4 * MIB, rng, 0.3, 0.1), None))
    for L in range(1, 41):  # 0xFF runs ending at every offset around a tile boundary
        for end in (ZTILE - 2, ZTILE - 1, ZTILE, ZTILE + 1, ZTILE + 2):
            s = rng.integers(2, 0xFE, ZTILE + 64).astype(np.uint8)
            s[end - L: end] = 0xFF
            out.append(("ff_run%d_end%d" % (L, end), s, None))
    for nd in range(1, 23):  # digit groups straddling the tile boundary at every split (a group of nd digits is >= 2^nd - 1 zeros)
        for split in range(0, nd + 1) if nd <= 20 else (0, 1, nd // 2, nd - 1, nd):
            s = rng.integers(2, 0xFE, ZTILE + 40).astype(np.uint8)
            start = ZTILE - split
            s[start: start + nd] = rng.integers(0, 2, nd)
            out.append(("group%d_split%d" % (nd, split), s, None))
    s = rng.integers(2, 0xFE, 2 * ZTILE).astype(np.uint8)
    s[ZTILE - 5: ZTILE + 1] = [1, 0, 1, 1, 0, 1]  # a group continued from the previous tile that ends on the tile's first byte
    out.append(("group_ends_first_byte", s, None))
    out.append(("lone_trailing_ff", _cat(rng.integers(2, 0xFE, 100), [0xFF]), None))
    out.append(("ff_pair_trailing", _cat(rng.integers(2, 0xFE, 100), [0xFF, 0xFF]), None))
    out.append(("group_at_end", _cat(rng.integers(2, 0xFE, 100), [1, 0, 1]), None))
    out.append(("only_ff", np.full(1, 0xFF, np.uint8), None))
    out.append(("group_then_lone_ff", _cat(rng.integers(2, 0xFE, 100), [1, 0, 0xFF]), None))
    # groups whose value (zeros + 1) is exactly cap - di, cap - di + 1 and cap - di + 2 (di = the output before the group)
    grp = [int(c) for c in bin(1000)[3:]]  # value 1000: 999 zeros
    for j in (0, 1, 2):
        for at_end in (True, False):
            body = _cat(rng.integers(2, 0xFE, 50), grp) if at_end else _cat(rng.integers(2, 0xFE, 50), grp, [5])
            out.append(("group_value_is_cap_minus_di%s_%s" % ("+%d" % j if j else "", "end" if at_end else "mid"), body, 50 + 1000 - j))
    # groups of 64 .. 66 digits: the reference's run length wraps modulo 2^64
    for tail in ([1], [0, 1], [1, 1], [0]):
        g = [0] * 64 + tail
        out.append(("group_wraps_%s" % "".join(map(str, tail)), _cat([5, 6], g, [7]), None))
        out.append(("group_wraps_%s_end" % "".join(map(str, tail)), _cat([5, 6], g), None))
    g = [0] * (ZTILE - 10) + [0] * 64 + [1]  # a wrapping group across a tile boundary
    out.append(("group_wraps_across_tile", _cat(np.full(10, 9), g, [3]), None))
    out.append(("group_40_digits", _cat([5], [1] + [0] * 39, [7]), 1 << 20))
    return out


def zrlt_large_cases():
    """(name, stream, cap): groups across a tile boundary that decode to 8 MiB and 16 MiB of zeros"""
    s24 = _cat(np.full(ZTILE - 10, 3), [1] + [0] * 23, [4])  # 2^24 zeros, then one byte
    return [("repro_8mib", zrlt_repro(), 8170 + (1 << 23) - 1 + 64), ("group24_across_tile", s24, ZTILE - 10 + (1 << 24) + 64)]


# ---- MM (FSDCodec.Inverse, FSDCodec.go:317-404) -----------------------------------------------------------------------------------------

MM_DISTS = (0, 1, 2, 3, 4, 5, 8, 16, 17)


def mm_payload(n, rng, p_ff=0.1):
    x = rng.integers(0, 256, n).astype(np.uint8)
    x[rng.random(n) < p_ff] = 0xFF
    return x


def mm_cases():
    """[(name, stream)]: every (mode, dist) header over random payloads, then escape shapes under the valid headers"""
    rng = np.random.default_rng(3003)
    out = []
    for mode in (0, 1, 2):
        for dist in MM_DISTS:
            for n in (0, 1, dist, dist + 1, 31, 32, 33, 1000):
                out.append(("m%d_d%d_n%d" % (mode, dist, n), _cat([mode, dist], mm_payload(n, rng))))
    for dist in (1, 2, 3, 4, 8, 16):
        h = [0, dist]
        for L in (1, 2, 3, 4, 5, 31, 32, 33, 34, 63, 64, 65, 66):  # 0xFF runs of both parities across 32-byte tiles and groups of tiles
            for end in (30, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025):
                p = rng.integers(0, 0xFF, 1100).astype(np.uint8)
                p[max(0, end - L): end] = 0xFF
                out.append(("ff_run%d_end%d_d%d" % (L, end, dist), _cat(h, p)))
        out.append(("escape_last_d%d" % dist, _cat(h, rng.integers(0, 0xFF, 100), [0xFF])))
        out.append(("escape_pair_last_d%d" % dist, _cat(h, rng.integers(0, 0xFF, 100), [0xFF, 0x00])))
        p = rng.integers(0, 0xFF, 64 * 32).astype(np.uint8)
        p[5::32] = 0xFF
        out.append(("escape_every_tile_d%d" % dist, _cat(h, p)))
        p = rng.integers(0, 0xFF, 4000).astype(np.uint8)
        for k in range(0, 3900, 97):  # an escape on each of the dist chains next to each other
            p[k: k + 2 * dist: 2] = 0xFF
        out.append(("escape_every_chain_d%d" % dist, _cat(h, p)))
        out.append(("all_ff_d%d" % dist, _cat(h, np.full(777, 0xFF))))
    for dist in (1, 3, 16):
        for mode in (0, 1):
            out.append(("large_m%d_d%d" % (mode, dist), _cat([mode, dist], mm_payload(3 * MIB + 17, rng, 0.05))))
    return out


# ---- PACK / DNA (AliasCodec.Inverse, AliasCodec.go:278-434) -----------------------------------------------------------------------------

def alias_cases():
    """[(name, stream, cap or None)]"""
    rng = np.random.default_rng(4004)
    out = []
    for n in (0, 1, 15):
        out.append(("n%d" % n, _cat([n], rng.integers(0, 256, 40)), None))
    for n in (16, 17, 100, 200, 239):  # the digram map: n entries of (2 bytes, index), src[1] trailing bytes
        for trail in (0, 1, 2, 7, 255):
            body = rng.integers(0, 256, 3 * n + 500).astype(np.uint8)
            out.append(("map%d_trail%d" % (n, trail), _cat([n, trail], body), None))
        out.append(("map%d_short" % n, _cat([n, 0], rng.integers(0, 256, 3 * n - 1)), None))
        out.append(("map%d_trail_past_end" % n, _cat([n, 255], rng.integers(0, 256, 3 * n)), None))
    for osize_delta in (-1, 0, 1):  # one symbol: 0xFF, the symbol, a 4-byte size; the cap is set to 1000
        osize = 1000 + osize_delta
        out.append(("one_symbol_osize_cap%+d" % osize_delta, _cat([255, 0x41], np.frombuffer(np.uint32(osize).tobytes(), np.uint8)), 1000))
    out.append(("one_symbol_short", _cat([255, 0x41, 1, 0]), None))
    for nsym in range(2, 17):
        for adjust in range(0, 5):
            body = rng.integers(0, 256, 300).astype(np.uint8)
            out.append(("sym%d_adj%d" % (nsym, adjust), _cat([256 - nsym], rng.integers(0, 256, nsym), [adjust], body), None))
        out.append(("sym%d_truncated" % nsym, _cat([256 - nsym], rng.integers(0, 256, nsym - 1)), None))
    for n in (1, 2, 5, 1000, 100000, 3 * MIB + 5):
        out.append(("random_%d" % n, rng.integers(0, 256, n).astype(np.uint8), None))
        out.append(("random_map_%d" % n, _cat([int(rng.integers(16, 240)), int(rng.integers(0, 4))], rng.integers(0, 256, n)), None))
        out.append(("random_sym4_%d" % n, _cat([252, 1, 2, 3, 4, int(rng.integers(0, 4))], rng.integers(0, 256, n)), None))
        out.append(("random_sym9_%d" % n, _cat([247], rng.integers(0, 256, 9), [int(rng.integers(0, 2))], rng.integers(0, 256, n)), None))
    return out


# ---- TEXT: mutations of the oracle's forward ---------------------------------------------------------------------------------------------

TEXT_BS = 1 << 20  # ctx["blockSize"] of every TEXT case


def _text_sources():
    t = synth.markov_text(60000, seed=5)
    crlf = bytes(t).replace(b"\n", b"\r\n")[:60000]
    xml = b"".join(b"<item id=\"%d\">%s</item>\n" % (k, bytes(t[k * 50: k * 50 + 40])) for k in range(1200))[:60000]
    return [("plain", t), ("crlf", np.frombuffer(crlf, np.uint8)), ("xml", np.frombuffer(xml, np.uint8)), ("short", t[:3000])]


def text_cases(oracle):
    """[(name, stream)]: the oracle's TEXT forward of text blocks, then flips / inserts / deletes at escape and index tokens and at 2 KiB
    tile boundaries, two blocks' token streams back to back, and truncations"""
    rng = np.random.default_rng(5005)
    out, fwd = [], []
    for name, x in _text_sources():
        f, _ = oracle.transform_forward(T_TEXT, _u8(x), block_size=TEXT_BS)
        assert f is not None, name
        fwd.append((name, f))
        out.append(("fwd_" + name, f))
    for name, f in fwd:
        esc = np.flatnonzero((f >= 0x80) | (f == 0x0F) | (f == 0x0E))  # dictionary index bytes and the escapes
        spots = list(rng.choice(esc, 12, replace=False)) + [2048 * k + d for k in range(1, 6) for d in (-1, 0)]
        for k, p in enumerate(spots):
            p = int(min(p, len(f) - 1))
            g = f.copy()
            g[p] ^= np.uint8(1 << (k % 8))
            out.append(("%s_flip%d_at%d" % (name, k, p), g))
            out.append(("%s_ins%d_at%d" % (name, k, p), _cat(f[:p], [int(f[p]) ^ 0x80], f[p:])))
            out.append(("%s_del%d_at%d" % (name, k, p), _cat(f[:p], f[p + 1:])))
        for cut in (1, 17, len(f) // 2, len(f) - 1):
            out.append(("%s_trunc%d" % (name, cut), f[:cut].copy()))
    out.append(("concat_plain_xml", _cat(fwd[0][1], fwd[2][1])))
    out.append(("concat_short_short", _cat(fwd[3][1], fwd[3][1])))
    return out


# ---- mutations, every stage --------------------------------------------------------------------------------------------------------------

def mutations(cases, count, seed, head=13):
    """count seeded mutants of the streams of cases [(name, stream)]: single-byte flips, truncations and rewrites of one of the first
    `head` bytes"""
    rng = np.random.default_rng(seed)
    base = [(n, s) for n, s in cases if len(s) >= 2]
    out = []
    for k in range(count):
        name, s = base[int(rng.integers(0, len(base)))]
        s = s.copy()
        kind = k % 3
        if kind == 0:
            p = int(rng.integers(0, len(s)))
            s[p] ^= np.uint8(int(rng.integers(1, 256)))
        elif kind == 1:
            s = s[: int(rng.integers(1, len(s)))].copy()
        else:
            p = int(rng.integers(0, min(head, len(s))))
            s[p] = np.uint8(int(rng.integers(0, 256)))
        out.append(("%s_mut%d_%s" % (name, k, ("flip", "trunc", "head")[kind]), s))
    return out


# ---- block records ---------------------------------------------------------------------------------------------------------------------

def block_record(stream):
    """an E_NONE block record of one transform that ran (encodingTask.encode, CompressedStream.go:836-887): the mode byte (data size
    bits, skip flags 0x7F >> 4), the stream's length in 1..4 bytes, big-endian, then the stream -> (bytes, bits)"""
    n = len(stream)
    ds = 1 if n < 256 else (n.bit_length() - 1 >> 3) + 1
    head = [((ds - 1) << 5) | 0x07] + [(n >> (8 * (ds - 1 - i))) & 255 for i in range(ds)]
    rec = _cat(head, stream)
    return rec, 8 * len(rec)
