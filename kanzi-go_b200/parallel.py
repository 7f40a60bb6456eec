"""One kanzi stream over several GPUs (BASELINE.json north_star, SURVEY.md §8e).

Blocks are independent (io/CompressedStream.go:896-898), so the block path shards: rank r takes a contiguous range of blocks. The only
exchange steps are the ones the reference's Writer / Reader do in memory:

  compress    rank 0 holds the slab  -> scatter of the block ranges (grouped NCCL send / recv)
              every rank: kz_compress_fragment_device (its block records `5 b | lw b | payload`, bit exact length)
              all_gather of the fragment bit lengths -> gather-v of the fragments to rank 0 (grouped send / recv)
              rank 0: ordered bit-granular commit (Writer.processBlock :951-976): header | fragments in rank order | end marker,
                      a segment table laid out on the host, one funnel-shift copy on the GPU (kz_concat_bits_device)
  decompress  rank 0 holds the stream -> header + walk over the block length prefixes (kz_stream_index_device, Reader :1816-1852)
              broadcast of the stream parameters and record boundaries -> scatter of the byte windows that hold each rank's records
              every rank: kz_decompress_fragment_device at its start bit -> gather of the decoded ranges to rank 0

torch.distributed carries device tensors (NCCL over NVLink on GPUs); the codec work goes through an *engine*: `GpuEngine` (the C ABI of
include/kanzi_b200.h) in production, and a CPU stand-in that tests/test_parallel_gloo.py builds around the oracle to run the same
plumbing with gloo and world_size 2 where no GPU exists.
"""
import numpy as np

BS_TYPE = 0x4B414E5A
BS_VERSION = 6


def block_ranges(nblocks, world):
    """Contiguous block ranges per rank: [(first, last_exclusive)] — ceil(nblocks / world) blocks each (SURVEY.md §8e)."""
    per = (nblocks + world - 1) // world if nblocks else 0
    return [(min(r * per, nblocks), min((r + 1) * per, nblocks)) for r in range(world)]


def header_checksum(ck_size, etype, t48, block_size, sz_mask, input_size):
    """Writer.writeHeader :498-512."""
    M = 0xFFFFFFFF
    H = 0x1E35A7BD
    ck = (H * ((0x01030507 * BS_VERSION) & M)) & M
    ck ^= (H * (~ck_size & M)) & M
    ck ^= (H * (~etype & M)) & M
    ck ^= (H * ((~t48 >> 32) & M)) & M
    ck ^= (H * (~t48 & M)) & M
    ck ^= (H * (~block_size & M)) & M
    if sz_mask:
        ck ^= (H * ((~input_size >> 32) & M)) & M
        ck ^= (H * (~input_size & M)) & M
    return ((ck >> 23) ^ (ck >> 3)) & 0xFFFFFF


def stream_header_bits(input_size):
    """Length of the stream header (io/CompressedStream.go:429-519): 32 + 4 + 2 + 5 + 48 + 28 + 2 + 16 * szMask + 15 + 24 bits."""
    if input_size <= 0 or input_size >= (1 << 48):
        sz_mask = 0
    elif input_size >= (1 << 32):
        sz_mask = 3
    elif input_size >= (1 << 16):
        sz_mask = 2
    else:
        sz_mask = 1
    return 160 + 16 * sz_mask


class GpuEngine:
    """Codec work of one rank through the C ABI; every buffer is a torch uint8 CUDA tensor of this rank's device."""

    def __init__(self, ctx, torch):
        self.ctx = ctx
        self.torch = torch
        self.device = torch.device("cuda", ctx.device)

    def empty(self, n):
        return self.torch.empty(int(n) + 256, dtype=self.torch.uint8, device=self.device)

    def zeros(self, n):
        return self.torch.zeros(int(n) + 256, dtype=self.torch.uint8, device=self.device)

    def compress_fragment(self, src, n, t48, et, block_size, checksum_bits):
        cap = int(self.ctx.lib.kz_max_stream_output(n, block_size))
        dst = self.zeros(cap)
        bits = self.ctx.compress_fragment_device(src.data_ptr(), n, dst.data_ptr(), cap, t48, et, block_size, checksum_bits) if n else 0
        return dst, bits

    def commit(self, t48, et, block_size, checksum_bits, input_size, frags, frag_bits, cap):
        hdr, hbits = self.ctx.stream_header(t48, et, block_size, checksum_bits, input_size)
        d_hdr = self.torch.from_numpy(hdr).to(self.device)
        d_end = self.torch.zeros(16, dtype=self.torch.uint8, device=self.device)
        out = self.zeros(cap)
        ptrs = [d_hdr.data_ptr()] + [f.data_ptr() for f in frags] + [d_end.data_ptr()]
        bits = [hbits] + [int(b) for b in frag_bits] + [8]
        total = self.ctx.concat_bits_device(ptrs, bits, out.data_ptr(), cap)
        return out, (total + 7) // 8

    def index(self, stream, nbytes, max_blocks):
        return self.ctx.stream_index_device(stream.data_ptr(), nbytes, max_blocks)

    def decompress_fragment(self, frag, frag_bytes, start_bit, nblocks, t48, et, block_size, checksum_bits, cap):
        dst = self.empty(cap)
        n = self.ctx.decompress_fragment_device(frag.data_ptr(), frag_bytes, start_bit, nblocks, dst.data_ptr(), cap, t48, et, block_size, checksum_bits)
        return dst, n


class ShardedStream:
    """compress / decompress of ONE stream by all ranks of a torch.distributed group; the slab / the stream live on rank 0."""

    def __init__(self, engine, dist, torch):
        self.e, self.dist, self.torch = engine, dist, torch
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.exchanged_bytes = 0  # bytes this rank sent or received over the collective fabric in the last call
        self.t_exchange = 0.0     # seconds spent in scatter / gather / broadcast (accumulated; with a device synchronise at the phase ends)
        self.t_codec = 0.0        # seconds spent in the engine (fragment encode / decode, commit, index)
        self._t0 = None

    def _tick(self):
        import time

        if self.torch.cuda.is_available():
            self.torch.cuda.synchronize()
        self._t0 = time.perf_counter()

    def _tock(self, what):
        import time

        if self.torch.cuda.is_available():
            self.torch.cuda.synchronize()
        dt = time.perf_counter() - self._t0
        if what == "x":
            self.t_exchange += dt
        else:
            self.t_codec += dt
        self._t0 = time.perf_counter()

    def _p2p(self, ops):
        if ops:
            for w in self.dist.batch_isend_irecv(ops):
                w.wait()

    # ------------------------------------------------------------------------------------------------------------------------------
    def compress(self, slab, n, t48, et, block_size, checksum_bits=0, input_size=0):
        """slab: uint8 tensor with the n input bytes on rank 0 (ignored elsewhere). Returns (stream tensor, bytes) on rank 0, (None, 0) elsewhere."""
        dist, torch, e = self.dist, self.torch, self.e
        nblocks = (n + block_size - 1) // block_size
        ranges = block_ranges(nblocks, self.world)
        lo, hi = ranges[self.rank]
        my_bytes = max(0, min(n, hi * block_size) - lo * block_size)
        self.exchanged_bytes = 0
        self._tick()
        # ---- scatter of the block ranges
        if self.rank == 0:
            ops = []
            for r in range(1, self.world):
                a, b = ranges[r]
                nb = max(0, min(n, b * block_size) - a * block_size)
                if nb:
                    ops.append(dist.P2POp(dist.isend, slab[a * block_size: a * block_size + nb], r))
                    self.exchanged_bytes += nb
            self._p2p(ops)
            mine = slab[lo * block_size: lo * block_size + my_bytes] if my_bytes else e.empty(0)
        else:
            mine = e.empty(my_bytes)
            if my_bytes:
                self._p2p([dist.P2POp(dist.irecv, mine[:my_bytes], 0)])
                self.exchanged_bytes += my_bytes
        self._tock("x")
        # ---- encode
        frag, bits = e.compress_fragment(mine, my_bytes, t48, et, block_size, checksum_bits)
        self._tock("c")
        # ---- gather of the bit lengths, gather-v of the fragments
        all_bits = torch.zeros(self.world, dtype=torch.int64, device=frag.device)
        mine_bits = torch.tensor([bits], dtype=torch.int64, device=frag.device)
        dist.all_gather_into_tensor(all_bits, mine_bits) if hasattr(dist, "all_gather_into_tensor") and frag.is_cuda else self._all_gather(all_bits, mine_bits)
        all_bits = [int(v) for v in all_bits.tolist()]
        if self.rank != 0:
            nb = (bits + 7) // 8
            if nb:
                self._p2p([dist.P2POp(dist.isend, frag[:nb], 0)])
                self.exchanged_bytes += nb
            self._tock("x")
            return None, 0
        frags, ops = [frag], []
        for r in range(1, self.world):
            nb = (all_bits[r] + 7) // 8
            buf = e.zeros(nb)
            if nb:
                ops.append(dist.P2POp(dist.irecv, buf[:nb], r))
                self.exchanged_bytes += nb
            frags.append(buf)
        self._p2p(ops)
        self._tock("x")
        # ---- ordered commit
        cap = sum((b + 7) // 8 for b in all_bits) + 64
        res = e.commit(t48, et, block_size, checksum_bits, input_size, frags, all_bits, cap)
        self._tock("c")
        return res

    def _all_gather(self, out, mine):
        parts = [self.torch.zeros_like(mine) for _ in range(self.world)]
        self.dist.all_gather(parts, mine)
        for r, p in enumerate(parts):
            out[r] = p[0]

    # ------------------------------------------------------------------------------------------------------------------------------
    def decompress(self, stream, nbytes, out_cap):
        """stream: the complete stream on rank 0. Returns (decoded tensor, bytes) on rank 0, (None, 0) elsewhere."""
        dist, torch, e = self.dist, self.torch, self.e
        self.exchanged_bytes = 0
        self._tick()
        dev = stream.device if self.rank == 0 else e.empty(0).device
        # ---- header + record boundaries on rank 0, broadcast: [t48, et, bs, ck, nblocks, rec_bit of every range boundary]
        meta = torch.zeros(6 + self.world + 1, dtype=torch.int64, device=dev)
        if self.rank == 0:
            max_blocks = out_cap // 1024 + 16
            ix = e.index(stream, nbytes, max_blocks)
            ranges = block_ranges(ix["nblocks"], self.world)
            vals = [ix["transform48"], ix["entropy"], ix["block_size"], ix["checksum_bits"], ix["nblocks"], nbytes]
            vals += [ix["rec_bit"][ranges[r][0]] for r in range(self.world)] + [ix["rec_bit"][ix["nblocks"]]]
            meta.copy_(torch.tensor(vals, dtype=torch.int64))
            self._tock("c")
        dist.broadcast(meta, 0)
        m = [int(v) for v in meta.tolist()]
        t48, et, bs, ck, nblocks, nbytes = m[:6]
        bounds = m[6:]
        ranges = block_ranges(nblocks, self.world)
        lo, hi = ranges[self.rank]

        def window(r):  # byte window of rank r's records, start aligned down to 16 bytes
            a = (bounds[r] // 8) & ~15
            b = (bounds[r + 1] + 7) // 8 if ranges[r][1] > ranges[r][0] else a
            return a, max(a, b)

        # ---- scatter of the windows
        a, b = window(self.rank)
        if self.rank == 0:
            ops = []
            for r in range(1, self.world):
                ra, rb = window(r)
                if rb > ra:
                    ops.append(dist.P2POp(dist.isend, stream[ra:rb], r))
                    self.exchanged_bytes += rb - ra
            self._p2p(ops)
            frag = stream[a:]
            frag_bytes = nbytes - a
        else:
            frag = e.zeros(b - a)
            frag_bytes = b - a
            if b > a:
                self._p2p([dist.P2POp(dist.irecv, frag[: b - a], 0)])
                self.exchanged_bytes += b - a
        self._tock("x")
        # ---- decode
        my_cap = (hi - lo) * bs + 4096
        dec, n = e.decompress_fragment(frag, frag_bytes, bounds[self.rank] - 8 * a, hi - lo, t48, et, bs, ck, my_cap) if hi > lo else (e.empty(0), 0)
        self._tock("c")
        # ---- gather of the decoded ranges (every range but the last is full blocks)
        sizes = torch.zeros(self.world, dtype=torch.int64, device=dec.device)
        mine_n = torch.tensor([n], dtype=torch.int64, device=dec.device)
        dist.all_gather_into_tensor(sizes, mine_n) if hasattr(dist, "all_gather_into_tensor") and dec.is_cuda else self._all_gather(sizes, mine_n)
        sizes = [int(v) for v in sizes.tolist()]
        if self.rank != 0:
            if n:
                self._p2p([dist.P2POp(dist.isend, dec[:n], 0)])
                self.exchanged_bytes += n
            self._tock("x")
            return None, 0
        total = sum(sizes)
        out = e.empty(max(total, out_cap))
        if n:
            out[:n].copy_(dec[:n])
        ops, off = [], n
        for r in range(1, self.world):
            if sizes[r]:
                ops.append(dist.P2POp(dist.irecv, out[off: off + sizes[r]], r))
                self.exchanged_bytes += sizes[r]
            off += sizes[r]
        self._p2p(ops)
        self._tock("x")
        return out, total
