"""kanzi-go_b200 — H100-native (sm_90a) drop-in for the per-block encode/decode path of flanglet/kanzi-go.

Python host-side mirror of the reference's operator interfaces for this path (the Go toolchain is absent from the
build image, so the parity tests and bench drive the C ABI of include/kanzi_b200.h through ctypes; INTEGRATION.md
shows the cgo binding a kanzi-go maintainer would add). Names follow the reference:

  EntropyEncoder / EntropyDecoder   v2/Definitions.go:154-179  (Write(block) / Read(block))
  ByteTransform                     v2/Definitions.go:78-91    (Forward / Inverse / MaxEncodedLen)
  Writer / Reader                   v2/io/CompressedStream.go  (NewWriter :216, NewReader :1047)

There is no CPU fallback: importing works without a GPU (so that the library's symbols can be checked), but creating a
Context without a CUDA device raises.
"""
import contextlib
import ctypes as C
import os

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libkanzi_b200.so")

E_NONE, E_HUFFMAN, E_RANGE, E_ANS0, E_ANS1 = 0, 1, 4, 5, 8
T_NONE, T_BWT, T_BWTS, T_LZ, T_ROLZ, T_LZX = 0, 1, 2, 3, 11, 16
T_ZRLT, T_MTFT, T_RANK = 6, 7, 8
T_PACK, T_DNA, T_MM, T_TEXT, T_UTF, T_EXE = 18, 19, 15, 10, 17, 9
ENTROPY_IDS = {"NONE": 0, "HUFFMAN": 1, "FPAQ": 2, "RANGE": 4, "ANS0": 5, "CM": 6, "TPAQ": 7, "ANS1": 8, "TPAQX": 9}
TRANSFORM_IDS = {"NONE": 0, "BWT": 1, "BWTS": 2, "LZ": 3, "RLT": 5, "ZRLT": 6, "MTFT": 7, "RANK": 8, "EXE": 9, "TEXT": 10, "ROLZ": 11,
                 "ROLZX": 12, "SRT": 13, "LZP": 14, "MM": 15, "LZX": 16, "UTF": 17, "PACK": 18, "DNA": 19}

ABI_SYMBOLS = [
    "kz_device_count", "kz_init", "kz_destroy", "kz_last_error", "kz_alloc_pinned", "kz_free_pinned", "kz_cuda_stream", "kz_launch_count",
    "kz_entropy_encode", "kz_entropy_decode", "kz_transform_forward", "kz_transform_inverse", "kz_transform_max_encoded_len",
    "kz_encode_blocks", "kz_decode_blocks", "kz_max_block_output", "kz_compress_stream", "kz_decompress_stream", "kz_max_stream_output",
    "kz_compress_stream_device", "kz_decompress_stream_device", "kz_profile", "kz_kernel_time", "kz_profile_reset", "kz_set_stream_block_size",
    "kz_stage_bytes", "kz_profile_names",
    "kz_compress_fragment_device", "kz_stream_header", "kz_concat_bits_device", "kz_stream_index_device", "kz_decompress_fragment_device",
    "kz_compress_streams", "kz_decompress_streams", "kz_compress_streams_device", "kz_decompress_streams_device",
    "kz_writer_open", "kz_writer_write", "kz_writer_finish", "kz_writer_free", "kz_reader_open", "kz_reader_read", "kz_reader_finish",
    "kz_reader_free", "kz_device_bytes", "kz_set_block_range", "kz_bwt_profile",
    "kz_set_headerless_writer", "kz_set_headerless_reader", "kz_clear_headerless_reader", "kz_set_skip_blocks",
    "kz_index_build", "kz_index_build_device", "kz_index_info", "kz_index_save", "kz_index_load", "kz_index_free", "kz_read_ranges",
    "kz_read_ranges_device", "kz_cache_create", "kz_cache_free", "kz_cache_clear", "kz_cache_stats", "kz_read_ranges_cached",
    "kz_read_ranges_cached_device", "kz_index_build_streams", "kz_index_build_streams_device", "kz_read_ranges_streams",
    "kz_read_ranges_streams_device", "kz_compress_streams_bs", "kz_compress_streams_bs_device", "kz_write_ranges", "kz_write_ranges_device",
    "kz_write_ranges_streams", "kz_write_ranges_streams_device",
]

WRITE_APPEND = (1 << 64) - 1  # KZ_WRITE_APPEND: a write's offset that means the end of the data as the call's earlier writes left it


class KanziError(RuntimeError):
    """Mirrors io.IOError{msg, code} (v2/io/CompressedStream.go:56-75)."""

    def __init__(self, code, msg):
        self.code = code
        super().__init__("%s (code %d)" % (msg, code))


def transform_type(names):
    """transform.GetType (v2/transform/Factory.go:288-328): "BWT+RANK+ZRLT" -> 48-bit id word."""
    res, shift, count = 0, 42, 0
    for tok in names.split("+"):
        t = TRANSFORM_IDS.get(tok.upper())
        if t is None:
            raise KanziError(18, "Unknown transform type: '%s'" % tok)
        if t != 0:
            count += 1
            if count > 8:
                raise KanziError(18, "Only 8 transforms allowed: '%s'" % names)
            res |= t << shift
            shift -= 6
    return res


def entropy_type(name):
    """entropy.GetType (v2/entropy/EntropyCodecFactory.go:170-206)."""
    t = ENTROPY_IDS.get(name.upper())
    if t is None:
        raise KanziError(18, "Unsupported entropy codec type: '%s'" % name)
    return t


_lib = None


def load_library(build_if_missing=True):
    """Loads libkanzi_b200.so (building it with nvcc when absent). Fails loudly: there is no fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise KanziError(4, "libkanzi_b200.so is missing; run python -c 'import __graft_entry__ as g; g.build()'")
        _build.build()
    L = C.CDLL(LIB_PATH)
    vp, sz, u32, u64, i32 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.c_int
    L.kz_device_count.restype = i32
    L.kz_init.argtypes = [i32, C.POINTER(vp)]
    L.kz_destroy.argtypes = [vp]
    L.kz_destroy.restype = None
    L.kz_last_error.argtypes = [vp]
    L.kz_last_error.restype = C.c_char_p
    L.kz_alloc_pinned.argtypes = [sz]
    L.kz_alloc_pinned.restype = vp
    L.kz_free_pinned.argtypes = [vp]
    L.kz_free_pinned.restype = None
    L.kz_cuda_stream.argtypes = [vp]
    L.kz_cuda_stream.restype = vp
    L.kz_launch_count.argtypes = [vp, i32]
    L.kz_launch_count.restype = u64
    L.kz_entropy_encode.argtypes = [vp, u32, vp, sz, vp, sz, C.POINTER(u64)]
    L.kz_entropy_decode.argtypes = [vp, u32, vp, sz, vp, sz, C.POINTER(u64)]
    L.kz_transform_forward.argtypes = [vp, u64, C.POINTER(i32), vp, sz, vp, sz, C.POINTER(sz)]
    L.kz_transform_inverse.argtypes = [vp, u64, vp, sz, vp, sz, C.POINTER(sz)]
    L.kz_transform_max_encoded_len.argtypes = [u64, sz]
    L.kz_transform_max_encoded_len.restype = sz
    L.kz_encode_blocks.argtypes = [vp, u64, u32, u32, vp, u64, vp, u32, vp, u64, vp, vp]
    L.kz_decode_blocks.argtypes = [vp, u64, u32, u32, vp, vp, vp, u32, u32, vp, u64, vp, vp]
    L.kz_max_block_output.argtypes = [sz]
    L.kz_max_block_output.restype = sz
    L.kz_compress_stream.argtypes = [vp, u64, u32, u32, u32, C.c_int64, vp, sz, vp, sz, C.POINTER(sz)]
    L.kz_decompress_stream.argtypes = [vp, vp, sz, vp, sz, C.POINTER(sz)]
    L.kz_max_stream_output.argtypes = [sz, u32]
    L.kz_max_stream_output.restype = sz
    L.kz_compress_stream_device.argtypes = [vp, u64, u32, u32, u32, C.c_int64, vp, sz, vp, sz, C.POINTER(sz)]
    L.kz_decompress_stream_device.argtypes = [vp, vp, sz, vp, sz, C.POINTER(sz)]
    L.kz_profile.argtypes = [vp, i32]
    L.kz_profile.restype = None
    L.kz_kernel_time.argtypes = [vp, C.c_char_p, C.POINTER(C.c_double)]
    L.kz_kernel_time.restype = u32
    L.kz_profile_reset.argtypes = [vp]
    L.kz_profile_reset.restype = None
    L.kz_set_stream_block_size.argtypes = [vp, C.c_uint64]
    L.kz_compress_fragment_device.argtypes = [vp, u64, u32, u32, u32, vp, sz, vp, sz, C.POINTER(u64)]
    L.kz_stream_header.argtypes = [u64, u32, u32, u32, C.c_int64, vp, C.POINTER(u32)]
    L.kz_concat_bits_device.argtypes = [vp, u32, C.POINTER(vp), C.POINTER(u64), vp, sz, C.POINTER(u64)]
    L.kz_stream_index_device.argtypes = [vp, vp, sz, u32, C.POINTER(u64), C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), C.POINTER(C.c_int64), C.POINTER(u64),
                                         C.POINTER(u32)]
    L.kz_decompress_fragment_device.argtypes = [vp, u64, u32, u32, u32, vp, sz, u64, u32, vp, sz, C.POINTER(sz)]
    L.kz_stage_bytes.argtypes = [vp, C.c_char_p, C.POINTER(u64), C.POINTER(u64)]
    L.kz_stage_bytes.restype = u32
    L.kz_profile_names.argtypes = [vp, C.c_char_p, sz]
    L.kz_profile_names.restype = sz
    L.kz_bwt_profile.argtypes = [vp, i32]
    L.kz_bwt_profile.restype = None
    L.kz_set_stream_block_size.restype = None
    L.kz_set_block_range.argtypes = [vp, C.c_int64, C.c_int64]
    L.kz_set_headerless_writer.argtypes = [vp, i32]
    L.kz_set_headerless_reader.argtypes = [vp, u64, u32, u32, u32, C.c_int64, u32]
    L.kz_clear_headerless_reader.argtypes = [vp]
    L.kz_set_skip_blocks.argtypes = [vp, i32]
    L.kz_compress_streams.argtypes = [vp, u64, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_compress_streams_device.argtypes = [vp, u64, u32, u32, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_compress_streams_bs.argtypes = [vp, u64, u32, vp, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_compress_streams_bs_device.argtypes = [vp, u64, u32, vp, u32, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_decompress_streams.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_decompress_streams_device.argtypes = [vp, u32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_writer_open.argtypes = [vp, u64, u32, u32, u32, u32, C.c_int64, C.POINTER(vp)]
    L.kz_writer_write.argtypes = [vp, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]
    L.kz_writer_finish.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.kz_writer_free.argtypes = [vp]
    L.kz_writer_free.restype = None
    L.kz_reader_open.argtypes = [vp, u32, C.POINTER(vp)]
    L.kz_reader_read.argtypes = [vp, vp, sz, C.POINTER(sz), vp, sz, C.POINTER(sz)]
    L.kz_reader_finish.argtypes = [vp, vp, sz, C.POINTER(sz)]
    L.kz_reader_free.argtypes = [vp]
    L.kz_reader_free.restype = None
    L.kz_device_bytes.argtypes = [vp]
    L.kz_device_bytes.restype = sz
    L.kz_index_build.argtypes = [vp, vp, sz, C.POINTER(vp)]
    L.kz_index_build_device.argtypes = [vp, vp, sz, C.POINTER(vp)]
    L.kz_index_info.argtypes = [vp, C.POINTER(u64), C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), C.POINTER(C.c_int64), C.POINTER(u64), C.POINTER(u64),
                                C.POINTER(C.c_int64)]
    L.kz_index_save.argtypes = [vp, vp, sz]
    L.kz_index_save.restype = sz
    L.kz_index_load.argtypes = [vp, sz, C.POINTER(vp)]
    L.kz_index_free.argtypes = [vp]
    L.kz_index_free.restype = None
    L.kz_read_ranges.argtypes = [vp, vp, vp, sz, u32, vp, vp, vp, vp, vp, vp]
    L.kz_read_ranges_device.argtypes = [vp, vp, vp, sz, u32, vp, vp, vp, vp, vp, vp]
    L.kz_cache_create.argtypes = [vp, u64, C.POINTER(vp)]
    L.kz_cache_free.argtypes = [vp]
    L.kz_cache_free.restype = None
    L.kz_cache_clear.argtypes = [vp]
    L.kz_cache_stats.argtypes = [vp] + [C.POINTER(u64)] * 8
    L.kz_read_ranges_cached.argtypes = [vp, vp, vp, vp, sz, u32, vp, vp, vp, vp, vp, vp]
    L.kz_read_ranges_cached_device.argtypes = [vp, vp, vp, vp, sz, u32, vp, vp, vp, vp, vp, vp]
    L.kz_index_build_streams.argtypes = [vp, u32, vp, vp, vp, vp, vp]
    L.kz_index_build_streams_device.argtypes = [vp, u32, vp, vp, vp, vp, vp]
    L.kz_read_ranges_streams.argtypes = [vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
    L.kz_read_ranges_streams_device.argtypes = [vp, vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp]
    L.kz_write_ranges.argtypes = [vp, vp, vp, sz, u32, vp, vp, vp, vp, vp, sz, C.POINTER(u64), C.POINTER(sz)]
    L.kz_write_ranges_device.argtypes = [vp, vp, vp, sz, u32, vp, vp, vp, vp, vp, sz, C.POINTER(u64), C.POINTER(sz)]
    L.kz_write_ranges_streams.argtypes = [vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.kz_write_ranges_streams_device.argtypes = [vp, u32, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    _lib = L
    return L


def _u8(a):
    if isinstance(a, np.ndarray):
        return np.ascontiguousarray(a, dtype=np.uint8)
    return np.frombuffer(a, dtype=np.uint8)


def _p(a):
    return a.ctypes.data if a.size else None


def _offsets(lens):
    """Exclusive prefix sums of lens (uint64)."""
    off = np.zeros(len(lens), np.uint64)
    if len(lens) > 1:
        off[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    return off


def _dptr(t):
    return t.data_ptr() if hasattr(t, "data_ptr") else t


class Context:
    """One engine context per GPU (kz_init). All codec objects of a process share it."""

    def __init__(self, device=0):
        self.lib = load_library()
        h = C.c_void_p()
        rc = self.lib.kz_init(device, C.byref(h))
        if rc != 0:
            raise KanziError(-rc, "cannot create the engine on CUDA device %d (no GPU / no driver?) - there is no CPU fallback" % device)
        self.h = h
        self.device = device
        self._range = (-1, -1)  # kz_set_block_range's (from, to) on this context
        self._hl_writer = False  # kz_set_headerless_writer's setting
        self._hl_reader = None   # kz_set_headerless_reader's arguments, None when it is off
        self._skip = False       # kz_set_skip_blocks's setting

    def close(self):
        if getattr(self, "h", None):
            self.lib.kz_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise KanziError(-rc, self.lib.kz_last_error(self.h).decode(errors="replace"))
        return rc

    # ---- raw ABI helpers -------------------------------------------------------------------------------------
    def entropy_encode(self, etype, block):
        a = _u8(block)
        cap = self.lib.kz_max_block_output(a.size)
        out = np.empty(cap, np.uint8)
        bits = C.c_uint64(0)
        self._check(self.lib.kz_entropy_encode(self.h, etype, _p(a), a.size, out.ctypes.data, cap, C.byref(bits)))
        return out[: (bits.value + 7) // 8].copy(), bits.value

    def entropy_decode(self, etype, stream, n):
        s = _u8(stream)
        out = np.empty(max(n, 1), np.uint8)
        used = C.c_uint64(0)
        self._check(self.lib.kz_entropy_decode(self.h, etype, _p(s), s.size, out.ctypes.data, n, C.byref(used)))
        return out[:n], used.value

    def set_stream_block_size(self, block_size):
        """ctx["blockSize"] for the following block / single-transform calls (only TEXT reads it); 0 = the longest block of the call"""
        self.lib.kz_set_stream_block_size(self.h, block_size)

    def transform_forward(self, ttype, block, data_type=0):
        """ByteTransform.Forward for one transform id -> (bytes or None when the transform declines, data_type after)."""
        a = _u8(block)
        cap = max(int(self.lib.kz_transform_max_encoded_len(ttype, a.size)), a.size) + 64
        out = np.empty(cap, np.uint8)
        n = C.c_size_t(0)
        dt = C.c_int(data_type)
        rc = self._check(self.lib.kz_transform_forward(self.h, ttype, C.byref(dt), _p(a), a.size, out.ctypes.data, cap, C.byref(n)))
        if rc == 1:
            return None, dt.value
        return out[: n.value].copy(), dt.value

    def transform_inverse(self, ttype, block, cap):
        a = _u8(block)
        out = np.empty(max(cap, 1), np.uint8)
        n = C.c_size_t(0)
        self._check(self.lib.kz_transform_inverse(self.h, ttype, _p(a), a.size, out.ctypes.data, cap, C.byref(n)))
        return out[: n.value].copy()

    def encode_blocks(self, transform48, etype, blocks, checksum_bits=0, skip_blocks=None):
        """blocks: list of byte arrays -> list of (bytes, nbits). One kz_encode_blocks call (Writer.processBlock batch). skip_blocks: see
        set_skip_blocks (None: the context's setting)."""
        nb = len(blocks)
        arrs = [_u8(b) for b in blocks]
        lens = np.array([a.size for a in arrs], np.uint32)
        stride = int((max(lens.max(initial=0), 1) + 15) // 16 * 16)
        slab = np.zeros(stride * max(nb, 1), np.uint8)
        for i, a in enumerate(arrs):
            slab[i * stride: i * stride + a.size] = a
        ostride = int((self.lib.kz_max_block_output(int(lens.max(initial=0))) + 15) // 16 * 16)
        out = np.zeros(ostride * max(nb, 1), np.uint8)
        bits = np.zeros(max(nb, 1), np.uint64)
        status = np.zeros(max(nb, 1), np.int32)
        with self._skip_blocks(skip_blocks):
            self._check(self.lib.kz_encode_blocks(self.h, transform48, etype, checksum_bits, slab.ctypes.data, stride, lens.ctypes.data, nb,
                                                  out.ctypes.data, ostride, bits.ctypes.data, status.ctypes.data))
        return [(out[i * ostride: i * ostride + (int(bits[i]) + 7) // 8].copy(), int(bits[i])) for i in range(nb)]

    def decode_blocks(self, transform48, etype, payloads, block_size, checksum_bits=0):
        """payloads: list of (bytes, nbits) -> list of decoded byte arrays (Reader.processBlock batch)."""
        nb = len(payloads)
        offs, bits, chunks, o = [], [], [], 0
        for p, nbits in payloads:
            a = _u8(p)
            offs.append(o)
            bits.append(nbits)
            chunks.append(a)
            o += a.size
        blob = np.concatenate(chunks) if chunks else np.zeros(0, np.uint8)
        offs = np.array(offs, np.uint64)
        bits = np.array(bits, np.uint64)
        ostride = int(block_size + block_size // 2 + 2048)
        out = np.zeros(ostride * max(nb, 1), np.uint8)
        lens = np.zeros(max(nb, 1), np.uint32)
        status = np.zeros(max(nb, 1), np.int32)
        self._check(self.lib.kz_decode_blocks(self.h, transform48, etype, checksum_bits, _p(blob), offs.ctypes.data, bits.ctypes.data, nb, block_size,
                                              out.ctypes.data, ostride, lens.ctypes.data, status.ctypes.data))
        return [out[i * ostride: i * ostride + int(lens[i])].copy() for i in range(nb)]

    def compress(self, data, transform="NONE", entropy="NONE", block_size=4 << 20, checksum_bits=0, input_size=0, headerless=None, skip_blocks=None):
        """headerless: True / False sets the headerless writer setting for this call (None: the context's setting). skip_blocks: the same
        for set_skip_blocks."""
        a = _u8(data)
        t48 = transform_type(transform) if isinstance(transform, str) else transform
        et = entropy_type(entropy) if isinstance(entropy, str) else entropy
        cap = self.lib.kz_max_stream_output(a.size, block_size)
        out = np.empty(cap, np.uint8)
        n = C.c_size_t(0)
        with self._headerless(writer=headerless), self._skip_blocks(skip_blocks):
            self._check(self.lib.kz_compress_stream(self.h, t48, et, block_size, checksum_bits, input_size, _p(a), a.size, out.ctypes.data, cap, C.byref(n)))
        return out[: n.value].copy()

    def decompress(self, stream, out_cap, from_block=None, to_block=None, headerless=None):
        """from_block / to_block: decode only that range of blocks (see set_block_range) for this call. headerless: a dict of
        set_headerless_reader's arguments, the headerless reader setting for this call (None: the context's setting)."""
        s = _u8(stream)
        out = np.empty(max(out_cap, 1), np.uint8)
        n = C.c_size_t(0)
        with self._block_range(from_block, to_block), self._headerless(reader=headerless):
            self._check(self.lib.kz_decompress_stream(self.h, _p(s), s.size, out.ctypes.data, out_cap, C.byref(n)))
        return out[: n.value]

    # ---- block range (kz_set_block_range): kanzi's ctx["from"] / ctx["to"] ---------------------------------------------------------
    def set_block_range(self, from_block=-1, to_block=-1):
        """Decode only blocks from_block <= id < to_block (ids start at 1; a negative value = not given) in the stream-level decodes that
        follow: decompress*, decompress_streams* and stream_reader (captured when the session opens)."""
        self._check(self.lib.kz_set_block_range(self.h, from_block, to_block))
        self._range = (from_block if from_block >= 0 else -1, to_block if to_block >= 0 else -1)

    @contextlib.contextmanager
    def _block_range(self, from_block, to_block):
        """Sets the range for one call when either bound is given, and restores the previous range afterwards."""
        if from_block is None and to_block is None:
            yield
            return
        prev = self._range
        self.set_block_range(-1 if from_block is None else from_block, -1 if to_block is None else to_block)
        try:
            yield
        finally:
            self.set_block_range(*prev)

    # ---- headerless streams (kz_set_headerless_writer / kz_set_headerless_reader): NewWriter(..., headerless) and NewHeaderlessReader -----
    def set_headerless_writer(self, on=True):
        """The stream-level encodes that follow (compress*, compress_streams*, stream_writer when it opens) write no stream header."""
        self._check(self.lib.kz_set_headerless_writer(self.h, 1 if on else 0))
        self._hl_writer = bool(on)

    def set_headerless_reader(self, transform, entropy, block_size, checksum_bits=0, output_size=-1, bs_version=6):
        """The stream-level decodes that follow (decompress*, decompress_streams*, stream_reader when it opens, stream_index_device) read
        no header and take these parameters (NewHeaderlessReader's). Checked now, as Reader.validateHeaderless does: a bad value raises and
        leaves the previous setting."""
        t48 = transform_type(transform) if isinstance(transform, str) else transform
        et = entropy_type(entropy) if isinstance(entropy, str) else entropy
        args = (t48, et, block_size, checksum_bits, output_size, bs_version)
        self._check(self.lib.kz_set_headerless_reader(self.h, *args))
        self._hl_reader = args

    def clear_headerless_reader(self):
        self._check(self.lib.kz_clear_headerless_reader(self.h))
        self._hl_reader = None

    @contextlib.contextmanager
    def _headerless(self, writer=None, reader=None):
        """Sets the headerless writer flag (writer: a bool) and / or the headerless reader parameters (reader: a dict of
        set_headerless_reader's arguments) for one call, and restores the previous settings afterwards. None leaves a setting as it is."""
        prev_w, prev_r = self._hl_writer, self._hl_reader
        try:
            if writer is not None:
                self.set_headerless_writer(writer)
            if reader is not None:
                self.set_headerless_reader(**reader)
            yield
        finally:
            if writer is not None:
                self.set_headerless_writer(prev_w)
            if reader is not None:
                if prev_r is None:
                    self.clear_headerless_reader()
                else:
                    self.set_headerless_reader(*prev_r)

    # ---- kanzi's skipBlocks option (kz_set_skip_blocks): store incompressible blocks raw ----------------------------------------------
    def set_skip_blocks(self, on=True):
        """The encodes that follow (encode_blocks, compress*, compress_streams*, compress_fragment_device, stream_writer when it opens) store
        every block of more than 15 bytes that starts with a compressed format's magic number or whose order-0 entropy reaches 973 / 1024
        as a COPY block, as kanzi c --skip does."""
        self._check(self.lib.kz_set_skip_blocks(self.h, 1 if on else 0))
        self._skip = bool(on)

    @contextlib.contextmanager
    def _skip_blocks(self, on):
        """Sets the skipBlocks setting for one call (on: a bool) and restores the previous one afterwards. None leaves it as it is."""
        if on is None:
            yield
            return
        prev = self._skip
        self.set_skip_blocks(on)
        try:
            yield
        finally:
            self.set_skip_blocks(prev)

    # ---- many independent streams in one call (kz_compress_streams / kz_decompress_streams) -----------------------------------
    # Per-stream failures do not raise: status[s] = 0 or -(kanzi error code), and outputs[s] is None for a failed stream.
    def compress_streams(self, inputs, transform, entropy, block_size, checksum_bits=0, input_sizes=None, headerless=None, skip_blocks=None):
        """One compressed stream per input, each equal to compress(inputs[s], ..., input_size=input_sizes[s]) -> (outputs, status).
        block_size: one int for every stream, or a sequence with one block size per stream (kanzi's `-b auto`: see auto_block_size); a
        stream whose block size compress refuses then fails alone with status -KZ_ERR_INVALID_PARAM."""
        arrs = [_u8(x) for x in inputs]
        t48 = transform_type(transform) if isinstance(transform, str) else transform
        et = entropy_type(entropy) if isinstance(entropy, str) else entropy
        src_len = np.array([a.size for a in arrs], np.uint64)
        src_off = _offsets(src_len)
        src = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
        bs = _block_sizes(block_size, len(arrs))
        sizes = [block_size] * len(arrs) if bs is None else [int(b) for b in bs]
        cap = np.array([self.lib.kz_max_stream_output(a.size, b) for a, b in zip(arrs, sizes)], np.uint64)
        dst_off = _offsets(cap)
        dst = np.empty(max(int(cap.sum()), 1), np.uint8)
        isz = None if input_sizes is None else np.ascontiguousarray(input_sizes, np.int64)
        out_len, status = np.zeros(len(arrs), np.uint64), np.zeros(len(arrs), np.int32)
        with self._headerless(writer=headerless), self._skip_blocks(skip_blocks):
            if bs is None:
                self.lib.kz_compress_streams(self.h, t48, et, block_size, checksum_bits, len(arrs), _p(src), _p(src_off), _p(src_len),
                                             None if isz is None else _p(isz), dst.ctypes.data, _p(dst_off), _p(cap), _p(out_len), _p(status))
            else:
                self.lib.kz_compress_streams_bs(self.h, t48, et, _p(bs), checksum_bits, len(arrs), _p(src), _p(src_off), _p(src_len),
                                                None if isz is None else _p(isz), dst.ctypes.data, _p(dst_off), _p(cap), _p(out_len), _p(status))
        outs = [dst[int(o): int(o) + int(n)].copy() if st == 0 else None for o, n, st in zip(dst_off, out_len, status)]
        return outs, status

    def decompress_streams(self, streams, caps, from_block=None, to_block=None, headerless=None):
        """Decodes every stream (headers may differ) into at most caps[s] bytes -> (outputs, status). from_block / to_block: the same block
        range for every stream. headerless: the same parameters for every stream (see decompress)."""
        arrs = [_u8(x) for x in streams]
        src_len = np.array([a.size for a in arrs], np.uint64)
        src_off = _offsets(src_len)
        src = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
        cap = np.ascontiguousarray(caps, np.uint64)
        dst_off = _offsets(cap)
        dst = np.empty(max(int(cap.sum()), 1), np.uint8)
        out_len, status = np.zeros(len(arrs), np.uint64), np.zeros(len(arrs), np.int32)
        with self._block_range(from_block, to_block), self._headerless(reader=headerless):
            self.lib.kz_decompress_streams(self.h, len(arrs), _p(src), _p(src_off), _p(src_len), dst.ctypes.data, _p(dst_off), _p(cap), _p(out_len),
                                           _p(status))
        outs = [dst[int(o): int(o) + int(n)].copy() if st == 0 else None for o, n, st in zip(dst_off, out_len, status)]
        return outs, status

    def compress_streams_device(self, src, src_off, src_len, dst, dst_off, dst_cap, transform, entropy, block_size, checksum_bits=0,
                                input_sizes=None, headerless=None, skip_blocks=None):
        """src / dst: CUDA uint8 tensors (or device addresses); offsets (multiples of 16) and lengths: host sequences -> (out_len, status).
        block_size: an int, or one block size per stream (as compress_streams)."""
        t48 = transform_type(transform) if isinstance(transform, str) else transform
        et = entropy_type(entropy) if isinstance(entropy, str) else entropy
        so, sl, do, dc = (np.ascontiguousarray(a, np.uint64) for a in (src_off, src_len, dst_off, dst_cap))
        isz = None if input_sizes is None else np.ascontiguousarray(input_sizes, np.int64)
        out_len, status = np.zeros(len(sl), np.uint64), np.zeros(len(sl), np.int32)
        bs = _block_sizes(block_size, len(sl))
        with self._headerless(writer=headerless), self._skip_blocks(skip_blocks):
            if bs is None:
                self.lib.kz_compress_streams_device(self.h, t48, et, block_size, checksum_bits, len(sl), _dptr(src), _p(so), _p(sl),
                                                    None if isz is None else _p(isz), _dptr(dst), _p(do), _p(dc), _p(out_len), _p(status))
            else:
                self.lib.kz_compress_streams_bs_device(self.h, t48, et, _p(bs), checksum_bits, len(sl), _dptr(src), _p(so), _p(sl),
                                                       None if isz is None else _p(isz), _dptr(dst), _p(do), _p(dc), _p(out_len), _p(status))
        return out_len, status

    def decompress_streams_device(self, src, src_off, src_len, dst, dst_off, dst_cap, from_block=None, to_block=None, headerless=None):
        """Device-resident decompress_streams: inputs need >= 64 readable bytes behind each -> (out_len, status)."""
        so, sl, do, dc = (np.ascontiguousarray(a, np.uint64) for a in (src_off, src_len, dst_off, dst_cap))
        out_len, status = np.zeros(len(sl), np.uint64), np.zeros(len(sl), np.int32)
        with self._block_range(from_block, to_block), self._headerless(reader=headerless):
            self.lib.kz_decompress_streams_device(self.h, len(sl), _dptr(src), _p(so), _p(sl), _dptr(dst), _p(do), _p(dc), _p(out_len), _p(status))
        return out_len, status

    # ---- device-resident entry points (pointers are CUDA device addresses, e.g. torch tensors' data_ptr()) -------
    def compress_device(self, d_src, n, d_dst, cap, transform48, etype, block_size, checksum_bits=0, input_size=0, headerless=None, skip_blocks=None):
        out_n = C.c_size_t(0)
        with self._headerless(writer=headerless), self._skip_blocks(skip_blocks):
            self._check(self.lib.kz_compress_stream_device(self.h, transform48, etype, block_size, checksum_bits, input_size, d_src, n, d_dst, cap,
                                                           C.byref(out_n)))
        return out_n.value

    def decompress_device(self, d_src, n, d_dst, cap, from_block=None, to_block=None, headerless=None):
        out_n = C.c_size_t(0)
        with self._block_range(from_block, to_block), self._headerless(reader=headerless):
            self._check(self.lib.kz_decompress_stream_device(self.h, d_src, n, d_dst, cap, C.byref(out_n)))
        return out_n.value

    def compress_host(self, src_ptr, n, dst_ptr, cap, transform48, etype, block_size, checksum_bits=0, input_size=0):
        out_n = C.c_size_t(0)
        self._check(self.lib.kz_compress_stream(self.h, transform48, etype, block_size, checksum_bits, input_size, src_ptr, n, dst_ptr, cap, C.byref(out_n)))
        return out_n.value

    def decompress_host(self, src_ptr, n, dst_ptr, cap):
        out_n = C.c_size_t(0)
        self._check(self.lib.kz_decompress_stream(self.h, src_ptr, n, dst_ptr, cap, C.byref(out_n)))
        return out_n.value

    # ---- sharded streams (one stream, blocks spread over ranks; kanzi-go_b200/parallel.py drives these) ---------------------
    def compress_fragment_device(self, d_src, n, d_dst, cap, transform48, etype, block_size, checksum_bits=0, skip_blocks=None):
        bits = C.c_uint64(0)
        with self._skip_blocks(skip_blocks):
            self._check(self.lib.kz_compress_fragment_device(self.h, transform48, etype, block_size, checksum_bits, d_src, n, d_dst, cap, C.byref(bits)))
        return bits.value

    def stream_header(self, transform48, etype, block_size, checksum_bits=0, input_size=0):
        out = np.zeros(32, np.uint8)
        bits = C.c_uint32(0)
        rc = self.lib.kz_stream_header(transform48, etype, block_size, checksum_bits, input_size, out.ctypes.data, C.byref(bits))
        if rc:
            raise KanziError(-rc, "kz_stream_header")
        return out, bits.value

    def concat_bits_device(self, seg_ptrs, seg_bits, d_dst, cap):
        n = len(seg_ptrs)
        ptrs = (C.c_void_p * max(n, 1))(*seg_ptrs)
        bits = (C.c_uint64 * max(n, 1))(*seg_bits)
        total = C.c_uint64(0)
        self._check(self.lib.kz_concat_bits_device(self.h, n, ptrs, bits, d_dst, cap, C.byref(total)))
        return total.value

    def stream_index_device(self, d_src, n, max_blocks, headerless=None):
        t48, et, bs, ck, isz, nb = C.c_uint64(0), C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_int64(0), C.c_uint32(0)
        rec = (C.c_uint64 * (max_blocks + 1))()
        with self._headerless(reader=headerless):
            self._check(self.lib.kz_stream_index_device(self.h, d_src, n, max_blocks, C.byref(t48), C.byref(et), C.byref(bs), C.byref(ck), C.byref(isz),
                                                        rec, C.byref(nb)))
        return {"transform48": t48.value, "entropy": et.value, "block_size": bs.value, "checksum_bits": ck.value, "input_size": isz.value,
                "rec_bit": [int(rec[i]) for i in range(nb.value + 1)], "nblocks": nb.value}

    def decompress_fragment_device(self, d_src, frag_bytes, start_bit, nblocks, d_dst, cap, transform48, etype, block_size, checksum_bits=0):
        out_n = C.c_size_t(0)
        self._check(self.lib.kz_decompress_fragment_device(self.h, transform48, etype, block_size, checksum_bits, d_src, frag_bytes, start_bit, nblocks, d_dst,
                                                           cap, C.byref(out_n)))
        return out_n.value

    def cuda_stream(self):
        return self.lib.kz_cuda_stream(self.h)

    # ---- stream index (kz_index_*): built once, then serves batched range reads (StreamIndex.read / read_many) ---------------------
    def index(self, stream, headerless=None):
        """The StreamIndex of a host stream: header fields and record positions; decodes nothing. headerless: as in decompress."""
        s = _u8(stream)
        h = C.c_void_p()
        with self._headerless(reader=headerless):
            self._check(self.lib.kz_index_build(self.h, _p(s), s.size, C.byref(h)))
        return StreamIndex(h, self)

    def index_device(self, d_src, n, headerless=None):
        """The StreamIndex of the stream of n bytes at d_src (16-byte aligned, >= 64 readable bytes behind it)."""
        h = C.c_void_p()
        with self._headerless(reader=headerless):
            self._check(self.lib.kz_index_build_device(self.h, _dptr(d_src), n, C.byref(h)))
        return StreamIndex(h, self)

    # ---- many streams per call (kz_index_build_streams / kz_read_ranges_streams): an object store's table of small objects ----------
    # Per-stream and per-request failures do not raise: status[s] / status[i] = 0 or -(kanzi error code).
    def index_streams(self, streams, headerless=None):
        """One StreamIndex per host stream, each what index(streams[s]) gives -> (indexes, status); indexes[s] is None when stream s failed."""
        arrs = [_u8(x) for x in streams]
        src_len = np.array([a.size for a in arrs], np.uint64)
        src = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
        return self._index_streams(self.lib.kz_index_build_streams, _p(src), _offsets(src_len), src_len, headerless)

    def index_streams_device(self, d_src, src_off, src_len, headerless=None):
        """index_streams of the streams d_src[src_off[s] : + src_len[s]] (16-byte aligned, >= 64 readable bytes behind each)."""
        so, sl = (np.ascontiguousarray(a, np.uint64) for a in (src_off, src_len))
        return self._index_streams(self.lib.kz_index_build_streams_device, _dptr(d_src), so, sl, headerless)

    def _index_streams(self, fn, src, so, sl, headerless):
        n = len(sl)
        hs = (C.c_void_p * max(n, 1))()
        status = np.zeros(n, np.int32)
        with self._headerless(reader=headerless):
            fn(self.h, n, src, _p(so), _p(sl), C.addressof(hs), _p(status))
        return [StreamIndex(hs[s], self) if hs[s] else None for s in range(n)], status

    @staticmethod
    def _index_slots(indexes):
        return (C.c_void_p * max(len(indexes), 1))(*[None if x is None else x.h for x in indexes])

    def read_streams(self, streams, indexes, requests, cache=None):
        """requests: [(stream_no, off, length), ...] on host streams with their indexes (None allowed) -> (list of bytes, status list):
        each request gets what indexes[stream_no].read_many(streams[stream_no], ...) gives it, in one call over all streams."""
        arrs = [_u8(x) for x in streams]
        src_len = np.array([a.size for a in arrs], np.uint64)
        src_off = _offsets(src_len)
        src = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
        ix = self._index_slots(indexes)
        rs = np.array([r[0] for r in requests], np.uint32)
        off = np.array([r[1] for r in requests], np.uint64)
        ln = np.array([r[2] for r in requests], np.uint64)
        dst_off = _offsets(ln)
        dst = np.empty(max(int(ln.sum()), 1), np.uint8)
        out_len, status = np.zeros(len(requests), np.uint64), np.zeros(len(requests), np.int32)
        self.lib.kz_read_ranges_streams(self.h, None if cache is None else cache.h, len(arrs), C.addressof(ix), _p(src), _p(src_off), _p(src_len),
                                        len(requests), _p(rs), _p(off), _p(ln), dst.ctypes.data, _p(dst_off), _p(out_len), _p(status))
        return [dst[int(o): int(o) + int(n)].tobytes() for o, n in zip(dst_off, out_len)], status.tolist()

    def read_streams_device(self, d_src, src_off, src_len, indexes, req_stream, off, length, d_dst, dst_off, cache=None):
        """Device-resident read_streams: d_src / d_dst are CUDA tensors or addresses, the rest host sequences -> (out_len, status)."""
        so, sl, o, ln, do = (np.ascontiguousarray(a, np.uint64) for a in (src_off, src_len, off, length, dst_off))
        rs = np.ascontiguousarray(req_stream, np.uint32)
        ix = self._index_slots(indexes)
        out_len, status = np.zeros(len(o), np.uint64), np.zeros(len(o), np.int32)
        self.lib.kz_read_ranges_streams_device(self.h, None if cache is None else cache.h, len(sl), C.addressof(ix), _dptr(d_src), _p(so), _p(sl), len(o),
                                               _p(rs), _p(o), _p(ln), _dptr(d_dst), _p(do), _p(out_len), _p(status))
        return out_len, status

    def write_streams(self, streams, indexes, writes):
        """writes: [(slot, off, data), ...] in order on host streams with their indexes (None allowed for slots no write names) ->
        (keeps, tails, status): slot s gets what indexes[s].write_many(streams[s], its writes) gives, as keeps[s] and tails[s], in one call
        over all slots (kz_write_ranges_streams). Failures do not raise: status[s] = 0 or -(kanzi error code), and a failed slot's index
        is unchanged. A slot whose tail did not fit is called again alone with the capacity it named."""
        arrs = [_u8(x) for x in streams]
        ns = len(arrs)
        src_len = np.array([a.size for a in arrs], np.uint64)
        src_off = _offsets(src_len)
        src = np.concatenate(arrs) if arrs else np.zeros(0, np.uint8)
        bufs = [_u8(w[2]) for w in writes]
        ws = np.array([int(w[0]) for w in writes], np.uint32)
        off = np.array([int(w[1]) for w in writes], np.uint64)
        ln = np.array([b.size for b in bufs], np.uint64)
        data = np.concatenate(bufs) if bufs else np.zeros(0, np.uint8)
        data_off = _offsets(ln)
        # write_many's capacity per slot: (n - keep) + k * kz_max_block_output(block_size) + 16, k bounded by the blocks the writes span
        cap = np.zeros(ns, np.uint64)
        for s in sorted(set(int(w) for w, n in zip(ws, ln) if n)):
            bs = indexes[s].info["block_size"] if indexes[s] is not None else 1024
            k = sum(int(n) // bs + 2 for w, n in zip(ws, ln) if n and w == s)
            cap[s] = src_len[s] + k * self.lib.kz_max_block_output(bs) + 16
        keeps, tails, status = [int(n) for n in src_len], [b""] * ns, [0] * ns
        todo = np.arange(ns)
        while True:
            # the slots still to serve, and the writes on them, renumbered
            slot = np.full(ns, -1, np.int64)
            slot[todo] = np.arange(len(todo))
            pick = np.array([i for i in range(len(writes)) if slot[ws[i]] >= 0], np.int64)
            sub = [arrs[s] for s in todo]
            t_len = src_len[todo]
            t_so = _offsets(t_len)
            t_src = np.concatenate(sub) if sub else np.zeros(0, np.uint8)
            t_cap = cap[todo]
            dst_off = _offsets(t_cap)
            dst = np.empty(max(int(t_cap.sum()), 1), np.uint8)
            keep, out_n, st = np.zeros(len(todo), np.uint64), np.zeros(len(todo), np.uint64), np.zeros(len(todo), np.int32)
            ix = self._index_slots([indexes[s] for s in todo])
            t_ws = slot[ws[pick]].astype(np.uint32) if len(pick) else np.zeros(0, np.uint32)
            t_off, t_ln, t_do = (np.ascontiguousarray(a[pick] if len(pick) else a[:0]) for a in (off, ln, data_off))
            self.lib.kz_write_ranges_streams(self.h, len(todo), C.addressof(ix), _p(t_src), _p(t_so), _p(t_len), len(pick), _p(t_ws),
                                             _p(t_off), _p(t_ln), _p(data), _p(t_do), dst.ctypes.data, _p(dst_off), _p(t_cap), _p(keep), _p(out_n),
                                             _p(st))
            again = []
            for j, s in enumerate(todo):
                if st[j] == -12 and out_n[j] > t_cap[j]:  # KZ_ERR_WRITE_FILE: the index is unchanged, call again with the capacity named
                    cap[s] = out_n[j]
                    again.append(s)
                    continue
                keeps[s], status[s] = int(keep[j]), int(st[j])
                tails[s] = dst[int(dst_off[j]): int(dst_off[j]) + int(out_n[j])].tobytes() if not st[j] else b""
            if not again:
                return keeps, tails, status
            todo = np.array(again, np.int64)

    def write_streams_device(self, d_src, src_off, src_len, indexes, w_stream, off, length, d_data, data_off, d_dst, dst_off, dst_cap):
        """Device-resident write_streams (kz_write_ranges_streams_device): d_src / d_data / d_dst are CUDA tensors or addresses, the rest
        host sequences -> (keep, out_n, status). On -KZ_ERR_WRITE_FILE (code 12) out_n[s] is the capacity slot s needs."""
        so, sl, o, ln, doff, dso, dcap = (np.ascontiguousarray(a, np.uint64) for a in (src_off, src_len, off, length, data_off, dst_off, dst_cap))
        ws = np.ascontiguousarray(w_stream, np.uint32)
        ix = self._index_slots(indexes)
        keep, out_n, status = np.zeros(len(sl), np.uint64), np.zeros(len(sl), np.uint64), np.zeros(len(sl), np.int32)
        self.lib.kz_write_ranges_streams_device(self.h, len(sl), C.addressof(ix), _dptr(d_src), _p(so), _p(sl), len(o), _p(ws), _p(o), _p(ln),
                                                _dptr(d_data), _p(doff), _dptr(d_dst), _p(dso), _p(dcap), _p(keep), _p(out_n), _p(status))
        return keep, out_n, status

    def block_cache(self, budget):
        """A BlockCache of decoded blocks in `budget` bytes of HBM (kz_cache_create), for StreamIndex.read / read_many /
        read_many_device(cache=...) on this context."""
        h = C.c_void_p()
        self._check(self.lib.kz_cache_create(self.h, budget, C.byref(h)))
        return BlockCache(self, h)

    # ---- streaming sessions (kz_writer_* / kz_reader_*): one stream of any length in bounded memory -------------------------------
    def stream_writer(self, transform, entropy, block_size, checksum_bits=0, batch_blocks=None, input_size=0, headerless=None, skip_blocks=None):
        """A StreamSession: write(data) -> bytes and finish() -> bytes give the stream compress() writes for the concatenated input.
        batch_blocks=None: about 256 MiB of input per batch. headerless, skip_blocks: as in compress (the session keeps the settings it
        opened with)."""
        t48 = transform_type(transform) if isinstance(transform, str) else transform
        et = entropy_type(entropy) if isinstance(entropy, str) else entropy
        if batch_blocks is None:
            batch_blocks = default_batch_blocks(block_size)
        h = C.c_void_p()
        with self._headerless(writer=headerless), self._skip_blocks(skip_blocks):
            self._check(self.lib.kz_writer_open(self.h, t48, et, block_size, checksum_bits, batch_blocks, input_size, C.byref(h)))
        return StreamSession(self, h, self.lib.kz_writer_write, self.lib.kz_writer_finish, self.lib.kz_writer_free)

    def stream_reader(self, batch_blocks=None, from_block=None, to_block=None, headerless=None):
        """A StreamSession: write(data) -> decoded bytes and finish() -> the rest. batch_blocks=None: about 256 MiB per batch, resolved
        from the block size in the stream's header. from_block / to_block: the session decodes only that range of blocks. headerless: as
        in decompress (the session keeps the setting it opened with)."""
        if batch_blocks is None:
            batch_blocks = 0
        h = C.c_void_p()
        with self._block_range(from_block, to_block), self._headerless(reader=headerless):
            self._check(self.lib.kz_reader_open(self.h, batch_blocks, C.byref(h)))
        return StreamSession(self, h, self.lib.kz_reader_read, self.lib.kz_reader_finish, self.lib.kz_reader_free)

    def device_bytes(self):
        """Device bytes held by this context's scratch and an open session's buffers (kz_device_bytes)."""
        return int(self.lib.kz_device_bytes(self.h))

    # ---- instrumentation ---------------------------------------------------------------------------------------
    def profile(self, on=True):
        self.lib.kz_profile(self.h, 1 if on else 0)

    def profile_reset(self):
        self.lib.kz_profile_reset(self.h)

    def kernel_time(self, name):
        ms = C.c_double(0)
        n = self.lib.kz_kernel_time(self.h, name.encode(), C.byref(ms))
        return n, ms.value

    def stage_bytes(self, name):
        """-> (batches, bytes_in, bytes_out) of "stage:fwd:<id>" / "stage:inv:<id>" since the last profile_reset"""
        a, b = C.c_uint64(0), C.c_uint64(0)
        k = self.lib.kz_stage_bytes(self.h, name.encode(), C.byref(a), C.byref(b))
        return k, a.value, b.value

    def profile_names(self):
        n = self.lib.kz_profile_names(self.h, None, 0)
        buf = C.create_string_buffer(n + 16)
        self.lib.kz_profile_names(self.h, buf, n + 16)
        return [x for x in buf.value.decode().split("\n") if x]

    def bwt_profile(self, time_rounds=False, wide_rounds=False, inverse_stride=0, inverse_stage=0):
        """BWT forward rounds (kz_bwt_profile): time every round under "bwt_round:<r>:<part>" (and the inverse's parts under
        "bwt_inverse:<part>") / run the 56-bit global sort in every round / the inverse's sub-list stride (a power of two) and staging
        bytes per sub-list (a multiple of 16); 0 = the default of each"""
        lg = inverse_stride.bit_length() - 1 if inverse_stride else 0
        if inverse_stride and (1 << lg) != inverse_stride or not 0 <= lg < 16:
            raise ValueError("inverse_stride must be a power of two below 65536")
        if inverse_stage % 16 or not 0 <= inverse_stage // 16 < 256:
            raise ValueError("inverse_stage must be a multiple of 16 below 4096")
        flags = (1 if time_rounds else 0) | (2 if wide_rounds else 0) | (lg << 8) | ((inverse_stage // 16) << 12)
        self.lib.kz_bwt_profile(self.h, flags)

    def launch_count(self, reset=False):
        return self.lib.kz_launch_count(self.h, 1 if reset else 0)


class StreamIndex:
    """Where every block record of one stream lies (kz_index): a host object, built by Context.index / index_device or loaded from a saved
    blob. read / read_many / read_many_device return decoded bytes [off, off + length) and decode only the blocks they touch; they take
    the stream again (the index does not own it) and the context to decode on (ctx=None: the one that built the index)."""

    def __init__(self, h, ctx=None):
        self.h, self.ctx = h, ctx
        self.lib = load_library()

    @classmethod
    def load(cls, blob, ctx=None):
        """An index from save()'s bytes; needs no GPU. A damaged blob raises KanziError(15)."""
        b = _u8(blob)
        h = C.c_void_p()
        rc = load_library().kz_index_load(_p(b), b.size, C.byref(h))
        if rc:
            raise KanziError(-rc, "not a stream index blob")
        return cls(h, ctx)

    def close(self):
        if getattr(self, "h", None):
            self.lib.kz_index_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def info(self):
        t48, ns, nb, isz, size = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_int64(0), C.c_int64(0)
        et, bs, ck = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        self.lib.kz_index_info(self.h, C.byref(t48), C.byref(et), C.byref(bs), C.byref(ck), C.byref(isz), C.byref(nb), C.byref(ns), C.byref(size))
        return {"transform48": t48.value, "entropy": et.value, "block_size": bs.value, "checksum_bits": ck.value, "input_size": isz.value,
                "nblocks": nb.value, "stream_bytes": ns.value, "size": size.value}

    @property
    def size(self):
        """Decoded bytes of the stream; -1 until a read has decoded the last block."""
        return self.info["size"]

    def save(self):
        n = self.lib.kz_index_save(self.h, None, 0)
        out = np.zeros(n, np.uint8)
        self.lib.kz_index_save(self.h, out.ctypes.data, n)
        return out.tobytes()

    def read_many(self, stream, requests, ctx=None, cache=None):
        """requests: [(off, length), ...] -> (list of bytes, status list). Failures do not raise: status[i] = 0 or -(kanzi error code); a
        short request gives fewer bytes, a failed one b"". A call-level failure (stale index, open session) sets every status.
        cache: a BlockCache of the context (kz_read_ranges_cached): the same results, blocks it holds are copied instead of decoded."""
        ctx = ctx or self.ctx
        s = _u8(stream)
        off = np.array([r[0] for r in requests], np.uint64)
        ln = np.array([r[1] for r in requests], np.uint64)
        dst_off = _offsets(ln)
        dst = np.empty(max(int(ln.sum()), 1), np.uint8)
        out_len, status = np.zeros(len(requests), np.uint64), np.zeros(len(requests), np.int32)
        args = (_p(s), s.size, len(requests), _p(off), _p(ln), dst.ctypes.data, _p(dst_off), _p(out_len), _p(status))
        if cache is None:
            self.lib.kz_read_ranges(ctx.h, self.h, *args)
        else:
            self.lib.kz_read_ranges_cached(ctx.h, cache.h, self.h, *args)
        return [dst[int(o): int(o) + int(n)].tobytes() for o, n in zip(dst_off, out_len)], status.tolist()

    def read(self, stream, off, length, ctx=None, cache=None):
        """Decoded bytes [off, off + length), short at the end of the data; raises when the block fails."""
        out, st = self.read_many(stream, [(off, length)], ctx, cache)
        if st[0]:
            (ctx or self.ctx)._check(st[0])
        return out[0]

    def read_many_device(self, d_src, n, off, length, d_dst, dst_off, ctx=None, cache=None):
        """Device-resident read_many: d_src / d_dst are CUDA tensors or addresses, the rest host sequences -> (out_len, status)."""
        ctx = ctx or self.ctx
        o, ln, do = (np.ascontiguousarray(a, np.uint64) for a in (off, length, dst_off))
        out_len, status = np.zeros(len(o), np.uint64), np.zeros(len(o), np.int32)
        args = (_dptr(d_src), n, len(o), _p(o), _p(ln), _dptr(d_dst), _p(do), _p(out_len), _p(status))
        if cache is None:
            self.lib.kz_read_ranges_device(ctx.h, self.h, *args)
        else:
            self.lib.kz_read_ranges_cached_device(ctx.h, cache.h, self.h, *args)
        return out_len, status

    def write_many(self, stream, writes, ctx=None):
        """writes: [(off, data), ...] in order (off = WRITE_APPEND: the current end) -> (keep, tail): the new stream is stream[:keep] + tail,
        what compress gives for the new data, and the index now describes it (kz_write_ranges). Only the blocks the writes touch are
        re-encoded. Raises KanziError, leaving the index as it was."""
        ctx = ctx or self.ctx
        s = _u8(stream)
        bufs = [_u8(d) for _, d in writes]
        off = np.array([int(o) for o, _ in writes], np.uint64)
        ln = np.array([b.size for b in bufs], np.uint64)
        data = np.concatenate(bufs) if bufs else np.zeros(0, np.uint8)
        bs = self.info["block_size"]
        # (n - keep) + k * kz_max_block_output(block_size) + 16 with k bounded by the blocks the writes span; a zero gap may add more, and
        # the call then names the capacity it needs
        k = sum(int(n) // bs + 2 for n in ln if n)
        cap = s.size + k * self.lib.kz_max_block_output(bs) + 16
        keep, out_n = C.c_uint64(0), C.c_size_t(0)
        data_off = _offsets(ln)  # held for the call: a temporary's buffer could be freed before the library reads it
        while True:
            dst = np.empty(max(cap, 1), np.uint8)
            rc = self.lib.kz_write_ranges(ctx.h, self.h, _p(s), s.size, len(writes), _p(off), _p(ln), _p(data), _p(data_off), dst.ctypes.data, cap,
                                          C.byref(keep), C.byref(out_n))
            if rc == -12 and out_n.value > cap:  # KZ_ERR_WRITE_FILE
                cap = out_n.value
                continue
            ctx._check(rc)
            return keep.value, dst[: out_n.value].tobytes()

    def write(self, stream, off, data, ctx=None):
        """data at decoded offset off (pwrite: past the end grows the data, a gap reads as zeros) -> (keep, tail), as write_many."""
        return self.write_many(stream, [(off, data)], ctx)

    def append(self, stream, data, ctx=None):
        """data behind the end of the data -> (keep, tail), as write_many."""
        return self.write_many(stream, [(WRITE_APPEND, data)], ctx)

    def write_many_device(self, d_src, n, off, length, d_data, data_off, d_dst, cap, ctx=None):
        """Device-resident write_many (kz_write_ranges_device): d_src / d_data / d_dst are CUDA tensors or addresses, off / length /
        data_off host sequences -> (keep, out_n). Raises KanziError; on -KZ_ERR_WRITE_FILE (code 12) its `needed` is the capacity the
        call needs."""
        ctx = ctx or self.ctx
        o, ln, do = (np.ascontiguousarray(a, np.uint64) for a in (off, length, data_off))
        keep, out_n = C.c_uint64(0), C.c_size_t(0)
        rc = self.lib.kz_write_ranges_device(ctx.h, self.h, _dptr(d_src), n, len(o), _p(o), _p(ln), _dptr(d_data), _p(do), _dptr(d_dst), cap,
                                             C.byref(keep), C.byref(out_n))
        try:
            ctx._check(rc)
        except KanziError as e:
            e.needed = out_n.value
            raise
        return keep.value, out_n.value


class BlockCache:
    """Decoded blocks kept in HBM between range reads (kz_cache_*), made by Context.block_cache(budget). Entries belong to the content
    of a record, so one cache serves every stream and index read on its context. A context manager: leaving the block frees the cache."""

    STATS = ("entries", "resident_bytes", "budget_bytes", "hits", "misses", "inserts", "evictions", "served_bytes")

    def __init__(self, ctx, h):
        self.ctx, self.h = ctx, h
        self.lib = load_library()

    @property
    def stats(self):
        v = [C.c_uint64(0) for _ in self.STATS]
        self.lib.kz_cache_stats(self.h, *[C.byref(x) for x in v])
        return {k: x.value for k, x in zip(self.STATS, v)}

    def clear(self):
        """Drops every entry; the counters stay."""
        self.ctx._check(self.lib.kz_cache_clear(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.lib.kz_cache_free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def auto_block_size(size, jobs):
    """The block size BlockCompressor's `-b auto` gives a file of `size` bytes compressed with `jobs` jobs (app/BlockCompressor.go:574-580):
    size / jobs, rounded up to a multiple of 64, clamped to [1 KiB, 1 GiB]."""
    bs = size // jobs
    bs = (bs + 63) & ~63
    return max(1024, min(bs, 1 << 30))


def _block_sizes(block_size, n):
    """None for one int block size; else the per-stream sizes as a uint32 array of n entries (values that do not fit go as 0, which every
    stream refuses)."""
    if isinstance(block_size, (int, np.integer)):
        return None
    sizes = [int(b) for b in block_size]
    if len(sizes) != n:
        raise KanziError(18, "block_size has %d entries for %d streams" % (len(sizes), n))
    return np.array([b if 0 <= b < (1 << 32) else 0 for b in sizes], np.uint32)


def default_batch_blocks(block_size):
    """Blocks per session batch that make about 256 MiB of input, in [1..1024]."""
    return max(1, min(1024, (256 << 20) // block_size))


class StreamSession:
    """One writer or reader session (Context.stream_writer / stream_reader) driven through its pump. A context manager: leaving the
    block frees the session, also mid-stream. out_cap: the output buffer each pump call fills."""

    def __init__(self, ctx, h, step, fin, free, out_cap=64 << 20):
        self.ctx, self.h, self._step, self._fin, self._free = ctx, h, step, fin, free
        self._out = np.empty(out_cap, np.uint8)

    def _live(self):
        if self.h is None or self.ctx.h is None:
            raise KanziError(18, "the session or its context is closed")

    def write(self, data):
        """Hands data to the session -> the finished bytes it gave back meanwhile."""
        self._live()
        a = _u8(data)
        parts, pos = [], 0
        used, made = C.c_size_t(0), C.c_size_t(0)
        while pos < a.size:  # bytes still in flight at the end come out of a later write() or finish()
            self.ctx._check(self._step(self.h, a.ctypes.data + pos, a.size - pos, C.byref(used), self._out.ctypes.data, self._out.size, C.byref(made)))
            pos += used.value
            if made.value:
                parts.append(self._out[: made.value].copy())
        return np.concatenate(parts) if parts else np.zeros(0, np.uint8)

    def finish(self):
        """End of input -> every remaining byte."""
        self._live()
        parts = []
        made = C.c_size_t(0)
        while True:
            rc = self.ctx._check(self._fin(self.h, self._out.ctypes.data, self._out.size, C.byref(made)))
            if made.value:
                parts.append(self._out[: made.value].copy())
            if rc == 0:
                break
        return np.concatenate(parts) if parts else np.zeros(0, np.uint8)

    def close(self):
        """Frees the session; legal after the context was closed too (kz_destroy closed the session then)."""
        if self.h:
            self._free(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None


def default_context():
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(int(os.environ.get("LOCAL_RANK", "0")))
    return _default_ctx


class OutputBitStream:
    """Minimal stand-in for kanzi.OutputBitStream (v2/Definitions.go:119-140) over a growing byte buffer: just what
    the codec mirrors need (WriteArray of the codec's bit string, Written). MSB first, like DefaultOutputBitStream."""

    def __init__(self):
        self._bits = []  # list of (np.uint8 array, nbits)
        self._written = 0

    def write_array(self, data, nbits):
        self._bits.append((np.array(_u8(data)[: (nbits + 7) // 8], copy=True), nbits))
        self._written += nbits

    def written(self):
        return self._written

    def to_bytes(self):
        """Zero padded bytes of everything written so far (bit-exact concatenation)."""
        total = np.zeros((self._written + 7) // 8 + 8, np.uint8)
        pos = 0
        for arr, nbits in self._bits:
            if nbits == 0:
                continue
            bits = np.unpackbits(arr)[:nbits]
            byte0, off = pos // 8, pos % 8
            padded = np.concatenate([np.zeros(off, np.uint8), bits])
            padded = np.concatenate([padded, np.zeros((-len(padded)) % 8, np.uint8)])
            chunk = np.packbits(padded)
            total[byte0: byte0 + len(chunk)] |= chunk
            pos += nbits
        return total[: (self._written + 7) // 8]


class EntropyEncoder:
    """kanzi.EntropyEncoder for the GPU codecs (entropy.NewEntropyEncoder(obs, ctx, type), EntropyCodecFactory.go:91-134)."""

    def __init__(self, bitstream, entropy, ctx=None):
        self.type = entropy_type(entropy) if isinstance(entropy, str) else entropy
        self.bs = bitstream
        self.ctx = ctx or default_context()

    def write(self, block):
        data, nbits = self.ctx.entropy_encode(self.type, block)
        self.bs.write_array(data, nbits)
        return len(block)

    def bit_stream(self):
        return self.bs

    def dispose(self):
        pass


class EntropyDecoder:
    """kanzi.EntropyDecoder (entropy.NewEntropyDecoder(ibs, ctx, type), EntropyCodecFactory.go:45-88). The input
    bit stream is the block-local byte buffer (io/CompressedStream.go:1875) plus a bit cursor."""

    def __init__(self, data, entropy, ctx=None, bit_offset=0):
        if bit_offset % 8:
            raise KanziError(18, "the block-local stream is byte aligned when the entropy decoder is created")
        self.type = entropy_type(entropy) if isinstance(entropy, str) else entropy
        self.data = _u8(data)[bit_offset // 8:]
        self.ctx = ctx or default_context()
        self.consumed = 0

    def read(self, n):
        out, used = self.ctx.entropy_decode(self.type, self.data, n)
        self.consumed = used
        return out

    def dispose(self):
        pass


class ByteTransform:
    """kanzi.ByteTransform (v2/Definitions.go:78-91) for the GPU transforms: transform.New(ctx, type) of a single id."""

    def __init__(self, name, ctx=None):
        self.type = TRANSFORM_IDS[name.upper()]
        self.ctx = ctx or default_context()
        self.data_type = 0

    def forward(self, src):
        """-> transformed bytes, or None when the transform declines (the reference returns an error = "skip me")."""
        out, self.data_type = self.ctx.transform_forward(self.type, src, self.data_type)
        return out

    def inverse(self, src, max_len):
        return self.ctx.transform_inverse(self.type, src, max_len)

    def max_encoded_len(self, n):
        return int(self.ctx.lib.kz_transform_max_encoded_len(self.type, n))


class Writer:
    """io.Writer (CompressedOutputStream): NewWriter(os, transform, entropy, blockSize, jobs, checksum, fileSize, headerless)
    (io/CompressedStream.go:216). write() buffers, close() compresses everything that was written in one GPU batch
    (the reference cuts batches of `jobs` blocks; batches do not change the bytes) and returns nothing; the stream
    bytes are in .getvalue(). headerless=True writes no stream header: a HeaderlessReader with the same parameters reads it.
    skip_blocks=True is ctx["skipBlocks"] (kanzi c --skip): incompressible blocks are stored raw (Context.set_skip_blocks)."""

    def __init__(self, transform="NONE", entropy="NONE", block_size=4 << 20, jobs=1, checksum=0, file_size=0, ctx=None, headerless=False,
                 skip_blocks=False):
        if not (1 <= jobs <= 64):
            raise KanziError(18, "The number of jobs must be in [1..64], got %d" % jobs)
        if block_size > (1 << 30):
            raise KanziError(18, "The block size must be at most 1024 MB")
        if block_size < 1024:
            raise KanziError(18, "The block size must be at least 1024")
        if block_size & 15:
            raise KanziError(18, "The block size must be a multiple of 16")
        self.t48 = transform_type(transform)
        self.etype = entropy_type(entropy)
        self.block_size = block_size
        self.checksum = checksum
        self.file_size = file_size
        self.headerless = bool(headerless)
        self.skip_blocks = bool(skip_blocks)
        self.ctx = ctx or default_context()
        self._chunks = []
        self._out = None

    def write(self, block):
        if self._out is not None:
            raise KanziError(12, "Stream closed")
        self._chunks.append(np.array(_u8(block), copy=True))
        return len(block)

    def close(self):
        if self._out is None:
            data = np.concatenate(self._chunks) if self._chunks else np.zeros(0, np.uint8)
            self._out = self.ctx.compress(data, self.t48, self.etype, self.block_size, self.checksum, self.file_size, headerless=self.headerless,
                                          skip_blocks=self.skip_blocks)

    def getvalue(self):
        self.close()
        return self._out


class Reader:
    """io.Reader (CompressedInputStream): NewReader(is, jobs) (io/CompressedStream.go:1047); from_block / to_block are ctx["from"] /
    ctx["to"] of NewReaderWithCtx (negative = not given): only blocks from_block <= id < to_block are decoded."""

    def __init__(self, stream, jobs=1, ctx=None, from_block=-1, to_block=-1):
        self.stream = _u8(stream)
        self.ctx = ctx or default_context()
        self.from_block, self.to_block = from_block, to_block

    def read_all(self, max_size):
        return self.ctx.decompress(self.stream, max_size, self.from_block, self.to_block)


class HeaderlessReader(Reader):
    """io.Reader over a stream without header: NewHeaderlessReader(is, jobs, transform, entropy, blockSize, checksum, originalSize,
    bsVersion) (io/CompressedStream.go:1060). The parameters are checked here, as Reader.validateHeaderless does (:1178-1280); a bad
    one raises KanziError with the code of kz_set_headerless_reader. original_size < 0 or >= 2^48 means "not given"."""

    def __init__(self, stream, jobs=1, transform="NONE", entropy="NONE", block_size=4 << 20, checksum=0, original_size=0, bs_version=6, ctx=None,
                 from_block=-1, to_block=-1):
        super().__init__(stream, jobs, ctx, from_block, to_block)
        self.params = dict(transform=transform, entropy=entropy, block_size=block_size, checksum_bits=checksum, output_size=original_size,
                           bs_version=bs_version)
        with self.ctx._headerless(reader=self.params):
            pass

    def read_all(self, max_size):
        return self.ctx.decompress(self.stream, max_size, self.from_block, self.to_block, headerless=self.params)
