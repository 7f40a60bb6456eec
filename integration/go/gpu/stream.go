// Streaming sessions: an io.WriteCloser / io.Reader over kz_writer_* / kz_reader_*, for a stream of any length or one that arrives from a
// pipe, in device and pinned memory that follows batchBlocks x blockSize, not the stream's length (the shape of CompressedOutputStream /
// CompressedInputStream, io/CompressedStream.go:524-710, :1556-1744). Lives at v2/gpu/stream.go. Not compiled (no Go toolchain here).
package gpu

/*
#include "kanzi_b200.h"
*/
import "C"

import (
	"io"
	"unsafe"
)

const streamBufSize = 4 << 20 // bytes handed to / taken from the pump per call

// StreamWriter compresses everything written to it into w. The session holds c until Close: make no other call on c meanwhile.
type StreamWriter struct {
	c      *Context
	w      io.Writer
	h      *C.kz_writer
	out    []byte
	closed bool
}

// NewStreamWriter opens a writer session: the bytes written to w are what CompressStream writes for the whole input with the same
// parameters. batchBlocks in [1..1024] is the role of kanzi's jobs; 0 takes about 256 MiB per batch.
func NewStreamWriter(c *Context, w io.Writer, transformType uint64, entropyType uint32, blockSize uint32, ckBits uint, batchBlocks uint32,
	inputSizeHint int64) (*StreamWriter, error) {
	if batchBlocks == 0 {
		batchBlocks = uint32(max(1, min(1024, (256<<20)/int(blockSize))))
	}
	c.mu.Lock() // held until Close: the session owns the context
	var h *C.kz_writer
	rc := C.kz_writer_open(c.h, C.uint64_t(transformType), C.uint32_t(entropyType), C.uint32_t(blockSize), C.uint32_t(ckBits),
		C.uint32_t(batchBlocks), C.int64_t(inputSizeHint), &h)
	if rc != 0 {
		err := c.err(rc)
		c.mu.Unlock()
		return nil, err
	}
	return &StreamWriter{c: c, w: w, h: h, out: make([]byte, streamBufSize)}, nil
}

func (s *StreamWriter) Write(p []byte) (int, error) {
	n := 0
	for n < len(p) {
		var used, made C.size_t
		rc := C.kz_writer_write(s.h, (*C.uint8_t)(unsafe.Pointer(&p[n])), C.size_t(len(p)-n), &used, (*C.uint8_t)(unsafe.Pointer(&s.out[0])),
			C.size_t(len(s.out)), &made)
		if rc != 0 {
			return n, s.c.err(rc)
		}
		n += int(used)
		if made > 0 {
			if _, err := s.w.Write(s.out[:made]); err != nil {
				return n, err
			}
		}
	}
	return n, nil
}

// Close writes the last block and the end marker, then frees the session and gives c back.
func (s *StreamWriter) Close() error {
	if s.closed {
		return nil
	}
	s.closed = true
	defer s.c.mu.Unlock()
	defer C.kz_writer_free(s.h)
	for {
		var made C.size_t
		rc := C.kz_writer_finish(s.h, (*C.uint8_t)(unsafe.Pointer(&s.out[0])), C.size_t(len(s.out)), &made)
		if rc < 0 {
			return s.c.err(rc)
		}
		if made > 0 {
			if _, err := s.w.Write(s.out[:made]); err != nil {
				return err
			}
		}
		if rc == 0 {
			return nil
		}
	}
}

// StreamReader decompresses the stream read from r. The session holds c until the end of the stream or Close. It feeds input only while
// no decoded bytes are pending, so its own memory stays at two 4 MiB buffers whatever the compression ratio.
type StreamReader struct {
	c          *Context
	r          io.Reader
	h          *C.kz_reader
	in, out    []byte
	inOff, inN int    // s.in[inOff:inN] is read from r and not yet consumed by the session
	pending    []byte // decoded bytes not yet returned (a slice of s.out)
	inEOF      bool
	finished   bool
	err        error
}

// NewStreamReader opens a reader session. batchBlocks in [1..1024]; 0 takes about 256 MiB per batch once the stream's block size is known.
// The session decodes the block range last set with SetBlockRange (all blocks by default).
func NewStreamReader(c *Context, r io.Reader, batchBlocks uint32) (*StreamReader, error) {
	c.mu.Lock()
	var h *C.kz_reader
	rc := C.kz_reader_open(c.h, C.uint32_t(batchBlocks), &h)
	if rc != 0 {
		err := c.err(rc)
		c.mu.Unlock()
		return nil, err
	}
	return &StreamReader{c: c, r: r, h: h, in: make([]byte, streamBufSize), out: make([]byte, streamBufSize)}, nil
}

func (s *StreamReader) Read(p []byte) (int, error) {
	for len(s.pending) == 0 {
		if s.err != nil {
			return 0, s.err
		}
		if s.finished {
			return 0, io.EOF
		}
		var made C.size_t
		if s.inOff < s.inN {
			var used C.size_t
			rc := C.kz_reader_read(s.h, (*C.uint8_t)(unsafe.Pointer(&s.in[s.inOff])), C.size_t(s.inN-s.inOff), &used,
				(*C.uint8_t)(unsafe.Pointer(&s.out[0])), C.size_t(len(s.out)), &made)
			if rc != 0 {
				s.fail(rc)
				return 0, s.err
			}
			s.inOff += int(used)
			s.pending = s.out[:made]
			continue
		}
		if !s.inEOF {
			k, err := s.r.Read(s.in)
			if err == io.EOF {
				s.inEOF = true
			} else if err != nil {
				return 0, err
			}
			s.inOff, s.inN = 0, k
			continue
		}
		rc := C.kz_reader_finish(s.h, (*C.uint8_t)(unsafe.Pointer(&s.out[0])), C.size_t(len(s.out)), &made)
		if rc < 0 {
			s.fail(rc)
			return 0, s.err
		}
		s.pending = s.out[:made]
		if rc == 0 {
			s.finished = true
			s.Close()
		}
	}
	n := copy(p, s.pending)
	s.pending = s.pending[n:]
	return n, nil
}

func (s *StreamReader) fail(rc C.int) {
	s.err = s.c.err(rc)
	s.Close()
}

// Close frees the session (also in the middle of the stream) and gives c back.
func (s *StreamReader) Close() error {
	if s.h != nil {
		C.kz_reader_free(s.h)
		s.h = nil
		s.c.mu.Unlock()
	}
	return nil
}

// BlockRange reads kanzi's ctx["from"] / ctx["to"], which NewReaderWithCtx checks to be ints (io/CompressedStream.go:1149-1159) and
// BlockDecompressor sets only when they are >= 0 (app/BlockDecompressor.go:411-417). A missing key gives -1, "not given".
func BlockRange(ctx map[string]any) (from, to int64) {
	from, to = -1, -1
	if v, ok := ctx["from"].(int); ok {
		from = int64(v)
	}
	if v, ok := ctx["to"].(int); ok {
		to = int64(v)
	}
	return from, to
}

// SetBlockRange is kz_set_block_range: the stream-level decodes that follow on c (DecompressStreams, and NewStreamReader, which keeps
// the range for its session) decode only the blocks with from <= id < to, ids counted from 1; a negative bound is not given.
func (c *Context) SetBlockRange(from, to int64) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.kz_set_block_range(c.h, C.int64_t(from), C.int64_t(to)); rc != 0 {
		return c.err(rc)
	}
	return nil
}

// NewStreamReaderWithCtx is NewStreamReader for the reader paths that carry a kanzi ctx (NewReaderWithCtx): the session decodes the
// block range of ctx["from"] / ctx["to"]. c's range is set for the open and restored to "not given" afterwards.
func NewStreamReaderWithCtx(c *Context, r io.Reader, batchBlocks uint32, ctx map[string]any) (*StreamReader, error) {
	from, to := BlockRange(ctx)
	if from < 0 && to < 0 {
		return NewStreamReader(c, r, batchBlocks)
	}
	if err := c.SetBlockRange(from, to); err != nil {
		return nil, err
	}
	s, err := NewStreamReader(c, r, batchBlocks)
	C.kz_set_block_range(c.h, -1, -1) // without c.mu, which the open session holds: the call is allowed while a session is open
	return s, err
}

// Headerless reads kanzi's ctx["headerless"], which NewWriterWithCtx checks to be a bool (io/CompressedStream.go:366) and
// NewHeaderlessReader sets to true (:1060). A missing key gives false.
func Headerless(ctx map[string]any) bool {
	v, ok := ctx["headerless"].(bool)
	return ok && v
}

// SetHeaderlessWriter is kz_set_headerless_writer: the stream-level encodes that follow on c (CompressStreams, and NewStreamWriter, which
// keeps the setting for its session) write no stream header, as Writer.writeHeader does for NewWriter(..., headerless = true) (:430).
func (c *Context) SetHeaderlessWriter(on bool) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	v := C.int(0)
	if on {
		v = 1
	}
	if rc := C.kz_set_headerless_writer(c.h, v); rc != 0 {
		return c.err(rc)
	}
	return nil
}

// SetHeaderlessReader is kz_set_headerless_reader: the stream-level decodes that follow on c (DecompressStreams, and NewStreamReader,
// which keeps the setting for its session) read no header and take these parameters. They are checked as Reader.validateHeaderless
// checks them (:1178-1280); a kanzi chain or codec the GPU lacks fails with ERR_CREATE_CODEC, and the caller keeps its CPU reader.
func (c *Context) SetHeaderlessReader(transformType uint64, entropyType uint32, blockSize uint32, ckBits uint, outputSize int64, bsVersion uint) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.kz_set_headerless_reader(c.h, C.uint64_t(transformType), C.uint32_t(entropyType), C.uint32_t(blockSize), C.uint32_t(ckBits),
		C.int64_t(outputSize), C.uint32_t(bsVersion)); rc != 0 {
		return c.err(rc)
	}
	return nil
}

// ClearHeaderlessReader turns the headerless reader setting off: the stream-level decodes read a header again.
func (c *Context) ClearHeaderlessReader() error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if rc := C.kz_clear_headerless_reader(c.h); rc != 0 {
		return c.err(rc)
	}
	return nil
}

// NewHeaderlessStreamReader is NewStreamReader for NewHeaderlessReader(is, jobs, transform, entropy, blockSize, checksum, originalSize,
// bsVersion) (:1060): the session reads a stream without header, with these parameters. c's setting is made for the open and cleared
// afterwards.
func NewHeaderlessStreamReader(c *Context, r io.Reader, batchBlocks uint32, transformType uint64, entropyType uint32, blockSize uint32,
	ckBits uint, originalSize int64, bsVersion uint) (*StreamReader, error) {
	if err := c.SetHeaderlessReader(transformType, entropyType, blockSize, ckBits, originalSize, bsVersion); err != nil {
		return nil, err
	}
	s, err := NewStreamReader(c, r, batchBlocks)
	C.kz_clear_headerless_reader(c.h) // without c.mu, which the open session holds: the call is allowed while a session is open
	return s, err
}
