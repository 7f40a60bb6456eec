// Batch entry points: one cgo call per batch of blocks instead of one goroutine per block
// (io/CompressedStream.go:621-710 Writer.processBlock, :1614-1744 Reader.processBlock). Lives at v2/gpu/batch.go.
package gpu

/*
#include "kanzi_b200.h"
*/
import "C"

import (
	"fmt"
	"time"
	"unsafe"

	kanzi "github.com/flanglet/kanzi-go/v2"
	"github.com/flanglet/kanzi-go/v2/internal"
)

// EncodedBlock is what encodingTask.encode leaves behind for the ordered commit (:951-976).
type EncodedBlock struct {
	Bits []byte // block-local bit string, zero padded
	N    uint64 // "written" (:914)
}

// EncodeBlocks replaces the goroutine fan-out of Writer.processBlock (:658-701). slab holds nbTasks blocks of lens[i] bytes at a
// distance of stride bytes (the Writer's buffers are carved from one kz_alloc_pinned slab). The four listener events of every block
// (:766-771 before transform, :850-855 after transform, :889-894 before entropy, :916-932 after entropy) are emitted here with the
// batch's timestamps: the post-transform length and the checksum are read back from the head of each block's bit string
// (mode byte, optional skip-flag byte, length on 1..4 bytes, checksum; :869-886), so the ABI needs no extra outputs.
func (c *Context) EncodeBlocks(transformType uint64, entropyType uint32, ckBits uint, slab []byte, stride uint64, lens []uint32, firstBlockID int,
	listeners []kanzi.Listener) ([]EncodedBlock, error) {
	n := len(lens)
	maxLen := uint32(0)
	for _, l := range lens {
		if l > maxLen {
			maxLen = l
		}
	}
	outStride := uint64(C.kz_max_block_output(C.size_t(maxLen)))
	out := make([]byte, outStride*uint64(n))
	bits := make([]C.uint64_t, n)
	status := make([]C.int32_t, n)
	hashType := kanzi.EVT_HASH_NONE
	if ckBits == 32 {
		hashType = kanzi.EVT_HASH_32BITS
	} else if ckBits == 64 {
		hashType = kanzi.EVT_HASH_64BITS
	}
	t0 := time.Now()
	for i := 0; i < n && len(listeners) > 0; i++ { // the checksum is not known yet: the reference computes it before this event, here it follows
		notify(listeners, kanzi.NewEvent(kanzi.EVT_BEFORE_TRANSFORM, firstBlockID+i, int64(lens[i]), 0, kanzi.EVT_HASH_NONE, t0))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_encode_blocks(c.h, C.uint64_t(transformType), C.uint32_t(entropyType), C.uint32_t(ckBits),
		(*C.uint8_t)(unsafe.Pointer(&slab[0])), C.uint64_t(stride), (*C.uint32_t)(unsafe.Pointer(&lens[0])), C.uint32_t(n),
		(*C.uint8_t)(unsafe.Pointer(&out[0])), C.uint64_t(outStride), &bits[0], &status[0])
	if rc != 0 {
		return nil, c.err(rc)
	}
	t1 := time.Now()
	res := make([]EncodedBlock, n)
	for i := 0; i < n; i++ {
		if status[i] != 0 {
			return nil, c.err(C.int(status[i]))
		}
		b := out[uint64(i)*outStride : uint64(i+1)*outStride]
		res[i] = EncodedBlock{Bits: b, N: uint64(bits[i])}
		if len(listeners) == 0 {
			continue
		}
		post, ck := parseBlockHead(b, ckBits)
		notify(listeners, kanzi.NewEvent(kanzi.EVT_AFTER_TRANSFORM, firstBlockID+i, int64(post), ck, hashType, t1))
		notify(listeners, kanzi.NewEvent(kanzi.EVT_BEFORE_ENTROPY, firstBlockID+i, int64(post), ck, hashType, t1))
		notify(listeners, kanzi.NewEvent(kanzi.EVT_AFTER_ENTROPY, firstBlockID+i, int64((uint64(bits[i])+7)>>3), ck, hashType, t1))
	}
	return res, nil
}

// Commit is the ordered section of encodingTask.encode (:951-976), unchanged.
func Commit(obs kanzi.OutputBitStream, blocks []EncodedBlock) {
	for _, b := range blocks {
		lw := uint(3)
		if b.N >= 8 {
			lw = uint(internal.Log2NoCheck(uint32(b.N>>3)) + 4)
		}
		obs.WriteBits(uint64(lw-3), 5)
		obs.WriteBits(b.N, lw)
		obs.WriteArray(b.Bits, uint(b.N))
	}
}

// DecodeBlocks replaces the decode goroutines of Reader.processBlock: in holds the block bit strings extracted by the serial
// section (:1816-1852), byte aligned at off[i], bits[i] long.
func (c *Context) DecodeBlocks(transformType uint64, entropyType uint32, ckBits uint, in []byte, off, bits []uint64, blockSize uint32,
	out []byte, outStride uint64) ([]uint32, error) {
	n := len(off)
	outLen := make([]uint32, n)
	status := make([]C.int32_t, n)
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_decode_blocks(c.h, C.uint64_t(transformType), C.uint32_t(entropyType), C.uint32_t(ckBits), (*C.uint8_t)(unsafe.Pointer(&in[0])),
		(*C.uint64_t)(unsafe.Pointer(&off[0])), (*C.uint64_t)(unsafe.Pointer(&bits[0])), C.uint32_t(n), C.uint32_t(blockSize),
		(*C.uint8_t)(unsafe.Pointer(&out[0])), C.uint64_t(outStride), (*C.uint32_t)(unsafe.Pointer(&outLen[0])), &status[0])
	if rc != 0 {
		return nil, c.err(rc)
	}
	for i := 0; i < n; i++ {
		if status[i] != 0 {
			return nil, c.err(C.int(status[i]))
		}
	}
	return outLen, nil
}

// StreamResult is what one file of a many-stream call produced: the stream (or decoded bytes), or the kanzi error of that file alone.
type StreamResult struct {
	Data []byte
	Err  error
}

// CompressStreams compresses every input as a stream of its own in one call, as BlockCompressor's multi-file path
// (app/BlockCompressor.go:543-613) would use it instead of one Writer per file. Stream i is byte for byte what a Writer with
// the same parameters and fileSize = inputSizes[i] writes for inputs[i]. All inputs share one block size; with `-b auto`, where every
// file has its own, use CompressStreamsBlockSizes. A file whose output does not fit fails alone; a transform or
// entropy failure on one file's data (the reference fails that file with ERR_PROCESS_BLOCK) fails the whole call, and the caller
// then compresses the files one by one. The call holds all inputs, encoded blocks and streams in device memory at once: split a
// large directory into calls of a size the GPU holds. After c.SetHeaderlessWriter(true) no stream carries a header (the Writer's
// headerless = true): that saves 20 to 26 bytes per file for callers that store the parameters once.
func (c *Context) CompressStreams(transformType uint64, entropyType uint32, blockSize uint32, ckBits uint, inputs [][]byte,
	inputSizes []int64) ([]StreamResult, error) {
	n := len(inputs)
	srcOff, srcLen := make([]uint64, n), make([]uint64, n)
	dstOff, dstCap := make([]uint64, n), make([]uint64, n)
	var srcTotal, dstTotal uint64
	for i, in := range inputs {
		srcOff[i], srcLen[i] = srcTotal, uint64(len(in))
		srcTotal += uint64(len(in))
		dstOff[i], dstCap[i] = dstTotal, uint64(C.kz_max_stream_output(C.size_t(len(in)), C.uint32_t(blockSize)))
		dstTotal += dstCap[i]
	}
	src := make([]byte, srcTotal+1)
	for i, in := range inputs {
		copy(src[srcOff[i]:], in)
	}
	dst := make([]byte, dstTotal+1)
	outLen, status := make([]uint64, n+1), make([]C.int32_t, n+1)
	var isz *C.int64_t
	if len(inputSizes) == n && n > 0 {
		isz = (*C.int64_t)(unsafe.Pointer(&inputSizes[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_compress_streams(c.h, C.uint64_t(transformType), C.uint32_t(entropyType), C.uint32_t(blockSize), C.uint32_t(ckBits), C.uint32_t(n),
		(*C.uint8_t)(unsafe.Pointer(&src[0])), u64p(srcOff), u64p(srcLen), isz, (*C.uint8_t)(unsafe.Pointer(&dst[0])), u64p(dstOff), u64p(dstCap),
		u64p(outLen), &status[0])
	return c.streamResults(rc, dst, dstOff, outLen, status, n)
}

// CompressStreamsBlockSizes is CompressStreams with one block size per file: blockSizes[i] for inputs[i], as BlockCompressor's `-b auto`
// gives every file (app/BlockCompressor.go:574-580, AutoBlockSize). All files still share one call and its passes. A block size that a
// Writer refuses (outside [1 KiB, 1 GiB] or not a multiple of 16) fails only its own file, with ERR_INVALID_PARAM.
func (c *Context) CompressStreamsBlockSizes(transformType uint64, entropyType uint32, blockSizes []uint32, ckBits uint, inputs [][]byte,
	inputSizes []int64) ([]StreamResult, error) {
	n := len(inputs)
	if len(blockSizes) != n {
		return nil, fmt.Errorf("kanzi gpu: %d block sizes for %d inputs", len(blockSizes), n)
	}
	srcOff, srcLen := make([]uint64, n), make([]uint64, n)
	dstOff, dstCap := make([]uint64, n), make([]uint64, n)
	var srcTotal, dstTotal uint64
	for i, in := range inputs {
		srcOff[i], srcLen[i] = srcTotal, uint64(len(in))
		srcTotal += uint64(len(in))
		dstOff[i], dstCap[i] = dstTotal, uint64(C.kz_max_stream_output(C.size_t(len(in)), C.uint32_t(blockSizes[i])))
		dstTotal += dstCap[i]
	}
	src := make([]byte, srcTotal+1)
	for i, in := range inputs {
		copy(src[srcOff[i]:], in)
	}
	dst := make([]byte, dstTotal+1)
	outLen, status := make([]uint64, n+1), make([]C.int32_t, n+1)
	bs := make([]uint32, n+1)
	copy(bs, blockSizes)
	var isz *C.int64_t
	if len(inputSizes) == n && n > 0 {
		isz = (*C.int64_t)(unsafe.Pointer(&inputSizes[0]))
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_compress_streams_bs(c.h, C.uint64_t(transformType), C.uint32_t(entropyType), (*C.uint32_t)(unsafe.Pointer(&bs[0])), C.uint32_t(ckBits),
		C.uint32_t(n), (*C.uint8_t)(unsafe.Pointer(&src[0])), u64p(srcOff), u64p(srcLen), isz, (*C.uint8_t)(unsafe.Pointer(&dst[0])), u64p(dstOff),
		u64p(dstCap), u64p(outLen), &status[0])
	return c.streamResults(rc, dst, dstOff, outLen, status, n)
}

// AutoBlockSize is the block size BlockCompressor's `-b auto` gives a file of size bytes with jobs jobs (app/BlockCompressor.go:574-580).
func AutoBlockSize(size int64, jobs uint) uint32 {
	bl := size / int64(jobs)
	bl = (bl + 63) &^ 63
	bl = min(bl, 1<<30)
	bl = max(bl, 1024)
	return uint32(bl)
}

// DecompressStreams decodes many streams in one call, as BlockDecompressor's multi-file path would: the streams may have different
// headers (transform, entropy, block size, checksum), and streams that differ only in block size share one set of passes. caps[i]
// bounds the decoded size of stream i (the file size its header records, or the caller's limit). A corrupt stream gets the error code a Reader would report for it; every other stream decodes normally.
// A stream whose transform or entropy codec the GPU path lacks fails the whole call with ERR_INVALID_CODEC: the caller then keeps
// the reference's Reader for the files of that call. The device holds every input and sum(caps) bytes of output at once.
// After c.SetHeaderlessReader(...) the streams have no header and all share its parameters (NewHeaderlessReader for every file).
func (c *Context) DecompressStreams(streams [][]byte, caps []uint64) ([]StreamResult, error) {
	n := len(streams)
	srcOff, srcLen, dstOff := make([]uint64, n), make([]uint64, n), make([]uint64, n)
	var srcTotal, dstTotal uint64
	for i, s := range streams {
		srcOff[i], srcLen[i] = srcTotal, uint64(len(s))
		srcTotal += uint64(len(s))
		dstOff[i] = dstTotal
		dstTotal += caps[i]
	}
	src := make([]byte, srcTotal+1)
	for i, s := range streams {
		copy(src[srcOff[i]:], s)
	}
	dst := make([]byte, dstTotal+1)
	outLen, status := make([]uint64, n+1), make([]C.int32_t, n+1)
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_decompress_streams(c.h, C.uint32_t(n), (*C.uint8_t)(unsafe.Pointer(&src[0])), u64p(srcOff), u64p(srcLen),
		(*C.uint8_t)(unsafe.Pointer(&dst[0])), u64p(dstOff), u64p(caps), u64p(outLen), &status[0])
	return c.streamResults(rc, dst, dstOff, outLen, status, n)
}

// StreamError is the kanzi error code (Definitions.go:25-46) one file of a many-stream call failed with.
type StreamError struct {
	Code int
}

func (e *StreamError) Error() string {
	return fmt.Sprintf("kanzi gpu: stream failed with error code %d", e.Code)
}

// streamResults splits a many-stream call's output (called with mu held). Every file carries its own result: its bytes, or a
// StreamError with its own code. The returned error is nil when every file succeeded; otherwise it is the context's message for the
// call (kz_last_error) with the code of the first failing file. A call-level failure (a bad argument, an unsupported codec, a CUDA
// error) gives every file that same code.
func (c *Context) streamResults(rc C.int, dst []byte, dstOff, outLen []uint64, status []C.int32_t, n int) ([]StreamResult, error) {
	res := make([]StreamResult, n)
	for i := 0; i < n; i++ {
		if status[i] != 0 {
			res[i].Err = &StreamError{Code: -int(status[i])}
			continue
		}
		res[i].Data = dst[dstOff[i] : dstOff[i]+outLen[i]]
	}
	if rc != 0 {
		return res, fmt.Errorf("%v (code %d)", c.err(rc), -int(rc))
	}
	return res, nil
}

func u64p(a []uint64) *C.uint64_t {
	if len(a) == 0 {
		return nil
	}
	return (*C.uint64_t)(unsafe.Pointer(&a[0]))
}

// parseBlockHead reads post-transform length and checksum back from a block-local bit string (:869-886).
func parseBlockHead(b []byte, ckBits uint) (uint64, uint64) {
	mode := b[0]
	p := 1
	if mode&0x80 == 0 && mode&0x10 != 0 { // not a copy block, _TRANSFORMS_MASK: a skip-flag byte follows
		p++
	}
	dataSize := int((mode>>5)&3) + 1
	var post uint64
	for i := 0; i < dataSize; i++ {
		post = post<<8 | uint64(b[p+i])
	}
	p += dataSize
	var ck uint64
	for i := 0; i < int(ckBits/8); i++ {
		ck = ck<<8 | uint64(b[p+i])
	}
	return post, ck
}

func notify(listeners []kanzi.Listener, evt *kanzi.Event) {
	defer func() { _ = recover() }() // panics in block listeners are ignored (:979-991)
	for _, l := range listeners {
		l.ProcessEvent(evt)
	}
}
