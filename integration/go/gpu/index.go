// Stream index and batched range reads: bytes [off, off+len) of the original data without decoding the stream
// (kz_index_*, kz_read_ranges in kanzi_b200.h). The reference has no counterpart: its Reader decodes from the first block, and
// --from / --to (:1858-1871) selects whole blocks after walking every record. Lives at v2/gpu/index.go.
package gpu

/*
#include "kanzi_b200.h"
*/
import "C"

import (
	"errors"
	"io"
	"unsafe"
)

// Index says where every block record of one stream lies. It does not own the stream; Save's bytes are kept beside it.
type Index struct {
	h *C.kz_index
}

// BuildIndex parses the header of stream (or takes the headerless reader setting of c) and walks its records. Nothing is decoded.
func (c *Context) BuildIndex(stream []byte) (*Index, error) {
	if len(stream) == 0 {
		return nil, errors.New("gpu: empty stream")
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	var h *C.kz_index
	if rc := C.kz_index_build(c.h, (*C.uint8_t)(unsafe.Pointer(&stream[0])), C.size_t(len(stream)), &h); rc != 0 {
		return nil, c.err(rc)
	}
	return &Index{h: h}, nil
}

// LoadIndex reads an index from Save's bytes. It needs no GPU; a damaged blob is ERR_INVALID_FILE.
func LoadIndex(blob []byte) (*Index, error) {
	if len(blob) == 0 {
		return nil, errors.New("gpu: empty index blob")
	}
	var h *C.kz_index
	if rc := C.kz_index_load((*C.uint8_t)(unsafe.Pointer(&blob[0])), C.size_t(len(blob)), &h); rc != 0 {
		return nil, errors.New("gpu: not a stream index blob")
	}
	return &Index{h: h}, nil
}

// Save returns the self-describing blob of the index (layout in kanzi_b200.h).
func (x *Index) Save() []byte {
	n := C.kz_index_save(x.h, nil, 0)
	out := make([]byte, int(n))
	C.kz_index_save(x.h, (*C.uint8_t)(unsafe.Pointer(&out[0])), n)
	return out
}

// Size is the decoded length of the stream, or -1 until a read has decoded the last block.
func (x *Index) Size() int64 {
	var size C.int64_t
	C.kz_index_info(x.h, nil, nil, nil, nil, nil, nil, nil, &size)
	return int64(size)
}

// Free releases the index.
func (x *Index) Free() {
	C.kz_index_free(x.h)
	x.h = nil
}

// Range is one request of ReadRanges: Len decoded bytes from Off, delivered into Dst[:N]. Err is the request's own failure
// (a StreamError with the block's code); a request that runs past the end of the data is short, not failed.
type Range struct {
	Off uint64
	Dst []byte
	N   int
	Err error
}

// ReadRanges serves every request in one call: each block the requests touch is decoded once. The returned error is a failure of
// the call as a whole (a stale index, a session open on c, a chain the GPU path lacks); failures of single blocks, and a CUDA error,
// which sets every request's status, are in the requests' Err.
func (c *Context) ReadRanges(x *Index, stream []byte, reqs []Range) error {
	return c.readRanges(nil, x, stream, reqs)
}

// ReadRangesCached is ReadRanges through the block cache k of c (kz_read_ranges_cached): the same results, and the blocks k holds are
// copied instead of decoded. Blocks decoded here are kept in k for later calls.
func (c *Context) ReadRangesCached(k *Cache, x *Index, stream []byte, reqs []Range) error {
	if k == nil {
		return errors.New("gpu: nil block cache")
	}
	return c.readRanges(k, x, stream, reqs)
}

func (c *Context) readRanges(k *Cache, x *Index, stream []byte, reqs []Range) error {
	n := len(reqs)
	if n == 0 {
		return nil
	}
	off := make([]C.uint64_t, n)
	ln := make([]C.uint64_t, n)
	dstOff := make([]C.uint64_t, n)
	outLen := make([]C.uint64_t, n)
	status := make([]C.int32_t, n)
	total := uint64(0)
	for i, r := range reqs {
		off[i], ln[i], dstOff[i] = C.uint64_t(r.Off), C.uint64_t(len(r.Dst)), C.uint64_t(total)
		total += uint64(len(r.Dst))
	}
	buf := make([]byte, total+1) // cgo must not see pointers into several Go slices: one buffer, then copies
	c.mu.Lock()
	defer c.mu.Unlock()
	src, dst := (*C.uint8_t)(unsafe.Pointer(&stream[0])), (*C.uint8_t)(unsafe.Pointer(&buf[0]))
	var rc C.int
	if k == nil {
		rc = C.kz_read_ranges(c.h, x.h, src, C.size_t(len(stream)), C.uint32_t(n), &off[0], &ln[0], dst, &dstOff[0], &outLen[0], &status[0])
	} else {
		rc = C.kz_read_ranges_cached(c.h, k.h, x.h, src, C.size_t(len(stream)), C.uint32_t(n), &off[0], &ln[0], dst, &dstOff[0], &outLen[0], &status[0])
	}
	if rc == -C.KZ_ERR_INVALID_PARAM || rc == -C.KZ_ERR_CREATE_CODEC { // no block fails with these: the call failed as a whole
		return c.err(rc)
	}
	for i := range reqs {
		reqs[i].N, reqs[i].Err = int(outLen[i]), nil
		if status[i] != 0 {
			reqs[i].Err = &StreamError{Code: int(-status[i])}
			continue
		}
		copy(reqs[i].Dst, buf[uint64(dstOff[i]):uint64(dstOff[i])+uint64(outLen[i])])
	}
	return nil
}

// ReaderAt is an io.ReaderAt over the original data of (stream, index): every ReadAt is one kz_read_ranges call of one request.
// Callers with many reads in hand use ReadRanges, which decodes each touched block once for all of them. With Cache set (a cache of
// C), each ReadAt goes through it: reading a block in small pieces decodes it once instead of once per piece.
type ReaderAt struct {
	C      *Context
	Index  *Index
	Stream []byte
	Cache  *Cache
}

func (r *ReaderAt) ReadAt(p []byte, off int64) (int, error) {
	if off < 0 {
		return 0, errors.New("gpu: negative offset")
	}
	req := []Range{{Off: uint64(off), Dst: p}}
	if err := r.C.readRanges(r.Cache, r.Index, r.Stream, req); err != nil {
		return 0, err
	}
	if req[0].Err != nil {
		return 0, req[0].Err
	}
	if req[0].N < len(p) {
		return req[0].N, io.EOF
	}
	return req[0].N, nil
}

// Cache keeps decoded blocks in HBM between reads of one Context (kz_cache_*). Entries belong to the content of a block record, so one
// cache serves every stream and index read through it. Free it before the Context is closed.
type Cache struct {
	c *Context // its calls take the context's lock: reads on other goroutines update the counters and the context's cache list
	h *C.kz_cache
}

// CacheStats are the counters of a Cache (kz_cache_stats): what it holds, and what it did since it was made.
type CacheStats struct {
	Entries, ResidentBytes, BudgetBytes, Hits, Misses, Inserts, Evictions, ServedBytes uint64
}

// NewBlockCache allocates a cache of budget bytes of HBM (rounded down to 64 KiB pages) on c, once.
func (c *Context) NewBlockCache(budget uint64) (*Cache, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var h *C.kz_cache
	if rc := C.kz_cache_create(c.h, C.uint64_t(budget), &h); rc != 0 {
		return nil, c.err(rc)
	}
	return &Cache{c: c, h: h}, nil
}

func (k *Cache) Stats() CacheStats {
	k.c.mu.Lock()
	defer k.c.mu.Unlock()
	var v [8]C.uint64_t
	C.kz_cache_stats(k.h, &v[0], &v[1], &v[2], &v[3], &v[4], &v[5], &v[6], &v[7])
	return CacheStats{uint64(v[0]), uint64(v[1]), uint64(v[2]), uint64(v[3]), uint64(v[4]), uint64(v[5]), uint64(v[6]), uint64(v[7])}
}

// Free releases the cache and its device memory.
func (k *Cache) Free() {
	k.c.mu.Lock()
	defer k.c.mu.Unlock()
	C.kz_cache_free(k.h)
	k.h = nil
}

// BuildIndexes indexes many streams in one kz_index_build_streams call: index i is what BuildIndex(streams[i]) gives. A stream that
// fails has a nil index and its error in errs[i]; the returned error is a failure of the call as a whole (a session open on c).
func (c *Context) BuildIndexes(streams [][]byte) (idx []*Index, errs []error, err error) {
	n := len(streams)
	idx, errs = make([]*Index, n), make([]error, n)
	if n == 0 {
		return idx, errs, nil
	}
	off := make([]C.uint64_t, n)
	ln := make([]C.uint64_t, n)
	total := 0
	for i, s := range streams {
		off[i], ln[i] = C.uint64_t(total), C.uint64_t(len(s))
		total += len(s)
	}
	buf := make([]byte, total+1) // cgo must not see pointers into several Go slices: one buffer
	for i, s := range streams {
		copy(buf[int(off[i]):], s)
	}
	hs := make([]*C.kz_index, n)
	status := make([]C.int32_t, n)
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_index_build_streams(c.h, C.uint32_t(n), (*C.uint8_t)(unsafe.Pointer(&buf[0])), &off[0], &ln[0], &hs[0], &status[0])
	if rc == -C.KZ_ERR_INVALID_PARAM { // no stream fails with this code: the call failed as a whole
		return idx, errs, c.err(rc)
	}
	for i := range streams {
		if hs[i] != nil {
			idx[i] = &Index{h: hs[i]}
		} else {
			errs[i] = &StreamError{Code: int(-status[i])}
		}
	}
	return idx, errs, nil
}

// StreamRange is one request of ReadRangesStreams: a Range of stream Stream, an index into the streams and indexes of the call.
type StreamRange struct {
	Stream int
	Range
}

// ReadRangesStreams serves requests on many streams in one kz_read_ranges_streams call, through the block cache k when it is not nil.
// Each request gets what ReadRanges (or ReadRangesCached) gives it on its own stream. A nil or stale index, or a chain the GPU path
// lacks, fails only the requests on that stream; streams no request names are not read, so callers may pass their whole object table.
// The returned error is a failure of the call as a whole (a request on a stream out of range, a session open on c, a cache of another
// context); every request then holds it too.
func (c *Context) ReadRangesStreams(k *Cache, idx []*Index, streams [][]byte, reqs []StreamRange) error {
	n, ns := len(reqs), len(streams)
	if n == 0 {
		return nil
	}
	if len(idx) != ns {
		return errors.New("gpu: one index per stream")
	}
	named := make([]bool, ns)
	for _, r := range reqs {
		if r.Stream < 0 || r.Stream >= ns {
			return errors.New("gpu: request on a stream out of range")
		}
		named[r.Stream] = true
	}
	srcOff := make([]C.uint64_t, ns)
	srcLen := make([]C.uint64_t, ns)
	hs := make([]*C.kz_index, ns)
	total := 0
	for s, b := range streams {
		if idx[s] != nil {
			hs[s] = idx[s].h
		}
		if named[s] { // only the named streams are copied: the others are neither checked nor read
			srcOff[s], srcLen[s] = C.uint64_t(total), C.uint64_t(len(b))
			total += len(b)
		}
	}
	src := make([]byte, total+1)
	for s, b := range streams {
		if named[s] {
			copy(src[int(srcOff[s]):], b)
		}
	}
	rs := make([]C.uint32_t, n)
	off := make([]C.uint64_t, n)
	ln := make([]C.uint64_t, n)
	dstOff := make([]C.uint64_t, n)
	outLen := make([]C.uint64_t, n)
	status := make([]C.int32_t, n)
	dtotal := uint64(0)
	for i, r := range reqs {
		rs[i], off[i], ln[i], dstOff[i] = C.uint32_t(r.Stream), C.uint64_t(r.Off), C.uint64_t(len(r.Dst)), C.uint64_t(dtotal)
		dtotal += uint64(len(r.Dst))
	}
	dst := make([]byte, dtotal+1)
	var kh *C.kz_cache
	if k != nil {
		kh = k.h
	}
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.kz_read_ranges_streams(c.h, kh, C.uint32_t(ns), &hs[0], (*C.uint8_t)(unsafe.Pointer(&src[0])), &srcOff[0], &srcLen[0], C.uint32_t(n), &rs[0],
		&off[0], &ln[0], (*C.uint8_t)(unsafe.Pointer(&dst[0])), &dstOff[0], &outLen[0], &status[0])
	whole := rc != 0
	for i := range reqs {
		reqs[i].N, reqs[i].Err = int(outLen[i]), nil
		if status[i] != rc {
			whole = false
		}
		if status[i] != 0 {
			reqs[i].Err = &StreamError{Code: int(-status[i])}
			continue
		}
		copy(reqs[i].Dst, dst[uint64(dstOff[i]):uint64(dstOff[i])+uint64(outLen[i])])
	}
	if whole && rc == -C.KZ_ERR_INVALID_PARAM {
		return c.err(rc)
	}
	return nil
}

// Write is one write of WriteRanges: Data at decoded offset Off, or at the current end of the data when Append is set.
type Write struct {
	Off    uint64
	Append bool
	Data   []byte
}

// WriteRanges applies writes in order to the data of (stream, x) with pwrite semantics (a later write wins where writes overlap, a
// write past the end grows the data and the gap reads as zeros) and re-encodes only the blocks they touch (kz_write_ranges). The new
// stream is stream[:keep] followed by tail, what a Writer with the stream's parameters writes for the new data; x then describes it.
// On error x and stream are unchanged.
func (c *Context) WriteRanges(x *Index, stream []byte, writes []Write) (keep int, tail []byte, err error) {
	if len(stream) == 0 {
		return 0, nil, errors.New("gpu: empty stream")
	}
	n := len(writes)
	off := make([]C.uint64_t, n+1)
	ln := make([]C.uint64_t, n+1)
	dataOff := make([]C.uint64_t, n+1)
	total := 0
	for i, w := range writes {
		off[i], ln[i], dataOff[i] = C.uint64_t(w.Off), C.uint64_t(len(w.Data)), C.uint64_t(total)
		if w.Append {
			off[i] = C.KZ_WRITE_APPEND
		}
		total += len(w.Data)
	}
	data := make([]byte, total+1) // one buffer for cgo, as in readRanges
	for i, w := range writes {
		copy(data[int(dataOff[i]):], w.Data)
	}
	var bs C.uint32_t
	C.kz_index_info(x.h, nil, nil, &bs, nil, nil, nil, nil, nil)
	blocks := 0
	for _, w := range writes {
		if len(w.Data) > 0 {
			blocks += len(w.Data)/int(bs) + 2
		}
	}
	capacity := len(stream) + blocks*int(C.kz_max_block_output(C.size_t(bs))) + 16
	c.mu.Lock()
	defer c.mu.Unlock()
	for {
		dst := make([]byte, capacity+1)
		var k C.uint64_t
		var outN C.size_t
		rc := C.kz_write_ranges(c.h, x.h, (*C.uint8_t)(unsafe.Pointer(&stream[0])), C.size_t(len(stream)), C.uint32_t(n), &off[0], &ln[0],
			(*C.uint8_t)(unsafe.Pointer(&data[0])), &dataOff[0], (*C.uint8_t)(unsafe.Pointer(&dst[0])), C.size_t(capacity), &k, &outN)
		if rc == -C.KZ_ERR_WRITE_FILE && int(outN) > capacity { // a zero gap added blocks: the call names the capacity it needs
			capacity = int(outN)
			continue
		}
		if rc != 0 {
			return 0, nil, c.err(rc)
		}
		return int(k), dst[:int(outN)], nil
	}
}

// Append writes p behind the end of the data of (stream, x): WriteRanges with one appending write.
func (c *Context) Append(x *Index, stream []byte, p []byte) (keep int, tail []byte, err error) {
	return c.WriteRanges(x, stream, []Write{{Append: true, Data: p}})
}

// StreamWrite is one write of WriteRangesStreams: a Write on stream Stream.
type StreamWrite struct {
	Stream int
	Write
}

// StreamTail is what WriteRangesStreams gives one stream: the new stream is stream[:Keep] followed by Tail, as WriteRanges gives it, or
// Err when that stream failed (its index and bytes are unchanged). A stream no write names keeps Keep = len(stream) and an empty Tail.
type StreamTail struct {
	Keep int
	Tail []byte
	Err  error
}

// WriteRangesStreams applies writes to many streams in one kz_write_ranges_streams call: each stream gets what WriteRanges gives it for
// its own writes, in order, and idx[s] then describes its new stream. A nil or stale index, a chain the GPU path lacks, a block that
// fails to decode or a data size past what an index holds fails only that stream; streams no write names are not read, so callers may
// pass their whole object table. A stream whose tail did not fit is written again alone with the capacity the call named. The returned
// error is a failure of the call as a whole (a write on a stream out of range, one index in two written slots, a session open on c, an
// encode failure), in which case no index changed. The call carries one extra slot that no write names: the library sets its status only
// when the whole call fails, which tells such a failure from every named stream failing with the same code.
func (c *Context) WriteRangesStreams(idx []*Index, streams [][]byte, writes []StreamWrite) ([]StreamTail, error) {
	ns, n := len(streams), len(writes)
	if len(idx) != ns {
		return nil, errors.New("gpu: one index per stream")
	}
	out := make([]StreamTail, ns)
	for s, b := range streams {
		out[s].Keep = len(b)
	}
	if ns == 0 || n == 0 {
		return out, nil
	}
	named := make([]bool, ns)
	blocks := make([]int, ns)
	for _, w := range writes {
		if w.Stream < 0 || w.Stream >= ns {
			return nil, errors.New("gpu: write on a stream out of range")
		}
		if len(w.Data) > 0 {
			named[w.Stream] = true
		}
	}
	// one slot more than the streams, named by no write: only a failure of the whole call sets its status
	srcOff := make([]C.uint64_t, ns+1)
	srcLen := make([]C.uint64_t, ns+1)
	dstCap := make([]C.uint64_t, ns+1)
	hs := make([]*C.kz_index, ns+1)
	total := 0
	for s, b := range streams {
		if idx[s] != nil {
			hs[s] = idx[s].h
		}
		if named[s] { // only the named streams are copied: the others are neither checked nor read
			srcOff[s], srcLen[s] = C.uint64_t(total), C.uint64_t(len(b))
			total += len(b)
		}
	}
	src := make([]byte, total+1)
	for s, b := range streams {
		if named[s] {
			copy(src[int(srcOff[s]):], b)
		}
	}
	ws := make([]C.uint32_t, n)
	off := make([]C.uint64_t, n)
	ln := make([]C.uint64_t, n)
	dataOff := make([]C.uint64_t, n)
	dtotal := 0
	for i, w := range writes {
		ws[i], off[i], ln[i], dataOff[i] = C.uint32_t(w.Stream), C.uint64_t(w.Off), C.uint64_t(len(w.Data)), C.uint64_t(dtotal)
		if w.Append {
			off[i] = C.KZ_WRITE_APPEND
		}
		dtotal += len(w.Data)
	}
	data := make([]byte, dtotal+1)
	for i, w := range writes {
		copy(data[int(dataOff[i]):], w.Data)
	}
	// WriteRanges's capacity per stream: len(stream) + k * kz_max_block_output(block_size) + 16, k bounded by the blocks the writes span
	for _, w := range writes {
		if len(w.Data) > 0 && idx[w.Stream] != nil {
			var bs C.uint32_t
			C.kz_index_info(idx[w.Stream].h, nil, nil, &bs, nil, nil, nil, nil, nil)
			blocks[w.Stream] += len(w.Data)/int(bs) + 2
			dstCap[w.Stream] = C.uint64_t(len(streams[w.Stream]) + blocks[w.Stream]*int(C.kz_max_block_output(C.size_t(bs))) + 16)
		}
	}
	keep := make([]C.uint64_t, ns+1)
	outN := make([]C.uint64_t, ns+1)
	status := make([]C.int32_t, ns+1)
	c.mu.Lock()
	defer c.mu.Unlock()
	for {
		dstOff := make([]C.uint64_t, ns+1)
		dcap := uint64(0)
		for s := range streams {
			dstOff[s] = C.uint64_t(dcap)
			dcap += uint64(dstCap[s])
		}
		dst := make([]byte, dcap+1)
		rc := C.kz_write_ranges_streams(c.h, C.uint32_t(ns+1), &hs[0], (*C.uint8_t)(unsafe.Pointer(&src[0])), &srcOff[0], &srcLen[0], C.uint32_t(n),
			&ws[0], &off[0], &ln[0], (*C.uint8_t)(unsafe.Pointer(&data[0])), &dataOff[0], (*C.uint8_t)(unsafe.Pointer(&dst[0])), &dstOff[0],
			&dstCap[0], &keep[0], &outN[0], &status[0])
		if status[ns] != 0 { // the call failed as a whole: no index changed
			return nil, c.err(rc)
		}
		// a stream whose tail did not fit keeps its index unchanged: it alone is written again, with the capacity the call named
		var again []int
		for s := range streams {
			if !named[s] {
				continue
			}
			if status[s] == -C.KZ_ERR_WRITE_FILE && outN[s] > dstCap[s] {
				dstCap[s] = outN[s]
				again = append(again, s)
				continue
			}
			out[s] = StreamTail{Keep: int(keep[s])}
			if status[s] != 0 {
				out[s].Keep, out[s].Err = len(streams[s]), &StreamError{Code: int(-status[s])}
				continue
			}
			out[s].Tail = append([]byte(nil), dst[uint64(dstOff[s]):uint64(dstOff[s])+uint64(outN[s])]...)
		}
		if len(again) == 0 {
			return out, nil
		}
		retry := make([]bool, ns)
		for _, s := range again {
			retry[s] = true
		}
		for s := range streams {
			named[s] = retry[s]
			if !retry[s] {
				dstCap[s] = 0
			}
		}
		ws, off, ln, dataOff = ws[:0], off[:0], ln[:0], dataOff[:0]
		dtotal = 0
		var left []StreamWrite
		for _, w := range writes {
			if !retry[w.Stream] {
				continue
			}
			o := C.uint64_t(w.Off)
			if w.Append {
				o = C.KZ_WRITE_APPEND
			}
			ws, off, ln = append(ws, C.uint32_t(w.Stream)), append(off, o), append(ln, C.uint64_t(len(w.Data)))
			dataOff = append(dataOff, C.uint64_t(dtotal))
			dtotal += len(w.Data)
			left = append(left, w)
		}
		writes, n = left, len(left)
		data = make([]byte, dtotal+1)
		for i, w := range writes {
			copy(data[int(dataOff[i]):], w.Data)
		}
	}
}
