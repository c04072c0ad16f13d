// cgo binding of include/ctmr_frontend.h: the CT wire-format front end (SURVEY.md §8(f)-2).
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain.  This is what a maintainer of
// jcjones/ct-mapreduce adds next to go/ctmr/ctmr.go to let the downloader hand get-entries bodies to the GPU
// instead of running ct.LogEntryFromLeaf per entry (cmd/ct-fetch/ct-fetch.go:446-484).
package ctmr

/*
#include <stdlib.h>
#include <string.h>
#include "ctmr_frontend.h"
*/
import "C"

import (
	"bytes"
	"encoding/base64"
	"encoding/json"
	"errors"
	"fmt"
	"runtime"
	"unsafe"
)

// EntryStatus mirrors CTMR_FE_*.
type EntryStatus uint8

const (
	FeOK EntryStatus = iota
	FeBadBase64
	FeBadLeaf
	FeUnknownType
	FeBadExtra
	FeBadCert
)

// RawPages accumulates get-entries response bodies in pinned memory (ctmr_host_alloc) together with the
// spans of their leaf_input / extra_data strings.  The downloader appends each body as it arrives
// (after LogClient's HTTP GET, before any JSON decoding) and flushes with DB.ProcessRaw.
type RawPages struct {
	Text      unsafe.Pointer // pinned, Cap bytes
	Cap, Used uint64
	LeafOff   []uint64
	LeafLen   []uint32
	ExtraOff  []uint64
	ExtraLen  []uint32
	Log       []uint32 // the log of each entry, for ProcessRawTrees (tree.go); NoTree for entries of Append
}

var (
	leafKey  = []byte(`"leaf_input":"`)
	extraKey = []byte(`"extra_data":"`)
)

// Append copies one response body into the pinned text and records its string spans.  A body whose
// strings carry JSON escapes (no CT log emits any) must be unescaped by the caller first.  Its entries belong to no
// tree (AppendLog).
func (p *RawPages) Append(body []byte) error {
	return p.AppendLog(body, NoTree)
}

// AppendLog is Append for a body of log `log`: ProcessRawTrees folds its entries into trees[log].
func (p *RawPages) AppendLog(body []byte, log uint32) error {
	if p.Used+uint64(len(body)) > p.Cap {
		return fmt.Errorf("raw page buffer full")
	}
	dst := unsafe.Slice((*byte)(unsafe.Add(p.Text, p.Used)), len(body))
	copy(dst, body)
	scan := func(key []byte, offs *[]uint64, lens *[]uint32) error {
		for at := 0; ; {
			i := bytes.Index(body[at:], key)
			if i < 0 {
				return nil
			}
			start := at + i + len(key)
			end := bytes.IndexByte(body[start:], '"')
			if end < 0 || bytes.IndexByte(body[start:start+end], '\\') >= 0 {
				return fmt.Errorf("malformed or escaped base64 string at %d", start)
			}
			*offs = append(*offs, p.Used+uint64(start))
			*lens = append(*lens, uint32(end))
			at = start + end
		}
	}
	if err := scan(leafKey, &p.LeafOff, &p.LeafLen); err != nil {
		return err
	}
	if err := scan(extraKey, &p.ExtraOff, &p.ExtraLen); err != nil {
		return err
	}
	if len(p.LeafOff) != len(p.ExtraOff) {
		return fmt.Errorf("get-entries body with %d leaf_input and %d extra_data strings", len(p.LeafOff), len(p.ExtraOff))
	}
	for len(p.Log) < len(p.LeafOff) {
		p.Log = append(p.Log, log)
	}
	p.Used += uint64(len(body))
	return nil
}

// RawResult holds the per-entry outputs of ProcessRaw (ctmr_raw_out).  Like Result, every array C writes lives in
// pinned C memory and the pointer table on the C heap (cgo: no Go pointer to memory holding Go pointers).
type RawResult struct {
	*Result                // the path's outputs, as for ProcessBatch
	raw                    *C.ctmr_raw_out
	EntryStatus, EntryType []uint8
	TimestampMs            []uint64
	Issuer                 []uint32
	LeafSrc                []uint8
	LeafOff, LeafLen       []uint32
}

func NewRawResult(n int, textBytes uint64) *RawResult {
	r := &RawResult{Result: NewResult(n, textBytes/4*3)}
	r.raw = (*C.ctmr_raw_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_raw_out{}))))
	C.memcpy(unsafe.Pointer(&r.raw.path), unsafe.Pointer(r.Result.out), C.size_t(unsafe.Sizeof(C.ctmr_out{}))) // C pointers only
	var p unsafe.Pointer
	p, r.EntryStatus = view[uint8](r.Result, n)
	r.raw.entry_status = (*C.uint8_t)(p)
	p, r.EntryType = view[uint8](r.Result, n)
	r.raw.entry_type = (*C.uint8_t)(p)
	p, r.TimestampMs = view[uint64](r.Result, n)
	r.raw.timestamp_ms = (*C.uint64_t)(p)
	p, r.Issuer = view[uint32](r.Result, n)
	r.raw.issuer = (*C.uint32_t)(p)
	p, r.LeafSrc = view[uint8](r.Result, n)
	r.raw.leaf_src = (*C.uint8_t)(p)
	p, r.LeafOff = view[uint32](r.Result, n)
	r.raw.leaf_off = (*C.uint32_t)(p)
	p, r.LeafLen = view[uint32](r.Result, n)
	r.raw.leaf_len = (*C.uint32_t)(p)
	return r
}

func (r *RawResult) Free() {
	C.free(unsafe.Pointer(r.raw))
	r.raw = nil
	r.Result.Free()
}

// ProcessRaw = GetRawEntries' base64 decode + ct.LogEntryFromLeaf + insertCTWorker + Store decisions for
// every entry of the accumulated pages, in page order, on one GPU or on every GPU of the group.
func (d *DB) ProcessRaw(p *RawPages, nowUnixNs int64, r *RawResult) error {
	return d.processRaw(p, nowUnixNs, r, nil, nil, false)
}

// processRaw also folds the entries into tree when it is not nil (ProcessRawTree, tree.go), or, when routed, each entry
// into trees[p.Log[i]] (ProcessRawTrees), on one GPU or on every GPU of the group.
func (d *DB) processRaw(p *RawPages, nowUnixNs int64, r *RawResult, tree *Tree, trees []Tree, routed bool) error {
	n := len(p.LeafOff)
	if n == 0 && tree == nil && !routed && !d.peer {
		return nil
	}
	b := (*C.ctmr_raw_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_raw_batch{}))))
	defer C.free(unsafe.Pointer(b))
	if n == 0 { // the roots of the trees as they stand; a peer DB's empty part of a collective call
		return d.rawCall(b, r, nil, tree, trees, routed)
	}
	// the span arrays are flat Go slices; the struct that points at them is C memory, and the pointers are only
	// stored for the duration of the call -> pin them (Go 1.21 runtime.Pinner) so that the store is legal
	var pin runtime.Pinner
	defer pin.Unpin()
	pin.Pin(&p.LeafOff[0])
	pin.Pin(&p.LeafLen[0])
	pin.Pin(&p.ExtraOff[0])
	pin.Pin(&p.ExtraLen[0])
	b.text = (*C.uint8_t)(p.Text)
	b.text_bytes = C.uint64_t(p.Used)
	b.leaf_input_off = (*C.uint64_t)(unsafe.Pointer(&p.LeafOff[0]))
	b.leaf_input_len = (*C.uint32_t)(unsafe.Pointer(&p.LeafLen[0]))
	b.extra_data_off = (*C.uint64_t)(unsafe.Pointer(&p.ExtraOff[0]))
	b.extra_data_len = (*C.uint32_t)(unsafe.Pointer(&p.ExtraLen[0]))
	b.n = C.uint64_t(n)
	b.now_unix_ns = C.int64_t(nowUnixNs)
	var log *C.uint32_t
	if routed {
		if len(p.Log) != n {
			return d.peerRefuse(fmt.Errorf("ProcessRawTrees: %d log ids for %d entries", len(p.Log), n))
		}
		log = (*C.uint32_t)(unsafe.Pointer(&p.Log[0])) // pointer-free Go memory, passed for the call only
	}
	return d.rawCall(b, r, log, tree, trees, routed)
}

// rawCall makes the plain, one-tree or routed call on the ctx, or on the group (several GPUs: one chunk per GPU per
// round, the same outputs in entry order and the same trees).
func (d *DB) rawCall(b *C.ctmr_raw_batch, r *RawResult, log *C.uint32_t, tree *Tree, trees []Tree, routed bool) error {
	switch {
	case routed && d.g != nil:
		return d.err(C.ctmr_group_process_raw_trees(d.g, b, r.raw, log, treesC(trees), C.uint32_t(len(trees))), "ctmr_group_process_raw_trees")
	case routed:
		return d.err(C.ctmr_process_raw_trees(d.h, b, r.raw, log, treesC(trees), C.uint32_t(len(trees))), "ctmr_process_raw_trees")
	case tree != nil && d.g != nil:
		return d.err(C.ctmr_group_process_raw_tree(d.g, b, r.raw, tree.c()), "ctmr_group_process_raw_tree")
	case tree != nil:
		return d.err(C.ctmr_process_raw_tree(d.h, b, r.raw, tree.c()), "ctmr_process_raw_tree")
	case d.g != nil:
		return d.err(C.ctmr_group_process_raw(d.g, b, r.raw), "ctmr_group_process_raw")
	}
	return d.err(C.ctmr_process_raw(d.h, b, r.raw), "ctmr_process_raw")
}

// ---- whole response bodies (ctmr_process_raw_bodies) -----------------------------------------------------------------

// BodyStatus mirrors CTMR_BODY_*.
type BodyStatus uint8

const (
	BodyOK BodyStatus = iota
	BodyBadJSON
	BodyBadType
	BodyTooMany
	BodyRepeatedEntries
)

// RawBodies accumulates whole get-entries response bodies in pinned memory (ctmr_host_alloc).  Nothing is scanned on
// the host: the GPU validates each body and finds its entries (DB.ProcessRawBodies).
type RawBodies struct {
	Text      unsafe.Pointer // pinned, Cap bytes
	Cap, Used uint64
	BodyOff   []uint64
	BodyLen   []uint32
	BodyMax   []uint32
	Start     []uint64 // the start of each body's get-entries request, for ProcessRawBodiesTree(s) (tree.go); 0 for Commit
	Log       []uint32 // the log of each body, for ProcessRawBodiesTrees; NoTree for bodies of Commit / AppendBody
}

// Room is the pinned space left after the bodies recorded so far: a downloader may read the next body straight into
// it and then call Commit, instead of AppendBody.
func (p *RawBodies) Room() []byte {
	return unsafe.Slice((*byte)(unsafe.Add(p.Text, p.Used)), int(p.Cap-p.Used))
}

// Commit records a body of n bytes read into Room(), for a get-entries request of maxEntries (end - start + 1).
func (p *RawBodies) Commit(n int, maxEntries uint32) error {
	return p.CommitLog(n, maxEntries, 0, NoTree)
}

// CommitLog is Commit for a body of log `log` that answers the get-entries request starting at log position `start`:
// ProcessRawBodiesTree(s) folds its entries from there.  A log may answer short, so pass the request's start, not the
// position where the previous answer ended.
func (p *RawBodies) CommitLog(n int, maxEntries uint32, start uint64, log uint32) error {
	if uint64(n) > p.Cap-p.Used || uint64(n) > 0xFFFFFFFF {
		return fmt.Errorf("raw body buffer full")
	}
	p.BodyOff = append(p.BodyOff, p.Used)
	p.BodyLen = append(p.BodyLen, uint32(n))
	p.BodyMax = append(p.BodyMax, maxEntries)
	p.Start = append(p.Start, start)
	p.Log = append(p.Log, log)
	p.Used += uint64(n)
	return nil
}

// AppendBody copies one response body into the pinned text.
func (p *RawBodies) AppendBody(body []byte, maxEntries uint32) error {
	return p.AppendBodyLog(body, maxEntries, 0, NoTree)
}

// AppendBodyLog copies one response body of log `log`, the answer to the request starting at `start`, into the pinned
// text (see CommitLog).
func (p *RawBodies) AppendBodyLog(body []byte, maxEntries uint32, start uint64, log uint32) error {
	if uint64(len(body)) > p.Cap-p.Used {
		return fmt.Errorf("raw body buffer full")
	}
	copy(p.Room(), body)
	return p.CommitLog(len(body), maxEntries, start, log)
}

// BodiesResult holds the outputs of ProcessRawBodies (ctmr_body_out): per entry found (sum of BodyMax rows, the first
// NEntries written) the RawResult arrays and where its strings lie in the text; per body its status and entries.
type BodiesResult struct {
	*RawResult
	body                       *C.ctmr_body_out
	BodyStatus                 []uint8
	BodyFirst                  []uint64
	BodyEntries                []uint32
	LeafInputOff, ExtraDataOff []uint64
	LeafInputLen, ExtraDataLen []uint32
	Escaped                    []uint8
	NEntries                   uint64
}

func NewBodiesResult(p *RawBodies) *BodiesResult {
	n := 0
	for _, m := range p.BodyMax {
		n += int(m)
	}
	r := &BodiesResult{RawResult: NewRawResult(n, p.Used)}
	r.body = (*C.ctmr_body_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_body_out{}))))
	C.memcpy(unsafe.Pointer(&r.body.raw), unsafe.Pointer(r.raw), C.size_t(unsafe.Sizeof(C.ctmr_raw_out{}))) // C pointers only
	var q unsafe.Pointer
	nb := len(p.BodyOff)
	q, r.BodyStatus = view[uint8](r.Result, nb)
	r.body.body_status = (*C.uint8_t)(q)
	q, r.BodyFirst = view[uint64](r.Result, nb)
	r.body.body_first = (*C.uint64_t)(q)
	q, r.BodyEntries = view[uint32](r.Result, nb)
	r.body.body_entries = (*C.uint32_t)(q)
	q, r.LeafInputOff = view[uint64](r.Result, n)
	r.body.leaf_input_off = (*C.uint64_t)(q)
	q, r.LeafInputLen = view[uint32](r.Result, n)
	r.body.leaf_input_len = (*C.uint32_t)(q)
	q, r.ExtraDataOff = view[uint64](r.Result, n)
	r.body.extra_data_off = (*C.uint64_t)(q)
	q, r.ExtraDataLen = view[uint32](r.Result, n)
	r.body.extra_data_len = (*C.uint32_t)(q)
	q, r.Escaped = view[uint8](r.Result, n)
	r.body.escaped = (*C.uint8_t)(q)
	return r
}

func (r *BodiesResult) Free() {
	C.free(unsafe.Pointer(r.body))
	r.body = nil
	r.RawResult.Free()
}

// appendDecoded records one entry whose strings the host decoded: their base64 text goes into the pinned text and
// its spans are appended as Append records them (no tree).
func (p *RawPages) appendDecoded(leaf, extra []byte) error {
	for k, b := range [2][]byte{leaf, extra} {
		n := uint64(base64.StdEncoding.EncodedLen(len(b)))
		if p.Used+n > p.Cap || n > 0xFFFFFFFF {
			return fmt.Errorf("raw page buffer full")
		}
		base64.StdEncoding.Encode(unsafe.Slice((*byte)(unsafe.Add(p.Text, p.Used)), int(n)), b)
		if k == 0 {
			p.LeafOff, p.LeafLen = append(p.LeafOff, p.Used), append(p.LeafLen, uint32(n))
		} else {
			p.ExtraOff, p.ExtraLen = append(p.ExtraOff, p.Used), append(p.ExtraLen, uint32(n))
		}
		p.Used += n
	}
	p.Log = append(p.Log, NoTree)
	return nil
}

// Repeated is where the entries of the BodyRepeatedEntries bodies of a ProcessRawBodies call went: those bodies (two
// top-level "entries" members, which encoding/json merges) are decoded on the host as the reference decodes them, and
// their entries go through one ProcessRaw call.  Entries[b] = {first, count} in Result for body b.
type Repeated struct {
	Result  *RawResult
	Entries map[int][2]int
}

// ProcessRawBodies finds the entries of every accumulated body on the GPU with encoding/json's rules and processes them
// as ProcessRaw does, on one GPU or on every GPU of the group.  The BodyRepeatedEntries bodies are then decoded on the
// host into `fallback` (an empty RawPages the caller owns) and processed with one ProcessRaw call into a RawResult from
// newResult(n).  A body whose host decode fails is the page error the reference retries: it is skipped, every other
// body is still processed, and the errors come back joined.  Every status other than BodyOK and BodyRepeatedEntries is
// that page error too; r.BodyStatus says which bodies to fetch again.
func (d *DB) ProcessRawBodies(p *RawBodies, nowUnixNs int64, r *BodiesResult, fallback *RawPages,
	newResult func(n int) *RawResult) (*Repeated, error) {
	return d.processRawBodies(p, nowUnixNs, r, fallback, newResult, nil, nil, false)
}

// processRawBodies: ProcessRawBodies and its tree forms (tree.go): one tree, or with `routed` one tree per log
func (d *DB) processRawBodies(p *RawBodies, nowUnixNs int64, r *BodiesResult, fallback *RawPages,
	newResult func(n int) *RawResult, tree *Tree, trees []Tree, routed bool) (*Repeated, error) {
	b := (*C.ctmr_body_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_body_batch{}))))
	defer C.free(unsafe.Pointer(b))
	var pin runtime.Pinner
	defer pin.Unpin()
	if n := len(p.BodyOff); n > 0 {
		pin.Pin(&p.BodyOff[0])
		pin.Pin(&p.BodyLen[0])
		pin.Pin(&p.BodyMax[0])
		b.text = (*C.uint8_t)(p.Text)
		b.text_bytes = C.uint64_t(p.Used)
		b.body_off = (*C.uint64_t)(unsafe.Pointer(&p.BodyOff[0]))
		b.body_len = (*C.uint32_t)(unsafe.Pointer(&p.BodyLen[0]))
		b.body_max = (*C.uint32_t)(unsafe.Pointer(&p.BodyMax[0]))
		b.n_bodies = C.uint64_t(n)
	} else if !d.peer && tree == nil && !routed {  // a tree call still writes the roots
		return nil, nil
	}
	b.now_unix_ns = C.int64_t(nowUnixNs)
	var start *C.uint64_t
	var log *C.uint32_t
	if n := len(p.BodyOff); n > 0 && (tree != nil || routed) {
		pin.Pin(&p.Start[0])
		pin.Pin(&p.Log[0])
		start = (*C.uint64_t)(unsafe.Pointer(&p.Start[0]))
		log = (*C.uint32_t)(unsafe.Pointer(&p.Log[0]))
	}
	var err error
	switch {
	case routed && d.g != nil:
		err = d.err(C.ctmr_group_process_raw_bodies_trees(d.g, b, r.body, log, start, treesC(trees), C.uint32_t(len(trees))),
			"ctmr_group_process_raw_bodies_trees")
	case routed:
		err = d.err(C.ctmr_process_raw_bodies_trees(d.h, b, r.body, log, start, treesC(trees), C.uint32_t(len(trees))),
			"ctmr_process_raw_bodies_trees")
	case tree != nil && d.g != nil:
		err = d.err(C.ctmr_group_process_raw_bodies_tree(d.g, b, r.body, start, tree.c()), "ctmr_group_process_raw_bodies_tree")
	case tree != nil:
		err = d.err(C.ctmr_process_raw_bodies_tree(d.h, b, r.body, start, tree.c()), "ctmr_process_raw_bodies_tree")
	case d.g != nil:
		err = d.err(C.ctmr_group_process_raw_bodies(d.g, b, r.body), "ctmr_group_process_raw_bodies")
	default:
		err = d.err(C.ctmr_process_raw_bodies(d.h, b, r.body), "ctmr_process_raw_bodies")
	}
	if err != nil {
		return nil, err
	}
	r.NEntries = uint64(r.body.n_entries)
	rep := &Repeated{Entries: map[int][2]int{}}
	var errs []error
	for i, s := range r.BodyStatus {
		if BodyStatus(s) != BodyRepeatedEntries {
			continue
		}
		body := unsafe.Slice((*byte)(unsafe.Add(p.Text, p.BodyOff[i])), int(p.BodyLen[i]))
		var resp struct {
			Entries []struct {
				LeafInput []byte `json:"leaf_input"`
				ExtraData []byte `json:"extra_data"`
			} `json:"entries"`
		}
		if err := json.Unmarshal(body, &resp); err != nil {
			errs = append(errs, fmt.Errorf("body %d: %w", i, err))
			continue
		}
		first := len(fallback.LeafOff)
		for _, e := range resp.Entries {
			if err := fallback.appendDecoded(e.LeafInput, e.ExtraData); err != nil {
				return nil, err
			}
		}
		rep.Entries[i] = [2]int{first, len(resp.Entries)}
	}
	if n := len(fallback.LeafOff); n > 0 {
		rep.Result = newResult(n)
		if err := d.ProcessRaw(fallback, nowUnixNs, rep.Result); err != nil {
			return nil, err
		}
	}
	return rep, errors.Join(errs...)
}
