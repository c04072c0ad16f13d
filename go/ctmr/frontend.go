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
