// cgo binding of the static-ct-api part of include/ctmr_frontend.h: data tiles in, the same outputs as ProcessRaw out.
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain.  This is what a maintainer adds next to
// go/ctmr/frontend.go to read logs that publish tile/data/<N> instead of serving get-entries.
package ctmr

/*
#include <stdlib.h>
#include <string.h>
#include "ctmr_frontend.h"
*/
import "C"

import (
	"crypto/sha256"
	"fmt"
	"runtime"
	"unsafe"
)

const (
	FeBadTile  EntryStatus = 6
	FeBadIndex EntryStatus = 7
)

// Tiles accumulates data tiles in pinned memory (ctmr_host_alloc): the downloader appends each tile body as it arrives.
type Tiles struct {
	Data      unsafe.Pointer // pinned, Cap bytes
	Cap, Used uint64
	Off       []uint64
	Len       []uint32
	Index     []uint64 // N of tile/data/<N>
	Width     []uint16 // 256, or W of a partial tile .p/<W>
	Log       []uint32 // the log of each tile, for ProcessTilesTrees (tree.go); NoTree for tiles of Append
}

func (t *Tiles) Append(body []byte, index uint64, width uint16) error {
	return t.AppendLog(body, index, width, NoTree)
}

// AppendLog is Append for a tile of log `log`: ProcessTilesTrees folds its entries into trees[log].
func (t *Tiles) AppendLog(body []byte, index uint64, width uint16, log uint32) error {
	if t.Used+uint64(len(body)) > t.Cap {
		return fmt.Errorf("tile buffer full")
	}
	copy(unsafe.Slice((*byte)(unsafe.Add(t.Data, t.Used)), len(body)), body)
	t.Off = append(t.Off, t.Used)
	t.Len = append(t.Len, uint32(len(body)))
	t.Index = append(t.Index, index)
	t.Width = append(t.Width, width)
	t.Log = append(t.Log, log)
	t.Used += uint64(len(body))
	return nil
}

// TileResult holds the per-entry outputs of ProcessTiles (ctmr_tile_out) in pinned C memory.
type TileResult struct {
	*Result
	out                    *C.ctmr_tile_out
	EntryStatus, EntryType []uint8
	TimestampMs, LeafIndex []uint64
	Issuer                 []uint32
	LeafOff                []uint64 // absolute in Tiles.Data
	LeafLen                []uint32
}

func NewTileResult(n int, dataBytes uint64) *TileResult {
	r := &TileResult{Result: NewResult(n, dataBytes)}
	r.out = (*C.ctmr_tile_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_tile_out{}))))
	C.memcpy(unsafe.Pointer(&r.out.path), unsafe.Pointer(r.Result.out), C.size_t(unsafe.Sizeof(C.ctmr_out{})))
	var p unsafe.Pointer
	p, r.EntryStatus = view[uint8](r.Result, n)
	r.out.entry_status = (*C.uint8_t)(p)
	p, r.EntryType = view[uint8](r.Result, n)
	r.out.entry_type = (*C.uint8_t)(p)
	p, r.TimestampMs = view[uint64](r.Result, n)
	r.out.timestamp_ms = (*C.uint64_t)(p)
	p, r.Issuer = view[uint32](r.Result, n)
	r.out.issuer = (*C.uint32_t)(p)
	p, r.LeafIndex = view[uint64](r.Result, n)
	r.out.leaf_index = (*C.uint64_t)(p)
	p, r.LeafOff = view[uint64](r.Result, n)
	r.out.leaf_off = (*C.uint64_t)(p)
	p, r.LeafLen = view[uint32](r.Result, n)
	r.out.leaf_len = (*C.uint32_t)(p)
	r.out.missing_fp = (*C.uint8_t)(C.malloc(256 * 32))
	r.out.missing_cap = 256
	return r
}

func (r *TileResult) Free() {
	C.free(unsafe.Pointer(r.out.missing_fp))
	C.free(unsafe.Pointer(r.out))
	r.out = nil
	r.Result.Free()
}

// RegisterChainCerts computes each certificate's SHA-256 fingerprint on the GPU and registers it (NewIssuer), so that
// tiles naming it resolve.  Call again after a snapshot restore.
func (d *DB) RegisterChainCerts(ders [][]byte) ([]uint32, error) {
	if len(ders) == 0 {
		return nil, nil
	}
	var blob []byte
	offs := make([]uint64, 1, len(ders)+1)
	for _, x := range ders {
		blob = append(blob, x...)
		offs = append(offs, uint64(len(blob)))
	}
	dense := make([]uint32, len(ders))
	cb := C.CBytes(blob)
	defer C.free(cb)
	var pin runtime.Pinner
	defer pin.Unpin()
	pin.Pin(&offs[0])
	pin.Pin(&dense[0])
	o, dp := (*C.uint64_t)(unsafe.Pointer(&offs[0])), (*C.uint32_t)(unsafe.Pointer(&dense[0]))
	if d.g != nil {
		return dense, d.err(C.ctmr_group_register_chain_certs(d.g, (*C.uint8_t)(cb), o, C.uint32_t(len(ders)), dp, nil), "ctmr_group_register_chain_certs")
	}
	return dense, d.err(C.ctmr_register_chain_certs(d.h, (*C.uint8_t)(cb), o, C.uint32_t(len(ders)), dp, nil), "ctmr_register_chain_certs")
}

// ProcessTiles runs every tile through the GPU.  When a tile names a chain certificate that was never registered, the
// call stops before it; fetch(fp) returns the DER served at issuer/<hex>, which is checked against the fingerprint and
// registered before the call resumes from that tile.  The result equals one call made with every certificate
// registered beforehand: every per-entry output of a resumed call, PEM included, lands at the entries it belongs to.
func (d *DB) ProcessTiles(t *Tiles, nowUnixNs int64, r *TileResult, fetch func(fp [32]byte) ([]byte, error)) error {
	return d.processTiles(t, nowUnixNs, r, fetch, nil, nil, false)
}

// processTiles also folds the entries into tree when it is not nil (ProcessTilesTree, tree.go), or, when routed, each
// tile into trees[t.Log[k]] (ProcessTilesTrees), on one GPU or on every GPU of the group: the library writes the trees
// back at every stop, so each resumed call carries them on from the tiles completed so far.
func (d *DB) processTiles(t *Tiles, nowUnixNs int64, r *TileResult, fetch func(fp [32]byte) ([]byte, error), tree *Tree,
	trees []Tree, routed bool) error {
	if routed && len(t.Log) != len(t.Off) {
		return d.peerRefuse(fmt.Errorf("ProcessTilesTrees: %d log ids for %d tiles", len(t.Log), len(t.Off)))
	}
	if len(t.Off) == 0 && !d.peer {
		if tree != nil || routed { // the roots of the trees as they stand
			b := (*C.ctmr_tile_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_tile_batch{}))))
			defer C.free(unsafe.Pointer(b))
			return d.err(d.tilesCall(b, r.out, nil, tree, trees, routed, true), "ctmr_process_tiles_tree(s)")
		}
		return nil
	}
	var log []uint32 // routed: the tiles' logs, the rest of a log whose fold a bad tile stopped turned to NoTree
	if routed {
		log = append([]uint32(nil), t.Log...)
	}
	var pin runtime.Pinner
	defer pin.Unpin()
	if len(t.Off) > 0 {
		pin.Pin(&t.Off[0])
		pin.Pin(&t.Len[0])
		pin.Pin(&t.Index[0])
		pin.Pin(&t.Width[0])
	}
	b := (*C.ctmr_tile_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_tile_batch{}))))
	defer C.free(unsafe.Pointer(b))
	o := (*C.ctmr_tile_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_tile_out{}))))
	defer C.free(unsafe.Pointer(o))
	pemBase := uint64(0)
	// A peer DB keeps calling while any rank of the collective call stopped: with nothing left, its part is empty.
	for t0, e0 := 0, 0; t0 < len(t.Off) || d.peer; {
		b.data, b.data_bytes = (*C.uint8_t)(t.Data), C.uint64_t(t.Used)
		b.tile_off, b.tile_len, b.tile_index, b.tile_width = nil, nil, nil, nil
		if t0 < len(t.Off) {
			b.tile_off = (*C.uint64_t)(unsafe.Pointer(&t.Off[t0]))
			b.tile_len = (*C.uint32_t)(unsafe.Pointer(&t.Len[t0]))
			b.tile_index = (*C.uint64_t)(unsafe.Pointer(&t.Index[t0]))
			b.tile_width = (*C.uint16_t)(unsafe.Pointer(&t.Width[t0]))
		}
		b.n_tiles, b.now_unix_ns = C.uint64_t(len(t.Off)-t0), C.int64_t(nowUnixNs)
		*o = *r.out
		shiftTileOut(o, e0, t0, pemBase) // a resumed call writes from entry e0, tile t0 and PEM byte pemBase on
		// a bad tile among the tiles completed before a stop ended the fold: the tree is final, the rest runs plain
		fold := tree != nil && (t0 == 0 || t0 == len(t.Off) || tree.Size >= 256*t.Index[t0])
		if routed && t0 > 0 { // a log whose tree stopped below its first remaining tile: a bad tile ended its fold
			stopped := map[uint32]bool{}
			for k := t0; k < len(log); k++ {
				if l := log[k]; l != NoTree {
					if _, seen := stopped[l]; !seen {
						stopped[l] = int(l) < len(trees) && trees[l].Size < 256*t.Index[k]
					}
					if stopped[l] {
						log[k] = NoTree
					}
				}
			}
		}
		var lp *C.uint32_t
		if routed && t0 < len(log) {
			lp = (*C.uint32_t)(unsafe.Pointer(&log[t0]))
		}
		rc := d.tilesCall(b, o, lp, tree, trees, routed, fold)
		done := int(o.tiles_done)
		e1 := e0
		for k := t0; k < t0+done; k++ {
			e1 += int(t.Width[k])
		}
		if r.out.path.pem != nil { // this call's pem_off[e0..e1] count from its own first byte
			for i := e0; i <= e1; i++ {
				r.PemOff[i] += pemBase
			}
			pemBase = r.PemOff[e1]
		}
		t0, e0 = t0+done, e1
		if rc != C.CTMR_E_UNKNOWN_ISSUER {
			if err := d.err(rc, "ctmr_process_tiles"); err != nil {
				if fetch != nil { // the others' resumed calls wait for this rank too
					return d.peerJoinResumes(err)
				}
				return err
			}
			// a peer DB whose part is done: another rank stopped, so it joins that rank's resumed call
			if stopped, err := d.peerStopped(); err != nil || stopped == 0 || fetch == nil {
				return err
			}
			continue
		}
		if fetch == nil {
			return fmt.Errorf("ctmr_process_tiles: tile %d names an unregistered chain certificate", t0)
		}
		missing := unsafe.Slice((*byte)(unsafe.Pointer(o.missing_fp)), 32*int(o.n_missing))
		ders := make([][]byte, 0, o.n_missing)
		for k := 0; k < int(o.n_missing); k++ {
			var fp [32]byte
			copy(fp[:], missing[32*k:])
			der, err := fetch(fp)
			if err != nil {
				return d.peerRefuse(err) // a peer DB that gives up still meets the others' resumed call
			}
			// a log serving the wrong bytes at issuer/<hex> would otherwise stop the loop at this tile for ever
			if sha256.Sum256(der) != fp {
				return d.peerRefuse(fmt.Errorf("ctmr_process_tiles: the certificate fetched for fingerprint %x has another SHA-256", fp))
			}
			ders = append(ders, der)
		}
		if _, err := d.RegisterChainCerts(ders); err != nil {
			return d.peerRefuse(err)
		}
	}
	return nil
}

// shiftTileOut points every per-entry output at entry e0, tile_status at tile t0 and the PEM text at byte pemBase.
func shiftTileOut(o *C.ctmr_tile_out, e0, t0 int, pemBase uint64) {
	add := func(p unsafe.Pointer, per int) unsafe.Pointer {
		if p == nil {
			return nil
		}
		return unsafe.Add(p, e0*per)
	}
	q := &o.path
	q.status = (*C.uint8_t)(add(unsafe.Pointer(q.status), 1))
	q.sha256 = (*C.uint8_t)(add(unsafe.Pointer(q.sha256), 32))
	q.exp_hour = (*C.int64_t)(add(unsafe.Pointer(q.exp_hour), 8))
	q.serial_off = (*C.uint32_t)(add(unsafe.Pointer(q.serial_off), 4))
	q.serial_len = (*C.uint32_t)(add(unsafe.Pointer(q.serial_len), 4))
	q.was_unknown = (*C.uint8_t)(add(unsafe.Pointer(q.was_unknown), 1))
	q.first_issuer_hour = (*C.uint8_t)(add(unsafe.Pointer(q.first_issuer_hour), 1))
	q.issuer_name_off = (*C.uint32_t)(add(unsafe.Pointer(q.issuer_name_off), 4))
	q.issuer_name_len = (*C.uint32_t)(add(unsafe.Pointer(q.issuer_name_len), 4))
	q.crldp_off = (*C.uint32_t)(add(unsafe.Pointer(q.crldp_off), 4))
	q.crldp_len = (*C.uint32_t)(add(unsafe.Pointer(q.crldp_len), 4))
	q.first_issuer_dn = (*C.uint8_t)(add(unsafe.Pointer(q.first_issuer_dn), 1))
	q.first_crldp = (*C.uint8_t)(add(unsafe.Pointer(q.first_crldp), 1))
	q.pem_off = (*C.uint64_t)(add(unsafe.Pointer(q.pem_off), 8))
	if q.pem != nil {
		q.pem = (*C.uint8_t)(unsafe.Add(unsafe.Pointer(q.pem), pemBase))
		q.pem_cap -= C.uint64_t(pemBase)
	}
	o.entry_status = (*C.uint8_t)(add(unsafe.Pointer(o.entry_status), 1))
	o.entry_type = (*C.uint8_t)(add(unsafe.Pointer(o.entry_type), 1))
	o.timestamp_ms = (*C.uint64_t)(add(unsafe.Pointer(o.timestamp_ms), 8))
	o.issuer = (*C.uint32_t)(add(unsafe.Pointer(o.issuer), 4))
	o.leaf_index = (*C.uint64_t)(add(unsafe.Pointer(o.leaf_index), 8))
	o.leaf_off = (*C.uint64_t)(add(unsafe.Pointer(o.leaf_off), 8))
	o.leaf_len = (*C.uint32_t)(add(unsafe.Pointer(o.leaf_len), 4))
	o.leaf_hash = (*C.uint8_t)(add(unsafe.Pointer(o.leaf_hash), 32))
	if o.tile_status != nil {
		o.tile_status = (*C.uint8_t)(unsafe.Add(unsafe.Pointer(o.tile_status), t0))
	}
}

// tilesCall makes the plain, one-tree (fold) or routed call on the ctx, or on the group (several GPUs: one chunk of
// whole tiles per GPU per round, the same outputs, stop and trees).
func (d *DB) tilesCall(b *C.ctmr_tile_batch, o *C.ctmr_tile_out, log *C.uint32_t, tree *Tree, trees []Tree, routed, fold bool) C.int {
	switch {
	case routed && d.g != nil:
		return C.ctmr_group_process_tiles_trees(d.g, b, o, log, treesC(trees), C.uint32_t(len(trees)))
	case routed:
		return C.ctmr_process_tiles_trees(d.h, b, o, log, treesC(trees), C.uint32_t(len(trees)))
	case fold && d.g != nil:
		return C.ctmr_group_process_tiles_tree(d.g, b, o, tree.c())
	case fold:
		return C.ctmr_process_tiles_tree(d.h, b, o, tree.c())
	case d.g != nil:
		return C.ctmr_group_process_tiles(d.g, b, o)
	}
	return C.ctmr_process_tiles(d.h, b, o)
}
