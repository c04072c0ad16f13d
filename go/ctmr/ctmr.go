// Package ctmr binds libctmr.so (include/ctmr.h) with cgo: the H100-native replacement for the
// loop body of insertCTWorker (cmd/ct-fetch/ct-fetch.go:191-245) and FilesystemDatabase.Store
// (storage/filesystemdatabase.go:158-211).
//
// cgo pointer rules (cmd/cgo "Passing pointers"): C may not be handed a Go pointer to memory that itself
// contains Go pointers.  ctmr_out is a table of pointers, so BOTH the table and every array it points to
// live in C memory here: the arrays in pinned memory from ctmr_host_alloc (which is also what lets the D2H
// copies of the pipeline run asynchronously), the table on the C heap.  Go code sees the arrays through
// unsafe.Slice views; nothing Go-allocated crosses the boundary except flat []byte / []uint64 arguments
// (Go pointers to pointer-free memory, which the rules allow for the duration of the call).
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain (bench.py probes `go version`
// on every GPU box and reports what it finds).  It is the binding a maintainer of jcjones/ct-mapreduce
// adds; see INTEGRATION.md.
package ctmr

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../ct_mapreduce_b200 -lctmr -Wl,-rpath,${SRCDIR}/../../ct_mapreduce_b200
#include <stdlib.h>
#include <string.h>
#include "ctmr.h"
*/
import "C"

import (
	"encoding/binary"
	"errors"
	"fmt"
	"runtime"
	"unsafe"
)

// Status mirrors CTMR_ST_*.
type Status uint8

const (
	StOK Status = iota
	StParseErr
	StFilterCA
	StFilterExpired
	StFilterCN
	StNoIssuer
	StIssuerParseErr
	StSerialTooLong // the reference has no serial-length limit: GPUDatabase hands these entries to the stock Store
)

const IssuerNone = 0xFFFFFFFF

type Config struct {
	Devices           []int  // GPUs of the box; one entry = a single ctx, several = a group (ctmr_group_*)
	TableCapacity     uint64 // known-certificate slots PER GPU
	MaxBatchEntries   uint64
	MaxBatchBytes     uint64
	MaxIssuers        uint32
	IssuerCNFilter    string // *ctconfig.IssuerCNFilter, passed verbatim (split on ',' without trimming)
	LogExpiredEntries bool   // *ctconfig.LogExpiredEntries
	NoFingerprint     bool
}

// DB is one ctx (one GPU) or one group (several GPUs of the box behind one handle): the fan-out is
// inside the library, invisible here (SURVEY.md §8(b)).
type DB struct {
	h            *C.ctmr_ctx
	g            *C.ctmr_group
	peer         bool   // attached to the DBs of other processes (PeerAttach): the batch calls and the front end are collective
	cascadeBytes uint64 // size of the last RevokedCascade: the next call's first buffer holds twice that
	stashBytes   uint64 // size of the last RevokedStash: the next call's first buffer holds twice that
	verifyList   uint64 // records the last RevokedVerify listed: the next call's first list holds twice that
}

func New(c Config) (*DB, error) {
	cfg := (*C.ctmr_config)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_config{}))))
	defer C.free(unsafe.Pointer(cfg))
	cfg.struct_size = C.uint32_t(unsafe.Sizeof(*cfg))
	cfg.table_capacity = C.uint64_t(c.TableCapacity)
	cfg.max_batch_entries = C.uint64_t(c.MaxBatchEntries)
	cfg.max_batch_bytes = C.uint64_t(c.MaxBatchBytes)
	cfg.max_issuers = C.uint32_t(c.MaxIssuers)
	if len(c.IssuerCNFilter) > 0 {
		filt := C.CBytes([]byte(c.IssuerCNFilter)) // C memory: the config struct must not hold a Go pointer
		defer C.free(filt)
		cfg.issuer_cn_filter = (*C.uint8_t)(filt)
		cfg.issuer_cn_filter_len = C.uint32_t(len(c.IssuerCNFilter))
	}
	if c.LogExpiredEntries {
		cfg.log_expired_entries = 1
	}
	if c.NoFingerprint {
		cfg.flags |= C.CTMR_F_NO_FINGERPRINT
	}
	db := &DB{}
	if len(c.Devices) <= 1 {
		if len(c.Devices) == 1 {
			cfg.device = C.int32_t(c.Devices[0])
		}
		if rc := C.ctmr_create(cfg, &db.h); rc != 0 {
			return nil, fmt.Errorf("ctmr_create: %d: %s", int(rc), C.GoString(C.ctmr_last_error(nil)))
		}
		return db, nil
	}
	devs := make([]C.int32_t, len(c.Devices))
	for i, d := range c.Devices {
		devs[i] = C.int32_t(d)
	}
	if rc := C.ctmr_group_create(cfg, &devs[0], C.uint32_t(len(devs)), &db.g); rc != 0 {
		return nil, fmt.Errorf("ctmr_group_create: %d: %s", int(rc), C.GoString(C.ctmr_group_last_error(nil)))
	}
	return db, nil
}

// PeerExport is the first step of one process per GPU (ctmr_peer_export): every process opens a DB on its own GPU with
// the same Config and exports a handle for a group of `world` processes.  Carry the handles to every process by any
// transport (they are plain bytes), then call PeerAttach everywhere.
func (d *DB) PeerExport(world int) ([]byte, error) {
	if d.g != nil {
		return nil, fmt.Errorf("PeerExport: a group DB drives its GPUs itself; open one DB per GPU")
	}
	h := make([]byte, C.CTMR_PEER_HANDLE_BYTES)
	rc := C.ctmr_peer_export(d.h, C.uint32_t(world), (*C.uint8_t)(unsafe.Pointer(&h[0])))
	return h, d.err(rc, "ctmr_peer_export")
}

// PeerAttach attaches this DB as rank `rank` to the handles of all `world` processes (handles[r] = rank r's PeerExport).
// From then on ProcessBatch, ProcessRaw, ProcessTiles and their tree forms are collective: every process makes the same
// sequence of calls, each with its own batch (an empty one when it has nothing to add).
func (d *DB) PeerAttach(rank, world int, handles [][]byte) error {
	if len(handles) != world {
		return fmt.Errorf("PeerAttach: %d handles for %d ranks", len(handles), world)
	}
	all := make([]byte, 0, world*int(C.CTMR_PEER_HANDLE_BYTES))
	for _, h := range handles {
		if len(h) != int(C.CTMR_PEER_HANDLE_BYTES) {
			return fmt.Errorf("PeerAttach: a handle of %d bytes", len(h))
		}
		all = append(all, h...)
	}
	if err := d.err(C.ctmr_peer_attach(d.h, C.uint32_t(rank), C.uint32_t(world), (*C.uint8_t)(unsafe.Pointer(&all[0]))), "ctmr_peer_attach"); err != nil {
		return err
	}
	d.peer = world > 1
	return nil
}

// peerStopped: ranks that stopped at an unknown chain certificate in the last collective front-end call of a peer DB
// (0 for other DBs)
func (d *DB) peerStopped() (uint32, error) {
	if !d.peer {
		return 0, nil
	}
	var n C.uint32_t
	err := d.err(C.ctmr_peer_frontend_stopped(d.h, &n), "ctmr_peer_frontend_stopped")
	return uint32(n), err
}

// peerRefuse: a peer DB that gives up on a front-end call before making it still makes it, with no batch, so that the
// other ranks return CTMR_E_PEER_FAILED instead of waiting at a barrier.  It returns err.
func (d *DB) peerRefuse(err error) error {
	return d.peerRefuseWith(err, func() { C.ctmr_process_raw(d.h, nil, nil) })
}

// peerRefuseWith: the same for any collective call; call makes it with no batch.  It returns err.
func (d *DB) peerRefuseWith(err error, call func()) error {
	if d.peer {
		call()
	}
	return err
}

// peerJoinResumes: a peer DB whose own call failed joins, with an empty batch, the calls that resume other ranks'
// stops, then returns err.
func (d *DB) peerJoinResumes(err error) error {
	for d.peer {
		if n, e := d.peerStopped(); e != nil || n == 0 {
			break
		}
		b := (*C.ctmr_tile_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_tile_batch{}))))
		o := (*C.ctmr_tile_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_tile_out{}))))
		rc := C.ctmr_process_tiles(d.h, b, o)
		C.free(unsafe.Pointer(b))
		C.free(unsafe.Pointer(o))
		if rc != 0 {
			break
		}
	}
	return err
}

func (d *DB) Close() {
	if d.g != nil {
		C.ctmr_group_destroy(d.g)
		d.g = nil
	}
	if d.h != nil {
		C.ctmr_destroy(d.h)
		d.h = nil
	}
}

// member 0 answers registry questions for a group
func (d *DB) ctx0() *C.ctmr_ctx {
	if d.g != nil {
		return C.ctmr_group_member(d.g, 0)
	}
	return d.h
}

func (d *DB) err(rc C.int, what string) error {
	if rc == 0 {
		return nil
	}
	if d.g != nil {
		return fmt.Errorf("%s: %d: %s", what, int(rc), C.GoString(C.ctmr_group_last_error(d.g)))
	}
	return fmt.Errorf("%s: %d: %s", what, int(rc), C.GoString(C.ctmr_last_error(d.h)))
}

// Batch is packed by the batcher goroutine into pinned C memory (ctmr_host_alloc): the H2D copies of
// the pipeline overlap the kernels, and no Go pointer is retained by C.
type Batch struct {
	N          int
	Blob       unsafe.Pointer // pinned, leaf DERs back to back
	Offsets    unsafe.Pointer // pinned uint64[N+1]
	IssuerIdx  unsafe.Pointer // pinned uint32[N], index into the batch's distinct Chain[0] list, IssuerNone = no chain
	IssuerBlob []byte         // flat, pointer-free: may be Go memory
	IssuerOffs []uint64
}

// Result owns the output arrays of one batch in pinned C memory and the C-heap ctmr_out that points at them.
type Result struct {
	n               int
	out             *C.ctmr_out
	Status          []uint8
	SHA256          []byte // N*32
	ExpHour         []int64
	SerialOff       []uint32
	SerialLen       []uint32
	WasUnknown      []uint8
	FirstIssuerHour []uint8
	IssuerNameOff   []uint32 // IssuerMetadata string reducers (SURVEY.md §8(f)-1)
	IssuerNameLen   []uint32
	CrlDpOff        []uint32
	CrlDpLen        []uint32
	FirstIssuerDN   []uint8
	FirstCrlDp      []uint8
	PEM             []byte   // texts of the NEW certificates, entry i = PEM[PemOff[i]:PemOff[i+1]]
	PemOff          []uint64 // N+1
	bufs            []unsafe.Pointer
}

func view[T any](r *Result, n int) (unsafe.Pointer, []T) {
	var z T
	p := C.ctmr_host_alloc(C.size_t(uintptr(n) * unsafe.Sizeof(z)))
	r.bufs = append(r.bufs, p)
	return p, unsafe.Slice((*T)(p), n)
}

// NewResult allocates every output of ctmr_out for n entries whose DER bytes total derBytes (PEM worst case: all new).
func NewResult(n int, derBytes uint64) *Result {
	r := &Result{n: n}
	r.out = (*C.ctmr_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_out{}))))
	var p unsafe.Pointer
	p, r.Status = view[uint8](r, n)
	r.out.status = (*C.uint8_t)(p)
	p, r.SHA256 = view[byte](r, 32*n)
	r.out.sha256 = (*C.uint8_t)(p)
	p, r.ExpHour = view[int64](r, n)
	r.out.exp_hour = (*C.int64_t)(p)
	p, r.SerialOff = view[uint32](r, n)
	r.out.serial_off = (*C.uint32_t)(p)
	p, r.SerialLen = view[uint32](r, n)
	r.out.serial_len = (*C.uint32_t)(p)
	p, r.WasUnknown = view[uint8](r, n)
	r.out.was_unknown = (*C.uint8_t)(p)
	p, r.FirstIssuerHour = view[uint8](r, n)
	r.out.first_issuer_hour = (*C.uint8_t)(p)
	p, r.IssuerNameOff = view[uint32](r, n)
	r.out.issuer_name_off = (*C.uint32_t)(p)
	p, r.IssuerNameLen = view[uint32](r, n)
	r.out.issuer_name_len = (*C.uint32_t)(p)
	p, r.CrlDpOff = view[uint32](r, n)
	r.out.crldp_off = (*C.uint32_t)(p)
	p, r.CrlDpLen = view[uint32](r, n)
	r.out.crldp_len = (*C.uint32_t)(p)
	p, r.FirstIssuerDN = view[uint8](r, n)
	r.out.first_issuer_dn = (*C.uint8_t)(p)
	p, r.FirstCrlDp = view[uint8](r, n)
	r.out.first_crldp = (*C.uint8_t)(p)
	pemCap := int(derBytes/3*4 + derBytes/48 + 64*uint64(n) + 256)
	p, r.PEM = view[byte](r, pemCap)
	r.out.pem = (*C.uint8_t)(p)
	r.out.pem_cap = C.uint64_t(pemCap)
	p, r.PemOff = view[uint64](r, n+1)
	r.out.pem_off = (*C.uint64_t)(p)
	return r
}

func (r *Result) Free() {
	for _, p := range r.bufs {
		C.ctmr_host_free(p)
	}
	r.bufs = nil
	C.free(unsafe.Pointer(r.out))
	r.out = nil
}

// PEMOf is what Store hands to StorageBackend.StoreCertificatePEM for entry i ("" unless the entry is new).
func (r *Result) PEMOf(i int) []byte { return r.PEM[r.PemOff[i]:r.PemOff[i+1]] }

// ProcessBatch = parse + certIsFilteredOut + Store decisions for every entry of the batch, on one GPU or,
// for a group, on every GPU of the box with globally exact results.  nowUnixNs replaces time.Now() at
// ct-fetch.go:52.
func (d *DB) ProcessBatch(b *Batch, nowUnixNs int64, r *Result) error {
	if b.N == 0 {
		return nil
	}
	var ib *C.uint8_t
	var io *C.uint64_t
	nIss := 0
	if len(b.IssuerOffs) > 1 {
		ib = (*C.uint8_t)(unsafe.Pointer(&b.IssuerBlob[0]))
		io = (*C.uint64_t)(unsafe.Pointer(&b.IssuerOffs[0]))
		nIss = len(b.IssuerOffs) - 1
	}
	if d.g != nil {
		rc := C.ctmr_group_process_batch(d.g, (*C.uint8_t)(b.Blob), (*C.uint64_t)(b.Offsets), C.uint64_t(b.N), ib, io,
			C.uint32_t(nIss), (*C.uint32_t)(b.IssuerIdx), C.int64_t(nowUnixNs), r.out)
		return d.err(rc, "ctmr_group_process_batch")
	}
	rc := C.ctmr_process_batch(d.h, (*C.uint8_t)(b.Blob), (*C.uint64_t)(b.Offsets), C.uint64_t(b.N), ib, io,
		C.uint32_t(nIss), (*C.uint32_t)(b.IssuerIdx), C.int64_t(nowUnixNs), r.out)
	return d.err(rc, "ctmr_process_batch")
}

// RegisterIssuers = NewIssuer(x509.ParseCertificate(Chain[0])) for the batch's distinct issuer certificates:
// dense indices (IssuerBad when one does not parse); IssuerDigest(idx) is SHA-256(SPKI), whose base64url is Issuer.ID().
func (d *DB) RegisterIssuers(blob []byte, offs []uint64) ([]uint32, error) {
	n := len(offs) - 1
	if n <= 0 {
		return nil, nil
	}
	out := make([]uint32, n)
	rc := C.ctmr_register_issuers(d.ctx0(), (*C.uint8_t)(unsafe.Pointer(&blob[0])), (*C.uint64_t)(unsafe.Pointer(&offs[0])),
		C.uint32_t(n), (*C.uint32_t)(unsafe.Pointer(&out[0])))
	return out, d.err(rc, "ctmr_register_issuers")
}

func (d *DB) IssuerDigest(idx uint32) ([32]byte, error) {
	var dg [32]byte
	rc := C.ctmr_issuer_digest(d.ctx0(), C.uint32_t(idx), (*C.uint8_t)(unsafe.Pointer(&dg[0])))
	return dg, d.err(rc, "ctmr_issuer_digest")
}

// IssuerCounts = per issuer, the sum over expDates of KnownCertificates.Count()
// (cmd/storage-statistics/storage-statistics.go:44-53).  Keys are raw SHA-256(SPKI) digests.
func (d *DB) IssuerCounts() (map[[32]byte]uint64, error) {
	n := C.size_t(C.ctmr_issuer_count(d.ctx0()))
	if n == 0 {
		return map[[32]byte]uint64{}, nil
	}
	dig := make([]byte, 32*int(n))
	cnt := make([]uint64, int(n))
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_issuer_counts(d.g, (*C.uint8_t)(unsafe.Pointer(&dig[0])), (*C.uint64_t)(unsafe.Pointer(&cnt[0])), &n)
	} else {
		rc = C.ctmr_issuer_counts(d.h, (*C.uint8_t)(unsafe.Pointer(&dig[0])), (*C.uint64_t)(unsafe.Pointer(&cnt[0])), &n)
	}
	if err := d.err(rc, "ctmr_issuer_counts"); err != nil {
		return nil, err
	}
	out := make(map[[32]byte]uint64, int(n))
	for i := 0; i < int(n); i++ {
		var k [32]byte
		copy(k[:], dig[32*i:32*i+32])
		out[k] = cnt[i]
	}
	return out, nil
}

// SetCardinality = RemoteCache.SetCardinality("serials::<expDate>::<issuer>") answered from the set's owner GPU: one probe.
func (d *DB) SetCardinality(expHour int64, issuerDigest [32]byte) (uint64, error) {
	var v C.uint64_t
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_set_cardinality(d.g, C.int64_t(expHour), (*C.uint8_t)(unsafe.Pointer(&issuerDigest[0])), &v)
	} else {
		rc = C.ctmr_set_cardinality(d.h, C.int64_t(expHour), (*C.uint8_t)(unsafe.Pointer(&issuerDigest[0])), &v)
	}
	return uint64(v), d.err(rc, "ctmr_set_cardinality")
}

// StatusCounters = the go-metrics counters certIsFilteredOut.{CA,expired,cn-filtered} and insertCTWorker.Inserted, indexed by Status.
func (d *DB) StatusCounters() ([8]uint64, error) {
	var out [8]uint64
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_status_counters(d.g, (*C.uint64_t)(unsafe.Pointer(&out[0])))
	} else {
		rc = C.ctmr_status_counters(d.h, (*C.uint64_t)(unsafe.Pointer(&out[0])))
	}
	return out, d.err(rc, "ctmr_status_counters")
}

// PreloadKnown seeds one "serials::<expDate>::<issuer>" set from KnownCertificates.Known() at start-up (warm start).
func (d *DB) PreloadKnown(expHour int64, issuerDigest [32]byte, serials [][]byte) error {
	offs := make([]uint64, len(serials)+1)
	var blob []byte
	for i, s := range serials {
		blob = append(blob, s...)
		offs[i+1] = uint64(len(blob))
	}
	if len(blob) == 0 {
		blob = []byte{0}
	}
	bp, op := (*C.uint8_t)(unsafe.Pointer(&blob[0])), (*C.uint64_t)(unsafe.Pointer(&offs[0]))
	dp := (*C.uint8_t)(unsafe.Pointer(&issuerDigest[0]))
	if d.g != nil {
		return d.err(C.ctmr_group_preload_known(d.g, C.int64_t(expHour), dp, bp, op, C.uint64_t(len(serials))), "ctmr_group_preload_known")
	}
	return d.err(C.ctmr_preload_known(d.h, C.int64_t(expHour), dp, bp, op, C.uint64_t(len(serials))), "ctmr_preload_known")
}

// EvictExpired applies the EXPIREAT the reference puts on every serials:: set (knowncertificates.go:98-104); call it hourly.
func (d *DB) EvictExpired(nowUnixSec int64) (uint64, error) {
	var n C.uint64_t
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_evict_expired(d.g, C.int64_t(nowUnixSec), &n)
	} else {
		rc = C.ctmr_evict_expired(d.h, C.int64_t(nowUnixSec), &n)
	}
	return uint64(n), d.err(rc, "ctmr_evict_expired")
}

// Snapshot / Restore of the derived device state: one ctx, or every shard of a group plus its one issuer registry.
// A snapshot restores into a DB of the same shape (capacities; for a group also the number of shards, because the
// owner of a set depends on it).  The []byte is only read / written during the call (cgo pins it).
func (d *DB) Snapshot() ([]byte, error) {
	var need, wrote C.uint64_t
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_snapshot_size(d.g, &need)
	} else {
		rc = C.ctmr_snapshot_size(d.h, &need)
	}
	if err := d.err(rc, "ctmr_snapshot_size"); err != nil {
		return nil, err
	}
	buf := make([]byte, int(need))
	if d.g != nil {
		rc = C.ctmr_group_snapshot_save(d.g, (*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &wrote)
	} else {
		rc = C.ctmr_snapshot_save(d.h, (*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &wrote)
	}
	return buf[:int(wrote)], d.err(rc, "ctmr_snapshot_save")
}

func (d *DB) Restore(snap []byte) error {
	if len(snap) == 0 {
		return fmt.Errorf("empty snapshot")
	}
	if d.g != nil {
		return d.err(C.ctmr_group_snapshot_load(d.g, (*C.uint8_t)(unsafe.Pointer(&snap[0])), C.uint64_t(len(snap))), "ctmr_group_snapshot_load")
	}
	return d.err(C.ctmr_snapshot_load(d.h, (*C.uint8_t)(unsafe.Pointer(&snap[0])), C.uint64_t(len(snap))), "ctmr_snapshot_load")
}

// Checkpoint returns this DB's part of a portable checkpoint (ctmr_checkpoint_save / ctmr_group_checkpoint_save): the
// live records, not the slot layout, so it loads into any table size and any number of GPUs.  A DB attached to peers
// (one process per GPU) saves its own part, collectively.
func (d *DB) Checkpoint() ([]byte, error) {
	var need, wrote C.uint64_t
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_checkpoint_size(d.g, &need)
	} else {
		rc = C.ctmr_checkpoint_size(d.h, &need)
	}
	if err := d.err(rc, "ctmr_checkpoint_size"); err != nil {
		return nil, err
	}
	buf := make([]byte, int(need)+1) // never empty: &buf[0] is valid
	if d.g != nil {
		rc = C.ctmr_group_checkpoint_save(d.g, (*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &wrote)
	} else {
		rc = C.ctmr_checkpoint_save(d.h, (*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &wrote)
	}
	return buf[:int(wrote)], d.err(rc, "ctmr_checkpoint_save")
}

// LoadCheckpoint replaces the state with a checkpoint: every part of it, in any order.
func (d *DB) LoadCheckpoint(parts ...[]byte) error {
	return withParts(parts, func(ptrs **C.uint8_t, sizes *C.uint64_t, n C.uint32_t) error {
		if d.g != nil {
			return d.err(C.ctmr_group_checkpoint_load(d.g, ptrs, sizes, n), "ctmr_group_checkpoint_load")
		}
		return d.err(C.ctmr_checkpoint_load(d.h, ptrs, sizes, n), "ctmr_checkpoint_load")
	})
}

// CheckpointDelta returns this DB's part of a delta checkpoint (ctmr_checkpoint_delta_save): the records first seen at
// or above since, the next index kept with the previous checkpoint or delta (NextIndex at that save, or PartNextIndex of its part).  A DB attached to
// peers saves its own part, collectively.  Refused when since lies past the next index or before the last reset or
// load: take a full Checkpoint there.
func (d *DB) CheckpointDelta(since uint64) ([]byte, error) {
	var need, wrote C.uint64_t
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_checkpoint_delta_size(d.g, C.uint64_t(since), &need)
	} else {
		rc = C.ctmr_checkpoint_delta_size(d.h, C.uint64_t(since), &need)
	}
	if err := d.err(rc, "ctmr_checkpoint_delta_size"); err != nil {
		return nil, err
	}
	buf := make([]byte, int(need)+1) // never empty: &buf[0] is valid
	if d.g != nil {
		rc = C.ctmr_group_checkpoint_delta_save(d.g, C.uint64_t(since), (*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &wrote)
	} else {
		rc = C.ctmr_checkpoint_delta_save(d.h, C.uint64_t(since), (*C.uint8_t)(unsafe.Pointer(&buf[0])), need, &wrote)
	}
	return buf[:int(wrote)], d.err(rc, "ctmr_checkpoint_delta_save")
}

// ApplyCheckpointDelta puts a delta checkpoint on top of the state (ctmr_checkpoint_apply): every part of it, in any
// order.  The state must stand at the delta's since: the base checkpoint loaded and the earlier deltas applied in order.
func (d *DB) ApplyCheckpointDelta(parts ...[]byte) error {
	return withParts(parts, func(ptrs **C.uint8_t, sizes *C.uint64_t, n C.uint32_t) error {
		if d.g != nil {
			return d.err(C.ctmr_group_checkpoint_apply(d.g, ptrs, sizes, n), "ctmr_group_checkpoint_apply")
		}
		return d.err(C.ctmr_checkpoint_apply(d.h, ptrs, sizes, n), "ctmr_checkpoint_apply")
	})
}

// NextIndex is the global index the next entry stored takes (ctmr_next_index).  One ctx only: a group has no index of
// its own to read; use PartNextIndex of its last checkpoint or delta part.
func (d *DB) NextIndex() (uint64, error) {
	if d.g != nil {
		return 0, fmt.Errorf("a group has no ctmr_next_index: use PartNextIndex")
	}
	var n C.uint64_t
	err := d.err(C.ctmr_next_index(d.h, &n), "ctmr_next_index")
	return uint64(n), err
}

// PartNextIndex is the next index a checkpoint or delta part was saved at: the since of the next delta.  Both headers
// keep it as the little-endian uint64 at byte 24.
func PartNextIndex(part []byte) (uint64, error) {
	if len(part) < 128 {
		return 0, fmt.Errorf("truncated checkpoint part")
	}
	return binary.LittleEndian.Uint64(part[24:32]), nil
}

// withParts calls call with the parts' addresses and sizes in C-allocated tables, the parts pinned for the call (cgo's
// rule on Go pointers in C memory).
func withParts(parts [][]byte, call func(ptrs **C.uint8_t, sizes *C.uint64_t, n C.uint32_t) error) error {
	if len(parts) == 0 {
		return fmt.Errorf("no checkpoint parts")
	}
	n := len(parts)
	ptrs := (*[1 << 20]*C.uint8_t)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(uintptr(0)))))[:n:n]
	sizes := (*[1 << 20]C.uint64_t)(C.malloc(C.size_t(n) * 8))[:n:n]
	defer C.free(unsafe.Pointer(&ptrs[0]))
	defer C.free(unsafe.Pointer(&sizes[0]))
	var pin runtime.Pinner
	defer pin.Unpin()
	for i, p := range parts {
		if len(p) == 0 {
			return fmt.Errorf("checkpoint part %d is empty", i)
		}
		pin.Pin(&p[0])
		ptrs[i] = (*C.uint8_t)(unsafe.Pointer(&p[0]))
		sizes[i] = C.uint64_t(len(p))
	}
	return call(&ptrs[0], &sizes[0], C.uint32_t(n))
}

// Resize rehashes the known-certificate, (issuer, expDate) and string-identity tables into the given sizes on the
// device (ctmr_resize / ctmr_group_resize); 0 keeps a table's size.  Afterwards the DB answers as one created with these
// capacities and loaded from a checkpoint taken just before, with its registered chain certificates kept.  All or
// nothing: on failure (CTMR_E_NOMEM, a *_TABLE_FULL for a target too small) the DB is unchanged.  A DB exported to peers
// is refused; resize it before PeerExport, or move the state through Checkpoint / LoadCheckpoint.
func (d *DB) Resize(tableCapacity uint64, pairLog2, metaLog2 uint32) error {
	if d.g != nil {
		return d.err(C.ctmr_group_resize(d.g, C.uint64_t(tableCapacity), C.uint32_t(pairLog2), C.uint32_t(metaLog2)), "ctmr_group_resize")
	}
	return d.err(C.ctmr_resize(d.h, C.uint64_t(tableCapacity), C.uint32_t(pairLog2), C.uint32_t(metaLog2)), "ctmr_resize")
}

// ErrNoMark is the error Rollback returns (wrapped, with the library's text) when the target is not the start of one of
// the last CTMR_ROLLBACK_MARKS entry-taking calls, lies above the next index or below the last reset or load: nothing was
// touched.  Load a checkpoint instead.  These are the only CTMR_E_INVALID refusals a DB can meet: the library's others
// (a NULL handle, a member ctx of a group) concern handles a DB never holds.
var ErrNoMark = errors.New("ctmr: no rollback mark at that index")

// Rollback takes the device state back to the start of an earlier entry-taking call (ctmr_rollback /
// ctmr_group_rollback): the records first seen at or above nextIndex go, the counts follow the remaining keys, the status
// counters are those at that call's start and the next index is nextIndex.  Then run the call again with the same
// indices: its outputs are a clean run's.  The registry and the chain certificates stay; restore the trees yourself.
// Collective on a DB attached to peers.
func (d *DB) Rollback(nextIndex uint64) error {
	var rc C.int
	what := "ctmr_rollback"
	if d.g != nil {
		rc, what = C.ctmr_group_rollback(d.g, C.uint64_t(nextIndex)), "ctmr_group_rollback"
	} else {
		rc = C.ctmr_rollback(d.h, C.uint64_t(nextIndex))
	}
	if rc == C.CTMR_E_INVALID {
		return fmt.Errorf("%w: %v", ErrNoMark, d.err(rc, what))
	}
	return d.err(rc, what)
}

// TableOccupancy returns the live slots and the slots of the known-certificate, (issuer, expDate) and string-identity
// tables, in that order (a group: sums over its shards).  Watch it to resize before a batch fails with *_TABLE_FULL.
func (d *DB) TableOccupancy() (used, capacity [3]uint64, err error) {
	var u, c [3]C.uint64_t
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_table_occupancy(d.g, &u[0], &c[0])
	} else {
		rc = C.ctmr_table_occupancy(d.h, &u[0], &c[0])
	}
	for k := range u {
		used[k], capacity[k] = uint64(u[k]), uint64(c[k])
	}
	return used, capacity, d.err(rc, "ctmr_table_occupancy")
}

func HostAlloc(n int) unsafe.Pointer { return C.ctmr_host_alloc(C.size_t(n)) }
func HostFree(p unsafe.Pointer)      { C.ctmr_host_free(p) }

// BindHostToDevice pins the calling OS thread (runtime.LockOSThread first) to the CPUs next to the GPU, so that the
// pinned buffers it allocates afterwards are NUMA-local.
func BindHostToDevice(device int) int { return int(C.ctmr_bind_host_to_device(C.int32_t(device))) }
