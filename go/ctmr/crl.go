package ctmr

/*
#include <stdlib.h>
#include "ctmr.h"
*/
import "C"

import (
	"fmt"
	"unsafe"
)

// Revoked is one revokedCertificates entry of a CRL handed to RevokedKnown, with its join against the
// "serials::<expDate>::<issuer>" sets the table holds.
type Revoked struct {
	Serial       []byte // INTEGER content octets (a view into the caller's CRL bytes)
	RevokedAt    int64  // unix seconds
	Reason       uint8  // reasonCode, 0xFF when absent
	Status       uint8  // CTMR_RV_*
	Known        bool   // some set serials::<h>::<issuer> holds the serial
	KnownExpHour int64  // the lowest such h
	KnownSets    uint32 // how many such h
}

// CRLResult is what RevokedKnown reports for one CRL.
type CRLResult struct {
	Status     uint8 // CTMR_CRL_*
	Flags      uint8 // bit 0 deltaCRLIndicator, bit 1 issuingDistributionPoint
	ThisUpdate int64
	NextUpdate int64 // math.MinInt64 when absent
	TBS        []byte // the signed bytes: verify the CRL's signature over them
	Entries    []Revoked
}

// RevokedKnown parses DER CRLs on the GPU and answers, per entry, whether the serial is a known certificate of the
// issuer whose crl:: set named the CRL (issuerIDs[i] is that Issuer.ID() digest, 32 bytes).  Read-only.  On a DB
// attached to peers the call is collective: every rank calls it with its own CRLs, none included, and gets the
// answers for its own CRLs against every rank's shard; a rank whose arguments are refused still makes the call.  Fewer
// issuer IDs than CRLs is an error (it used to be an index-out-of-range panic).
func (d *DB) RevokedKnown(crls [][]byte, issuerIDs [][32]byte) ([]CRLResult, error) {
	n := len(crls)
	if n == 0 {
		if !d.peer {
			return nil, nil
		}
		b := (*C.ctmr_crl_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_crl_batch{}))))
		defer C.free(unsafe.Pointer(b))
		out := (*C.ctmr_crl_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_crl_out{}))))
		defer C.free(unsafe.Pointer(out))
		return nil, d.err(C.ctmr_revoked_known(d.h, b, out), "ctmr_revoked_known")
	}
	if len(issuerIDs) < n { // one issuer ID per CRL; extra IDs are ignored, as before
		err := fmt.Errorf("RevokedKnown: %d issuer IDs for %d CRLs", len(issuerIDs), n)
		return nil, d.peerRefuseWith(err, func() { C.ctmr_revoked_known(d.h, nil, nil) })
	}
	total := 0
	for _, c := range crls {
		total += len(c)
	}
	// flat C copies of the inputs: the batch struct itself holds pointers
	data := C.malloc(C.size_t(total + 1))
	defer C.free(data)
	offs := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(8 * n)))[:n:n]
	lens := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(8 * n)))[:n:n]
	dig := C.malloc(C.size_t(32 * n))
	defer C.free(unsafe.Pointer(&offs[0]))
	defer C.free(unsafe.Pointer(&lens[0]))
	defer C.free(dig)
	flat := unsafe.Slice((*byte)(data), total+1)
	o := 0
	for i, c := range crls {
		copy(flat[o:], c)
		offs[i], lens[i] = C.uint64_t(o), C.uint64_t(len(c))
		copy(unsafe.Slice((*byte)(dig), 32*n)[32*i:], issuerIDs[i][:])
		o += len(c)
	}
	capEntries := total/18 + 1
	b := (*C.ctmr_crl_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_crl_batch{}))))
	defer C.free(unsafe.Pointer(b))
	b.data, b.data_bytes = (*C.uint8_t)(data), C.uint64_t(total)
	b.crl_off, b.crl_len = &offs[0], &lens[0]
	b.issuer_digest, b.n_crls = (*C.uint8_t)(dig), C.uint64_t(n)
	out := (*C.ctmr_crl_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_crl_out{}))))
	defer C.free(unsafe.Pointer(out))
	alloc := func(per, count int) unsafe.Pointer {
		p := C.calloc(C.size_t(count), C.size_t(per))
		return p
	}
	ptrs := []unsafe.Pointer{
		alloc(1, n), alloc(1, n), alloc(8, n), alloc(8, n), alloc(8, n), alloc(4, n), alloc(8, n), alloc(4, n),
		alloc(8, capEntries), alloc(1, capEntries), alloc(8, capEntries), alloc(1, capEntries), alloc(1, capEntries),
		alloc(1, capEntries), alloc(8, capEntries), alloc(4, capEntries),
	}
	for _, p := range ptrs {
		defer C.free(p)
	}
	out.crl_status, out.crl_flags = (*C.uint8_t)(ptrs[0]), (*C.uint8_t)(ptrs[1])
	out.this_update, out.next_update = (*C.int64_t)(ptrs[2]), (*C.int64_t)(ptrs[3])
	out.tbs_off, out.tbs_len = (*C.uint64_t)(ptrs[4]), (*C.uint32_t)(ptrs[5])
	out.crl_first, out.crl_entries = (*C.uint64_t)(ptrs[6]), (*C.uint32_t)(ptrs[7])
	out.serial_off, out.serial_len = (*C.uint64_t)(ptrs[8]), (*C.uint8_t)(ptrs[9])
	out.revoked_at, out.reason = (*C.int64_t)(ptrs[10]), (*C.uint8_t)(ptrs[11])
	out.entry_status, out.known = (*C.uint8_t)(ptrs[12]), (*C.uint8_t)(ptrs[13])
	out.known_exp_hour, out.known_sets = (*C.int64_t)(ptrs[14]), (*C.uint32_t)(ptrs[15])
	out.entry_cap = C.uint64_t(capEntries)
	var rc C.int
	if d.g != nil {
		rc = C.ctmr_group_revoked_known(d.g, b, out)
	} else {
		rc = C.ctmr_revoked_known(d.h, b, out)
	}
	if err := d.err(rc, "ctmr_revoked_known"); err != nil {
		return nil, err
	}
	u8 := func(i, cnt int) []uint8 { return unsafe.Slice((*uint8)(ptrs[i]), cnt) }
	i64 := func(i, cnt int) []int64 { return unsafe.Slice((*int64)(ptrs[i]), cnt) }
	u64 := func(i, cnt int) []uint64 { return unsafe.Slice((*uint64)(ptrs[i]), cnt) }
	u32 := func(i, cnt int) []uint32 { return unsafe.Slice((*uint32)(ptrs[i]), cnt) }
	ne := int(out.n_entries)
	res := make([]CRLResult, n)
	for k := 0; k < n; k++ {
		base := int(offs[k])
		r := CRLResult{Status: u8(0, n)[k], Flags: u8(1, n)[k], ThisUpdate: i64(2, n)[k], NextUpdate: i64(3, n)[k]}
		if r.Status == C.CTMR_CRL_OK || r.Status == C.CTMR_CRL_UNKNOWN_ISSUER {
			to := int(u64(4, n)[k]) - base
			r.TBS = crls[k][to : to+int(u32(5, n)[k])]
		}
		first, cnt := int(u64(6, n)[k]), int(u32(7, n)[k])
		for e := first; e < first+cnt && e < ne; e++ {
			so := int(u64(8, ne)[e]) - base
			r.Entries = append(r.Entries, Revoked{
				Serial: crls[k][so : so+int(u8(9, ne)[e])], RevokedAt: i64(10, ne)[e], Reason: u8(11, ne)[e],
				Status: u8(12, ne)[e], Known: u8(13, ne)[e] != 0, KnownExpHour: i64(14, ne)[e], KnownSets: u32(15, ne)[e],
			})
		}
		res[k] = r
	}
	return res, nil
}

// Cascade is CRLite's filter cascade as RevokedCascade builds it (include/ctmr.h "CRLite filter cascade" states the
// layout and the query rule).
type Cascade struct {
	Bytes     []byte  // the serialized cascade
	CRLStatus []uint8 // per CRL, CTMR_CRL_*
	Issuers   uint32  // issuers covered: registered, in the batch, every CRL of theirs CTMR_CRL_OK
	Levels    uint32
	Revoked   uint64 // key records included (R)
	Valid     uint64 // key records excluded (S)
}

// Stash is CRLite's stash as RevokedStash computes it (include/ctmr.h "CRLite stash" states the layout and the rules).
type Stash struct {
	Bytes        []byte  // the serialized stash: units of u32 n, u8 32, digest, n entries of u8 len, serial
	CRLStatus    []uint8 // per CRL, CTMR_CRL_*
	Issuers      uint32  // issuers covered (RevokedCascade's rule)
	StashIssuers uint32  // issuer units written
	Revoked      uint64  // key records in R
	InFilter     uint64  // of them: the filter answers revoked
	InStashes    uint64  // of the rest: an earlier stash lists their (issuer, serial)
	Serials      uint64  // (issuer, serial) entries written
}

// cCRLBatch copies crls and their issuer IDs (at least one per CRL) into C memory as one ctmr_crl_batch: the batch
// holds pointers, so it cannot point into Go memory.  free releases all of it.
func cCRLBatch(crls [][]byte, issuerIDs [][32]byte) (*C.ctmr_crl_batch, func()) {
	n := len(crls)
	total := 0
	for _, c := range crls {
		total += len(c)
	}
	data := C.malloc(C.size_t(total + 1))
	offs := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(8*n + 8)))[: n+1 : n+1]
	lens := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(8*n + 8)))[: n+1 : n+1]
	dig := C.malloc(C.size_t(32*n + 32))
	flat := unsafe.Slice((*byte)(data), total+1)
	o := 0
	for i, c := range crls {
		copy(flat[o:], c)
		offs[i], lens[i] = C.uint64_t(o), C.uint64_t(len(c))
		copy(unsafe.Slice((*byte)(dig), 32*n)[32*i:], issuerIDs[i][:])
		o += len(c)
	}
	b := (*C.ctmr_crl_batch)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_crl_batch{}))))
	b.data, b.data_bytes = (*C.uint8_t)(data), C.uint64_t(total)
	b.crl_off, b.crl_len = &offs[0], &lens[0]
	b.issuer_digest, b.n_crls = (*C.uint8_t)(dig), C.uint64_t(n)
	return b, func() {
		C.free(unsafe.Pointer(b))
		C.free(dig)
		C.free(unsafe.Pointer(&lens[0]))
		C.free(unsafe.Pointer(&offs[0]))
		C.free(data)
	}
}

// RevokedCascade builds the filter cascade of the covered issuers' live known certificates on the GPU: the revoked
// ones included, every other one excluded.  crls and issuerIDs as for RevokedKnown, verified CRLs only; salt is at most
// 32 bytes.  Read-only.  The output buffer holds 16 MiB, or twice the DB's last cascade if that is more; a larger cascade
// is built twice (the first build only reports its size).  On a DB attached to peers the call is collective: every rank
// calls it with its own CRLs (none will do) and the same nowUnixSec and salt, and every rank gets the cascade of every
// shard and every rank's CRLs; CRLStatus covers the rank's own CRLs.  A buffer too small on any rank is too small on
// every rank, so every rank builds it the second time together.  A rank whose arguments are refused here still makes
// the call, with no batch, so that the other ranks fail instead of waiting.
func (d *DB) RevokedCascade(crls [][]byte, issuerIDs [][32]byte, nowUnixSec int64, salt []byte) (*Cascade, error) {
	n := len(crls)
	if len(issuerIDs) < n {
		err := fmt.Errorf("RevokedCascade: %d issuer IDs for %d CRLs", len(issuerIDs), n)
		return nil, d.peerRefuseWith(err, func() { C.ctmr_revoked_cascade(d.h, nil, 0, nil, 0, nil) })
	}
	b, free := cCRLBatch(crls, issuerIDs)
	defer free()
	cs := C.malloc(C.size_t(len(salt) + 1))
	defer C.free(cs)
	copy(unsafe.Slice((*byte)(cs), len(salt)+1), salt)
	status := C.calloc(C.size_t(n+1), 1)
	defer C.free(status)
	out := (*C.ctmr_cascade_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_cascade_out{}))))
	defer C.free(unsafe.Pointer(out))
	call := func() C.int {
		if d.g != nil {
			return C.ctmr_group_revoked_cascade(d.g, b, C.int64_t(nowUnixSec), (*C.uint8_t)(cs), C.uint32_t(len(salt)), out)
		}
		return C.ctmr_revoked_cascade(d.h, b, C.int64_t(nowUnixSec), (*C.uint8_t)(cs), C.uint32_t(len(salt)), out)
	}
	size := uint64(16 << 20)
	if 2*d.cascadeBytes > size {
		size = 2 * d.cascadeBytes
	}
	buf := C.malloc(C.size_t(size)) // a larger cascade is built again into a buffer of the size it reported
	out.buf, out.cap, out.crl_status = (*C.uint8_t)(buf), C.uint64_t(size), (*C.uint8_t)(status)
	rc := call()
	if rc == C.CTMR_E_BATCH_TOO_LARGE && out.bytes > 0 {
		C.free(buf)
		buf = C.malloc(C.size_t(out.bytes))
		out.buf, out.cap = (*C.uint8_t)(buf), out.bytes
		rc = call()
	}
	defer C.free(buf)
	if err := d.err(rc, "ctmr_revoked_cascade"); err != nil {
		return nil, err
	}
	d.cascadeBytes = uint64(out.bytes)
	return &Cascade{
		Bytes:     C.GoBytes(buf, C.int(out.bytes)),
		CRLStatus: C.GoBytes(status, C.int(n)),
		Issuers:   uint32(out.issuers),
		Levels:    uint32(out.levels),
		Revoked:   uint64(out.revoked),
		Valid:     uint64(out.valid),
	}, nil
}

// RevokedStash computes CRLite's next stash on the GPU: every (issuer, serial) of RevokedCascade's revoked set for these
// CRLs and nowUnixSec that the published filter answers "not revoked" and that none of stashes lists (every stash
// published since the filter, back to back; may be empty).  crls and issuerIDs as for RevokedCascade.  Read-only.  The
// output buffer holds 1 MiB, or twice the DB's last stash if that is more; a larger stash is computed twice (the first
// call only reports its size).  Not on a DB attached to peers: every rank gets CTMR_E_INVALID.
func (d *DB) RevokedStash(crls [][]byte, issuerIDs [][32]byte, nowUnixSec int64, filter, stashes []byte) (*Stash, error) {
	n := len(crls)
	if len(issuerIDs) < n {
		return nil, fmt.Errorf("RevokedStash: %d issuer IDs for %d CRLs", len(issuerIDs), n)
	}
	b, free := cCRLBatch(crls, issuerIDs)
	defer free()
	cf := C.malloc(C.size_t(len(filter) + 1))
	defer C.free(cf)
	copy(unsafe.Slice((*byte)(cf), len(filter)+1), filter)
	cst := C.malloc(C.size_t(len(stashes) + 1))
	defer C.free(cst)
	copy(unsafe.Slice((*byte)(cst), len(stashes)+1), stashes)
	status := C.calloc(C.size_t(n+1), 1)
	defer C.free(status)
	out := (*C.ctmr_stash_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_stash_out{}))))
	defer C.free(unsafe.Pointer(out))
	call := func() C.int {
		f, fn := (*C.uint8_t)(cf), C.uint64_t(len(filter))
		s, sn := (*C.uint8_t)(cst), C.uint64_t(len(stashes))
		if d.g != nil {
			return C.ctmr_group_revoked_stash(d.g, b, C.int64_t(nowUnixSec), f, fn, s, sn, out)
		}
		return C.ctmr_revoked_stash(d.h, b, C.int64_t(nowUnixSec), f, fn, s, sn, out)
	}
	size := uint64(1 << 20)
	if 2*d.stashBytes > size {
		size = 2 * d.stashBytes
	}
	buf := C.malloc(C.size_t(size)) // a larger stash is computed again into a buffer of the size it reported
	out.buf, out.cap, out.crl_status = (*C.uint8_t)(buf), C.uint64_t(size), (*C.uint8_t)(status)
	rc := call()
	if rc == C.CTMR_E_BATCH_TOO_LARGE && out.bytes > 0 {
		C.free(buf)
		buf = C.malloc(C.size_t(out.bytes))
		out.buf, out.cap = (*C.uint8_t)(buf), out.bytes
		rc = call()
	}
	defer C.free(buf)
	if err := d.err(rc, "ctmr_revoked_stash"); err != nil {
		return nil, err
	}
	d.stashBytes = uint64(out.bytes)
	return &Stash{
		Bytes:        C.GoBytes(buf, C.int(out.bytes)),
		CRLStatus:    C.GoBytes(status, C.int(n)),
		Issuers:      uint32(out.issuers),
		StashIssuers: uint32(out.stash_issuers),
		Revoked:      uint64(out.revoked),
		InFilter:     uint64(out.in_filter),
		InStashes:    uint64(out.in_stashes),
		Serials:      uint64(out.serials),
	}, nil
}

// VerifyCounts are key records of the covered issuers, counted as RevokedCascade counts them.
type VerifyCounts struct {
	Revoked uint64 // in R, answered revoked
	Missed  uint64 // in R, answered not revoked
	Valid   uint64 // in S, answered not revoked
	Blocked uint64 // in S, answered revoked
}

// VerifyMiss is one key record the filter and the stashes answer wrongly.
type VerifyMiss struct {
	IssuerID   [32]byte
	ExpHour    int64
	FirstIndex uint64 // the record's first-seen global index
	Serial     []byte
	Blocked    bool   // an S record answered revoked; false: an R record answered not revoked
}

// Verify is what RevokedVerify reports (include/ctmr.h "CRLite verify" states the rules).
type Verify struct {
	CRLStatus []uint8      // per CRL, CTMR_CRL_*
	Issuers   uint32       // issuers covered (RevokedCascade's rule)
	Levels    uint32       // levels of the filter
	Before    VerifyCounts // records first seen at a global index below coveredBelow
	Since     VerifyCounts // the others
	List      []VerifyMiss // the Before records answered wrongly, by issuer ID, serial and hour
}

// RevokedVerify checks a published filter, with every stash published since it (back to back; may be empty), against
// the table on the GPU: every live known certificate of the covered issuers, revoked by these CRLs or not, is queried.
// coveredBelow is DB.NextIndex read when the filter was built (math.MaxUint64: every record counts in Before).  crls and
// issuerIDs as for RevokedCascade.  Read-only.  The list holds 4096 records, or twice the DB's last list if that is
// more; a longer list is computed twice (the first call only reports its length).  On a DB attached to peers the call
// is collective: every rank calls it with its own CRLs (none will do) and the same nowUnixSec, filter, stashes and
// coveredBelow, and every rank gets the same counts and list.  A rank whose arguments are refused here still makes the
// call, with no batch, so that the other ranks fail instead of waiting.
func (d *DB) RevokedVerify(crls [][]byte, issuerIDs [][32]byte, nowUnixSec int64, filter, stashes []byte, coveredBelow uint64) (*Verify, error) {
	n := len(crls)
	if len(issuerIDs) < n {
		err := fmt.Errorf("RevokedVerify: %d issuer IDs for %d CRLs", len(issuerIDs), n)
		return nil, d.peerRefuseWith(err, func() { C.ctmr_revoked_verify(d.h, nil, 0, nil, 0, nil, 0, 0, nil) })
	}
	b, free := cCRLBatch(crls, issuerIDs)
	defer free()
	cf := C.malloc(C.size_t(len(filter) + 1))
	defer C.free(cf)
	copy(unsafe.Slice((*byte)(cf), len(filter)+1), filter)
	cst := C.malloc(C.size_t(len(stashes) + 1))
	defer C.free(cst)
	copy(unsafe.Slice((*byte)(cst), len(stashes)+1), stashes)
	status := C.calloc(C.size_t(n+1), 1)
	defer C.free(status)
	out := (*C.ctmr_verify_out)(C.calloc(1, C.size_t(unsafe.Sizeof(C.ctmr_verify_out{}))))
	defer C.free(unsafe.Pointer(out))
	call := func() C.int {
		f, fn := (*C.uint8_t)(cf), C.uint64_t(len(filter))
		s, sn := (*C.uint8_t)(cst), C.uint64_t(len(stashes))
		if d.g != nil {
			return C.ctmr_group_revoked_verify(d.g, b, C.int64_t(nowUnixSec), f, fn, s, sn, C.uint64_t(coveredBelow), out)
		}
		return C.ctmr_revoked_verify(d.h, b, C.int64_t(nowUnixSec), f, fn, s, sn, C.uint64_t(coveredBelow), out)
	}
	size := uint64(4096)
	if 2*d.verifyList > size {
		size = 2 * d.verifyList
	}
	rec := C.size_t(unsafe.Sizeof(C.ctmr_verify_miss{}))
	list := C.malloc(C.size_t(size) * rec) // a longer list is computed again into one of the length it reported
	out.list, out.list_cap, out.crl_status = (*C.ctmr_verify_miss)(list), C.uint64_t(size), (*C.uint8_t)(status)
	rc := call()
	if rc == C.CTMR_E_BATCH_TOO_LARGE && out.n_list > 0 {
		C.free(list)
		list = C.malloc(C.size_t(out.n_list) * rec)
		out.list, out.list_cap = (*C.ctmr_verify_miss)(list), out.n_list
		rc = call()
	}
	defer C.free(list)
	if err := d.err(rc, "ctmr_revoked_verify"); err != nil {
		return nil, err
	}
	d.verifyList = uint64(out.n_list)
	counts := func(c C.ctmr_verify_counts) VerifyCounts {
		return VerifyCounts{uint64(c.revoked), uint64(c.missed), uint64(c.valid), uint64(c.blocked)}
	}
	v := &Verify{
		CRLStatus: C.GoBytes(status, C.int(n)),
		Issuers:   uint32(out.issuers),
		Levels:    uint32(out.levels),
		Before:    counts(out.before),
		Since:     counts(out.since),
	}
	for _, m := range unsafe.Slice((*C.ctmr_verify_miss)(list), int(out.n_list)) {
		e := VerifyMiss{ExpHour: int64(m.exp_hour), FirstIndex: uint64(m.first_index), Blocked: m.blocked != 0}
		copy(e.IssuerID[:], C.GoBytes(unsafe.Pointer(&m.digest[0]), 32))
		e.Serial = C.GoBytes(unsafe.Pointer(&m.serial[0]), C.int(m.serial_len))
		v.List = append(v.List, e)
	}
	return v, nil
}
