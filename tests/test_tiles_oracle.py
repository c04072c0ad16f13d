"""static-ct-api data tiles on the CPU: the Python encoders of ct_mapreduce_b200/frontend.py against the test oracle's own
split (tests/tiles_oracle.py), the get-entries equivalence, leaf hashes, libctmr's host tile generator, and the C
struct layouts of ctmr_tile_batch / ctmr_tile_out."""
import ctypes as C
import hashlib
import struct

import numpy as np
import pytest

import tiles_oracle as to
from ct_mapreduce_b200 import frontend as fe

TS0 = 1_690_000_000_000


def small_corpus(ora, n, **kw):
    cfg = ora.synth_cfg(n, **kw)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    issuers = [iblob[int(ioffs[k]):int(ioffs[k + 1])].tobytes() for k in range(ioffs.size - 1)]
    leaves = [blob[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]
    return leaves, [int(x) for x in idx], issuers


def mixed_tile(ora, N=3, width=40):
    leaves, idx, issuers = small_corpus(ora, width)
    fps = {hashlib.sha256(d).digest(): d for d in issuers}
    fp_of = [hashlib.sha256(d).digest() for d in issuers]
    out = []
    for j in range(width):
        k = idx[j]
        chain = [fp_of[(k + m) % len(issuers)] for m in range(j % 4)]   # chains of 0..3 fingerprints
        ext = fe.leaf_index_extension(256 * N + j) + (b"\x07\x00\x01\xaa" if j % 5 == 0 else b"")
        if j % 3 == 0:
            out.append(fe.tile_leaf_precert(TS0 + j, fp_of[k], fe.tbs_of(leaves[j]), leaves[j], chain, ext))
        else:
            out.append(fe.tile_leaf_x509(TS0 + j, leaves[j], chain, ext))
    return out, leaves, fps


def test_encoders_against_the_oracle_split(ora):
    tl, leaves, fps = mixed_tile(ora)
    tile = fe.data_tile(tl)
    parts = to.split(tile, len(tl))
    assert parts is not None and len(parts) == len(tl)
    assert [len(x) for x in tl] == [p["te_len"] + (3 + p["pre"][1] if p["pre"] else 0) + 2 + 32 * len(p["fps"]) for p in parts]
    for j, p in enumerate(parts):
        assert to.leaf_index_of(p["ext"]) == 256 * 3 + j
        span = p["pre"] if p["type"] == 1 else p["body"]
        assert tile[span[0]:span[0] + span[1]] == leaves[j]
        assert len(p["fps"]) == j % 4
    assert fe.split_tile(tile, len(tl)) is not None
    # width too high / too low, truncated, trailing byte: no split on either side
    for bad, w in ((tile, len(tl) + 1), (tile, len(tl) - 1), (tile[:-1], len(tl)), (tile + b"\x00", len(tl))):
        assert to.split(bad, w) is None and fe.split_tile(bad, w) is None


@pytest.mark.parametrize("how", ["type", "chain31", "zero_cert", "past_end"])
def test_framing_failures_are_bad_tiles(ora, how):
    tl, _, _ = mixed_tile(ora, width=4)
    b = bytearray(tl[1])   # an x509 TileLeaf
    if how == "type":
        b[8:10] = b"\x00\x02"
    elif how == "chain31":
        b[-2 - 32:] = struct.pack(">H", 31) + bytes(32)[:31] + b"\x00"
    elif how == "zero_cert":
        b[10:13] = b"\x00\x00\x00"
    else:
        b[10:13] = b"\xff\xff\xff"
    tile = fe.data_tile([tl[0], bytes(b)] + tl[2:])
    assert to.split(tile, 4) is None and fe.split_tile(tile, 4) is None


def test_leaf_index_rules():
    idx = fe.leaf_index_extension
    assert to.leaf_index_of(idx(5)) == 5
    assert to.leaf_index_of(b"") is None                                     # missing
    assert to.leaf_index_of(idx(5) + idx(5)) is None                         # duplicated
    assert to.leaf_index_of(b"\x00\x00\x04" + bytes(4)) is None              # wrong length
    assert to.leaf_index_of(b"\x09\x00\x00" + idx(7) + b"\x01\x00\x02ab") == 7  # other extensions are ignored
    assert to.leaf_index_of(idx(5)[:-1]) is None                             # malformed list


def test_tile_to_get_entries_round_trip(ora):
    tl, leaves, fps = mixed_tile(ora)
    entries = fe.tile_to_get_entries(fe.data_tile(tl), fps, width=len(tl))
    for j, (li, ed) in enumerate(entries):
        st, e = ora.entry_from_leaf(li, ed)
        assert st == 0, (j, st)
        assert e.entry_type == (1 if j % 3 == 0 else 0) and e.timestamp_ms == TS0 + j
        src = ed if e.leaf_src else li
        assert src[e.leaf_off:e.leaf_off + e.leaf_len] == leaves[j]
        assert e.chain_count == j % 4
        if j % 4:
            assert ed[e.chain0_off:e.chain0_off + e.chain0_len] == fps[fe.split_tile(fe.data_tile(tl), len(tl))[j][3][0]]


def test_leaf_hashes_against_hashlib(ora):
    tl, _, fps = mixed_tile(ora)
    for (li, _), p in zip(fe.tile_to_get_entries(fe.data_tile(tl), fps, width=len(tl)), fe.split_tile(fe.data_tile(tl), len(tl))):
        want = hashlib.sha256(b"\x00" + li).digest()   # RFC 6962 §2.1: SHA-256(0x00 || MerkleTreeLeaf)
        assert fe.leaf_hash(p[0]) == want


def test_host_tile_generator_matches_the_python_encoders(ora):
    from ct_mapreduce_b200 import build, capi
    build.build()
    first, nt = 2, 3
    n = 256 * (first + nt)
    cfg = capi.synth_cfg(n, dup_mode=1, len_mode=1, len_lo=400, len_hi=3000)
    ocfg = ora.synth_cfg(n, dup_mode=1, len_mode=1, len_lo=400, len_hi=3000)
    iblob, ioffs = ora.synth_issuers(ocfg)
    issuers = [iblob[int(ioffs[k]):int(ioffs[k + 1])].tobytes() for k in range(ioffs.size - 1)]
    fps = np.frombuffer(b"".join(hashlib.sha256(d).digest() for d in issuers), np.uint8).copy()
    L = capi.load()
    need = L.ctmr_synth_tiles_host(C.byref(cfg), first, nt, capi.ptr(fps), None, 0, None, None)
    data = np.zeros(need, np.uint8)
    off, ln = np.zeros(nt, np.uint64), np.zeros(nt, np.uint32)
    assert L.ctmr_synth_tiles_host(C.byref(cfg), first, nt, capi.ptr(fps), capi.ptr(data), need, capi.ptr(off), capi.ptr(ln)) == need
    blob, offs, idx = ora.synth_corpus(ocfg, 0, n)
    want = []
    for N in range(first, first + nt):
        leaves = []
        for j in range(256):
            i = 256 * N + j
            leaf, k = blob[int(offs[i]):int(offs[i + 1])].tobytes(), int(idx[i])
            chain = [fps[32 * k:32 * k + 32].tobytes(), fps[32 * ((k + 1) % len(issuers)):32 * ((k + 1) % len(issuers)) + 32].tobytes()][:1 + i % 2]
            ext = fe.leaf_index_extension(i)
            if i % 3 == 0:
                leaves.append(fe.tile_leaf_precert(TS0 + i, hashlib.sha256(issuers[k]).digest(), fe.tbs_of(leaf), leaf, chain, ext))
            else:
                leaves.append(fe.tile_leaf_x509(TS0 + i, leaf, chain, ext))
        want.append(fe.data_tile(leaves))
    assert data.tobytes() == b"".join(want)
    assert ln.tolist() == [len(x) for x in want] and off.tolist() == list(np.cumsum([0] + [len(x) for x in want[:-1]]))


def test_tile_struct_layouts_match_header(tmp_path):
    import subprocess
    from conftest import ROOT
    from ct_mapreduce_b200 import capi
    src = tmp_path / "probe.c"
    src.write_text('#include "include/ctmr_frontend.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %d %d\\n", sizeof(ctmr_tile_batch), sizeof(ctmr_tile_out),'
                   'offsetof(ctmr_tile_batch, tile_width), offsetof(ctmr_tile_out, leaf_hash), offsetof(ctmr_tile_out, missing_cap),'
                   'offsetof(ctmr_tile_out, tiles_done), offsetof(ctmr_tile_out, n_missing), CTMR_FE_BAD_TILE * 10 + CTMR_FE_BAD_INDEX,'
                   'CTMR_E_UNKNOWN_ISSUER);return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(capi.TileBatch), C.sizeof(capi.TileOut), capi.TileBatch.tile_width.offset, capi.TileOut.leaf_hash.offset,
                   capi.TileOut.missing_cap.offset, capi.TileOut.tiles_done.offset, capi.TileOut.n_missing.offset,
                   capi.FE_BAD_TILE * 10 + capi.FE_BAD_INDEX, capi.E_UNKNOWN_ISSUER]


def test_tile_and_page_generators_describe_the_same_entries(ora):
    """ctmr_synth_tiles_host and ctmr_synth_raw_pages_host (the two inputs of tools/bench_tiles.py) give the same entries:
    the same extra_data, and leaf_input equal up to the tile's leaf_index extension."""
    import base64
    from ct_mapreduce_b200 import build, capi
    build.build()
    nt = 2
    n = 256 * nt
    cfg = capi.synth_cfg(n, dup_mode=1)
    L = capi.load()
    ocfg = ora.synth_cfg(n, dup_mode=1)
    iblob, ioffs = ora.synth_issuers(ocfg)
    certs = [iblob[int(ioffs[k]):int(ioffs[k + 1])].tobytes() for k in range(ioffs.size - 1)]
    by_fp = {hashlib.sha256(d).digest(): d for d in certs}
    fps = np.frombuffer(b"".join(hashlib.sha256(d).digest() for d in certs), np.uint8).copy()
    need = L.ctmr_synth_tiles_host(C.byref(cfg), 0, nt, capi.ptr(fps), None, 0, None, None)
    data, off, ln = np.zeros(need, np.uint8), np.zeros(nt, np.uint64), np.zeros(nt, np.uint32)
    L.ctmr_synth_tiles_host(C.byref(cfg), 0, nt, capi.ptr(fps), capi.ptr(data), need, capi.ptr(off), capi.ptr(ln))
    need = L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, 100, None, 0, None, None, None, None)
    text = np.zeros(need, np.uint8)
    lo, ll, xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, 100, capi.ptr(text), need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl))
    tb = text.tobytes()
    for t in range(nt):
        ents = fe.tile_to_get_entries(data[int(off[t]):int(off[t]) + int(ln[t])].tobytes(), by_fp)
        for j, (li, ed) in enumerate(ents):
            i = 256 * t + j
            pli = base64.b64decode(tb[int(lo[i]):int(lo[i]) + int(ll[i])])
            ped = base64.b64decode(tb[int(xo[i]):int(xo[i]) + int(xl[i])])
            assert ed == ped, i
            assert li[-10:] == b"\x00\x08" + fe.leaf_index_extension(i) and li[:-10] == pli[:-2] and pli[-2:] == b"\x00\x00", i
