"""The hashlib Merkle tree model (tests/merkle_model.py) pinned by the RFC 6962 reference vectors, and the ctmr_tree
layout: CPU only."""
import ctypes as C
import hashlib

import merkle_model as mm

LEAVES = [bytes.fromhex(x) for x in ("", "00", "10", "2021", "3031", "40414243", "5051525354555657",
                                     "606162636465666768696a6b6c6d6e6f")]
ROOTS = [
    "6e340b9cffb37a989ca544e6bb780a2c78901d3fb33738768511a30617afa01d",
    "fac54203e7cc696cf0dfcb42c92a1d9dbaf70ad9e621f4bd8d98662f00e3c125",
    "aeb6bcfe274b70a14fb067a5e5578264db0fa9b51af5e0ba159158f329e06e77",
    "d37ee418976dd95753c1c73862b9398fa2a2cf9b4ff0fdfe8b30cd95209614b7",
    "4e3bbb1f7b478dcfe71fb631631519a3bca12c9aefca1612bfce4c13a86264d4",
    "76e67dadbcdf1e10e1b74ddc608abd2f98dfb16fbce75277b5232a127f2087ef",
    "ddb89be403809e325750d3d263cd78929c2942b7942a34b77e122c9594a74c8c",
    "5dc9da79a70659a9ad559cb701ded9a2ab9d823aad2f4960cfe370eff4604328",
]


def test_rfc6962_reference_roots():
    for size in range(1, 9):
        assert mm.mth(LEAVES[:size]).hex() == ROOTS[size - 1], size
        hashes = [mm.leaf_hash(x) for x in LEAVES[:size]]
        assert mm.root(mm.edge(hashes, size), size).hex() == ROOTS[size - 1], size


def test_empty_tree():
    assert mm.mth([]) == hashlib.sha256(b"").digest()
    assert mm.root({}, 0) == hashlib.sha256(b"").digest()


def test_extend_matches_mth_everywhere():
    leaves = [i.to_bytes(4, "big") * (i % 5) for i in range(300)]
    hashes = [mm.leaf_hash(x) for x in leaves]
    prefix_roots = [mm.mth_hashes(hashes[:m]) for m in range(301)]
    for s in range(301):
        e = mm.edge(hashes, s)
        assert mm.root(e, s) == prefix_roots[s]
        e2, size = e, s
        for n in range(1, 301 - s):   # extend(edge(s), leaves[s:s+n]), one more leaf onto the previous n
            e2, size = mm.extend(e2, size, hashes[s + n - 1:s + n])
            assert size == s + n
            assert mm.root(e2, size) == prefix_roots[s + n], (s, n)
            assert e2 == mm.edge(hashes, size) or n % 37, (s, n)
        assert mm.extend(e, s, hashes[s:])[0] == e2


def test_extend_ignores_rows_of_clear_bits():
    hashes = [mm.leaf_hash(bytes([i])) for i in range(40)]
    e = mm.edge(hashes, 21)
    junk = dict(e)
    for k in range(64):
        if not (21 >> k) & 1:
            junk[k] = b"\xab" * 32
    assert mm.extend(junk, 21, hashes[21:])[0] == mm.extend(e, 21, hashes[21:])[0]


def test_tree_struct_layout_matches_header(tmp_path):
    import subprocess
    from conftest import ROOT
    from ct_mapreduce_b200 import capi
    src = tmp_path / "probe.c"
    src.write_text('#include "include/ctmr_frontend.h"\n#include <stdio.h>\n#include <stddef.h>\n'
                   'int main(){printf("%zu %zu %zu %zu\\n", sizeof(ctmr_tree), offsetof(ctmr_tree, size),'
                   'offsetof(ctmr_tree, edge), offsetof(ctmr_tree, root));return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [2088, 0, 8, 2056]
    assert got == [C.sizeof(capi.Tree), capi.Tree.size.offset, capi.Tree.edge.offset, capi.Tree.root.offset]
