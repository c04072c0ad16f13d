"""The C-ABI shared library: loads, exports every symbol include/ctmr.h declares, and refuses to
run without a GPU (no CPU fallback).  No compute calls here -- those are the -m gpu tests."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    from ct_mapreduce_b200 import build, capi
    build.build()
    return capi.load()


def _declared_functions():
    text = open(os.path.join(ROOT, "include", "ctmr.h")).read() + open(os.path.join(ROOT, "include", "ctmr_frontend.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ctmr_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(lib):
    names = _declared_functions()
    assert len(names) >= 24
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/ctmr.h but not exported by libctmr.so"


def test_python_binding_covers_header(lib):
    from ct_mapreduce_b200 import capi
    assert sorted(capi.EXPORTS) == _declared_functions()


def test_abi_version(lib):
    assert lib.ctmr_abi_version() == 3  # 3: ctmr_group_* / ctmr_peer_* (several GPUs behind the ABI), per-table error codes


def test_struct_layouts_match_header(tmp_path):
    """ctypes mirrors vs. the header itself, measured by compiling a probe with gcc."""
    import subprocess
    from ct_mapreduce_b200 import capi
    src = tmp_path / "probe.c"
    src.write_text('#include "include/ctmr_frontend.h"\n#include "ct_mapreduce_b200/csrc/ctmr_synth.h"\n#include <stdio.h>\n'
                   '#include <stddef.h>\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(ctmr_config), sizeof(ctmr_out),'
                   'sizeof(ctmr_dev_batch), sizeof(ctmr_dev_out), sizeof(ctmr_synth_cfg), sizeof(ctmr_key),'
                   'offsetof(ctmr_key, serial), offsetof(ctmr_key, valid), sizeof(ctmr_raw_batch), sizeof(ctmr_raw_out),'
                   'offsetof(ctmr_raw_out, entry_status), offsetof(ctmr_dev_batch, lens));return 0;}\n')
    exe = tmp_path / "probe"
    subprocess.run(["gcc", "-I", ROOT, str(src), "-o", str(exe)], check=True, cwd=ROOT)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(capi.Config), C.sizeof(capi.Out), C.sizeof(capi.DevBatch), C.sizeof(capi.DevOut),
                   C.sizeof(capi.SynthCfg), capi.KEY_DTYPE.itemsize, capi.KEY_DTYPE.fields["serial"][1],
                   capi.KEY_DTYPE.fields["valid"][1], C.sizeof(capi.RawBatch), C.sizeof(capi.RawOut),
                   capi.RawOut.entry_status.offset, capi.DevBatch.lens.offset]
    assert capi.KEY_DTYPE.itemsize == 64


def _sass_of(kernel_substr):
    import shutil
    import subprocess
    from ct_mapreduce_b200 import capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not installed")
    elf = subprocess.run([cuobjdump, "-lelf", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in elf and "sm_100" not in elf
    sass = subprocess.run([cuobjdump, "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    out = [blk for blk in sass.split("Function : ")[1:] if kernel_substr in blk.split("\n", 1)[0]]
    return out


def test_shipped_hot_kernel_is_what_design_md_says():
    """The library carries sm_90a SASS only, its one streaming map kernel stages certificates with asynchronous
    global->shared copies and keeps SHA-256's additions off the ALU pipe; the measured-and-rejected variants (TMA bulk
    loader, v1, dynamic scheduling, see DESIGN.md) are not in it."""
    blocks = _sass_of("map_stream_kernel")
    assert len(blocks) == 1, [b.split("\n", 1)[0] for b in blocks]   # one streaming map kernel
    hot = blocks[0]
    assert "LDGSTS" in hot            # per-lane cp.async staging
    assert "UBLKCP" not in hot        # no TMA bulk loader, see DESIGN.md
    assert hot.count("SHF.") > 150 and hot.count("IMAD") > 100   # rotations on ALU, additions on the FMA pipe
    assert not _sass_of("map_kernel_v1") and not _sass_of("map_dyn_kernel")


def test_library_reads_no_tuning_switches():
    """What the library computes, and how fast, does not hang on environment variables: the only ones it reads are the
    rounds of the collective call (documented in include/ctmr.h), the peer barrier's timeout and the front end's text
    capacity (which the tests shrink)."""
    kept = {"CTMR_PEER_ROUNDS", "CTMR_PEER_TIMEOUT_MS", "CTMR_FE_TEXT_CAP"}
    csrc = os.path.join(ROOT, "ct_mapreduce_b200", "csrc")
    read = {}
    for f in sorted(os.listdir(csrc)):
        txt = open(os.path.join(csrc, f), errors="ignore").read()
        for name in re.findall(r'\b(?:getenv|env_int)\(\s*"([^"]*)"', txt):
            read.setdefault(name, []).append(f)
        # a name that is not a literal could hide a switch from this test: only env_int's own body passes one on
        assert re.findall(r'\bgetenv\(\s*(?!")([^)]*)\)', txt) in ([], ["name"]), f
    assert "CTMR_PEER_ROUNDS" in read
    assert set(read) <= kept, {k: v for k, v in read.items() if k not in kept}


def test_table_atomics_are_local_and_only_string_identities_cross_gpus():
    """Known-certificate / (issuer, hour) table operations are device-scope atomics in the owner's own HBM (keys travel as
    bulk records instead); only the O(issuers) string-identity inserts of a group use system-scope atomics over NVLink."""
    ins = _sass_of("ctmr13insert_kernel") + _sass_of("ctmr19inbox_insert_kernel")
    def atomics(block):
        return [ln for ln in block.splitlines() if "ATOM" in ln or "RED." in ln]
    assert ins and all(atomics(b_) for b_ in ins) and not any(".SYS" in ln for b_ in ins for ln in atomics(b_))
    meta = _sass_of("ctmr18meta_insert_kernel")
    assert meta and any(".SYS" in ln for b_ in meta for ln in atomics(b_))


def test_no_cpu_fallback_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ct_mapreduce_b200 import capi, engine
    with pytest.raises(capi.CtmrError) as ei:
        engine.GpuCertDatabase()
    assert ei.value.code == capi.E_NO_DEVICE


def test_group_has_no_cpu_fallback_either(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ct_mapreduce_b200 import capi, engine
    with pytest.raises(capi.CtmrError) as ei:
        engine.GpuCertGroup([0, 0])
    assert ei.value.code == capi.E_NO_DEVICE
    assert lib.ctmr_peer_rounds() == capi.PEER_ROUNDS and lib.ctmr_peer_round_entries(10_000_000) == 1_379_311


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under ct_mapreduce_b200/ or include/ may reference it."""
    bad = []
    for base in ("ct_mapreduce_b200", "include"):
        for dp, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                    txt = open(os.path.join(dp, f), errors="ignore").read()
                    if re.search(r"\boracle\b", txt) and "ora_" in txt or "import oracle" in txt or "from oracle" in txt:
                        bad.append(os.path.join(dp, f))
    assert not bad, bad
