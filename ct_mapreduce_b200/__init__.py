"""H100-native drop-in for ct-mapreduce's per-entry worker (parse -> filter -> known-certificate dedup -> per-issuer counts).

The product is the C-ABI library `libctmr.so` (include/ctmr.h, include/ctmr_frontend.h) built from csrc/ by build.py.
The Python modules are bindings and host-side mirrors used by bench.py and the tests:

    build      nvcc recipe for libctmr.so (sm_90a only)
    capi       ctypes declarations of every exported entry point
    engine     GpuCertDatabase / GpuCertGroup: the storage.CertDatabase-shaped mirror over one ctx or a group of shards
    sharded    the one-process-per-GPU form: peer-handle exchange over torch.distributed, round / index arithmetic

Nothing here computes on the CPU: without the CUDA library and a device every entry point raises.
"""
