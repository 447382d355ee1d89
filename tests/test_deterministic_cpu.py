"""CPU tests of the deterministic backward's C ABI (include/surfel_deterministic.h): the sr_batch_det layout, the header
against the library and the ctypes table, the scratch size, the SR_EINVAL checks that run before any device work, and the
Python switch."""
import ctypes as C
import os
import re
import subprocess

import torch

from .conftest import ROOT

D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def test_batch_det_layout_matches_c(built, tmp_path):
    """ctypes' SrBatchDet against the C compiler's sr_batch_det: size, member offsets and the flag bit."""
    from vidu4d_b200 import _capi
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "surfel_deterministic.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %u\\n", sizeof(sr_batch_det), offsetof(sr_batch_det, batch),'
                   ' offsetof(sr_batch_det, scratch), offsetof(sr_batch_det, scratch_bytes), SR_BATCH_DETERMINISTIC);'
                   ' return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, off_batch, off_scratch, off_bytes, bit = (int(v) for v in subprocess.check_output([str(exe)]).split())
    assert size == C.sizeof(_capi.SrBatchDet)
    assert off_batch == _capi.SrBatchDet.batch.offset == 0
    assert off_scratch == _capi.SrBatchDet.scratch.offset and off_bytes == _capi.SrBatchDet.scratch_bytes.offset
    assert bit == _capi.SR_BATCH_DETERMINISTIC
    assert bit & _capi.SR_BATCH_SUM_SHARED == 0


def test_det_header_and_abi_version_match_library_and_binding(built):
    """include/surfel_deterministic.h <-> libsurfel_raster.so <-> _capi.DET_PROTOTYPES, kept apart from surfel_raster.h's
    table; the SR_ABI_VERSION surfel_raster.h defines is the library's and the binding's."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "surfel_deterministic.h")).read(), flags=re.S)
    protos = re.findall(r"SR_API\s+([\w\s\*]+?)\b(sr_\w+)\s*\(([^)]*)\)", hdr)
    assert {name for _, name, _ in protos} == set(_capi.DET_SYMBOLS) == {"sr_backward_det_bytes"}
    kinds = {"int32_t": C.c_int32, "int64_t": C.c_int64}
    rets = {"size_t": C.c_size_t}
    for ret, name, params in protos:
        assert hasattr(lib, name)
        want = [kinds[p.split()[0]] for p in params.split(",")]
        assert _capi.DET_PROTOTYPES[name] == (rets[ret.strip()], want), name
    assert not set(_capi.DET_SYMBOLS) & set(_capi.SYMBOLS)
    raster = open(os.path.join(ROOT, "include", "surfel_raster.h")).read()
    assert lib.sr_abi_version() == _capi.ABI_VERSION == int(re.search(r"#define SR_ABI_VERSION (\d+)", raster).group(1))


def test_scratch_bytes():
    """One 80-byte slot per instance plus F floats per instance, each region 256-byte aligned."""
    from vidu4d_b200 import _capi
    lib = _capi.load()

    def al(x):
        return (x + 255) // 256 * 256
    for cap, F in ((1, 0), (4096, 0), (4096, 22), (1000003, 32), (256, 1)):
        assert lib.sr_backward_det_bytes(cap, F) == al(cap * 80) + al(cap * F * 4), (cap, F)
    assert lib.sr_backward_det_bytes(4096, 22) > lib.sr_backward_det_bytes(4096, 8) > lib.sr_backward_det_bytes(4096, 0)


def _bwd_args(fr, bt, F=0, cap=4096):
    """sr_backward arguments that pass every other argument check (placeholder device pointers)."""
    feats = (D, F, 0) if F else (None, 0, 0)
    bgc = 3 + F if F else 3
    dfo = (D, 0) if F else (None, 0)
    return ([C.byref(fr), C.byref(bt), D, bgc, D, None, D, D, D, *feats, D, D, D, D, D, 0, *dfo, D, None, None, D, D, D, cap]
            + [D] * 8 + [D if F else None, None])


def test_null_or_short_scratch_is_einval_before_any_device_work(built):
    """SR_BATCH_DETERMINISTIC with a NULL, short or misaligned scratch fails with its own message (these calls would
    otherwise need a GPU); the size checked is sr_backward_det_bytes(capacity, F) per frame."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fr = _capi.SrFrame(100, 0, 0, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    for M, F in ((1, 0), (3, 0), (2, 22)):
        need = M * lib.sr_backward_det_bytes(4096, F)
        bd = _capi.SrBatchDet(_capi.SrBatch(M, _capi.SR_BATCH_DETERMINISTIC | _capi.SR_BATCH_SUM_SHARED, 0, 0, 0, 0, 0, 0),
                              None, need)
        bt = bd.batch                                            # shares bd's memory
        assert lib.sr_backward(*_bwd_args(fr, bt, F)) == -1 and b"scratch pointer is NULL" in lib.sr_last_error()
        bd.scratch = D
        bd.scratch_bytes = need - 1
        assert lib.sr_backward(*_bwd_args(fr, bt, F)) == -1
        assert f"needs {need}".encode() in lib.sr_last_error(), lib.sr_last_error()
        bd.scratch_bytes = -1
        assert lib.sr_backward(*_bwd_args(fr, bt, F)) == -1 and b"scratch has" in lib.sr_last_error()
        bd.scratch, bd.scratch_bytes = D + 4, need
        assert lib.sr_backward(*_bwd_args(fr, bt, F)) == -1 and b"16-byte aligned" in lib.sr_last_error()
    # the other checks still come first: a bad capacity is reported as such
    bd = _capi.SrBatchDet(_capi.SrBatch(1, _capi.SR_BATCH_DETERMINISTIC, 0, 0, 0, 0, 0, 0), None, 0)
    assert lib.sr_backward(*_bwd_args(fr, bd.batch, cap=0)) == -1 and b"capacity" in lib.sr_last_error()


def test_switch_follows_set_deterministic_and_torch():
    from vidu4d_b200 import rasterizer as RZ
    was = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        RZ.set_deterministic(False)
        assert not RZ.deterministic()
        RZ.set_deterministic(True)
        assert RZ.deterministic()
        RZ.set_deterministic(False)
        torch.use_deterministic_algorithms(True)
        assert RZ.deterministic()
    finally:
        torch.use_deterministic_algorithms(was)
        RZ.set_deterministic(False)
