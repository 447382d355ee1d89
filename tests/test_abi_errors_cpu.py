"""CPU: every int-returning entry point of the C ABI reports its own failure through sr_last_error(), both for a bad
argument and for a failing CUDA call, instead of leaving an earlier call's message behind."""
import ctypes as C
import os
import subprocess
import sys

from .conftest import ROOT

D = 1 << 20      # placeholder DEVICE pointer: never dereferenced (the calls fail before any device work)


def _calls():
    """{entry point: (valid arguments, invalid arguments)}.  The valid arguments pass every argument check; the pointers
    the header documents as HOST pointers are real host buffers.  Returns the ctypes objects too, to keep them alive."""
    from vidu4d_b200 import _capi
    lib = _capi.load()
    fr, bad_fr = _capi.SrFrame(100, 0, 0, 64, 48, 0.5, 0.5, 1.0, 0, 0, 0), _capi.SrFrame(100, 0, 0, -5, 48, 0.5, 0.5, 1.0, 0, 0, 0)
    bt = _capi.SrBatch(1, 0, 0, 0, 0, 0, 0, 0)
    layout = _capi.SrDebugLayout()
    begin, lr = (C.c_int64 * 3)(0, 100, 300), (C.c_float * 2)(1e-3, 1e-3)
    width, ob, nb = (C.c_int32 * 2)(3, 4), (C.c_int64 * 2)(0, 300), (C.c_int64 * 2)(0, 300)
    bmin, bmax = (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(1, 1, 1)
    keep = (fr, bad_fr, bt, layout, begin, lr, width, ob, nb, bmin, bmax)

    def fwd(f=fr, cap=4096):
        return ([C.byref(f), C.byref(bt), D, 3, D, None, D, D, D, D, None, 0, 0, D, D, D, D, 0, None, 0, D, D, D, D, D, cap, D,
                 None, None])

    def bwd(cap=4096):
        return ([C.byref(fr), C.byref(bt), D, 3, D, None, D, D, D, None, 0, 0, D, D, D, D, D, 0, None, 0, D, None, None, D, D, D,
                 cap] + [D] * 8 + [None, None])

    def warp(n, P=100, B=25, M=2):
        return [P, B, M] + [D] * n + [None]

    def post(n, W=64):
        return [W, 48, 0.5, 0.5, 0.0] + [D] * n + [None]

    def loss(M=2):
        return [M, 64, 48, 0.5, 0.5, 0.0] + [D] * 8 + [1.0] * 4 + [D] * 5 + [None]

    def feat_loss(F=22):
        return [2, 64, 48, F, 16, 21] + [D] * 9 + [None]

    def match(n, K=8):
        return [2, 48, 64, 100, 64, K] + [D] * n + [None]

    def reproj_fwd(hxy_dim=3):
        return [2, 48, 64, 25, hxy_dim, 256.0] + [D] * 19 + [None]

    def rows(n, M=2, Cf=16):
        return [100, M, 25, Cf] + [D] * n + [None]

    def adam(step=1):
        return [2, begin, lr, 0.9, 0.999, 1e-15, step, 1.0, D, D, D, D, None]

    def compact(P_new=100):
        return [2, width, ob, nb, 0, 1, P_new] + [D] * 11 + [None]

    def knn(P=100):
        return [P, D, bmin, bmax, D, D, None]

    def outlier(nb_points=20):
        return [100, D, 0.004, nb_points, D, None, D, int(lib.sr_radius_outlier_scratch_bytes(100)), None]

    calls = {
        "sr_forward": (fwd(), fwd(f=bad_fr)),
        "sr_backward": (bwd(), bwd(cap=0)),
        "sr_mark_visible": ([100, D, D, D, D, None], [-1, D, D, D, D, None]),
        "sr_debug_view": ([100, 64, 48, 4096, C.byref(layout)], [100, 64, 48, 4096, None]),
        "sr_post_forward": (post(9), [64, 48, 0.5, 0.5, 0.0, None] + [D] * 8 + [None]),
        "sr_post_backward": (post(11), [64, 48, 0.5, 0.5, 0.0] + [D] * 10 + [None, None]),
        "sr_render_loss_batch": (loss(), loss(M=0)),
        "sr_feature_loss_batch": (feat_loss(), feat_loss(F=0)),
        "sr_bob_warp_forward": (warp(13), warp(13, B=0)),
        "sr_bob_warp_backward": (warp(17), warp(17, B=65)),
        "sr_global_match_forward": (match(9), match(9, K=0)),
        "sr_global_match_backward": (match(12), match(12, K=9)),
        "sr_reproj_loss_forward": (reproj_fwd(), reproj_fwd(hxy_dim=4)),
        "sr_reproj_loss_backward": ([2, 48, 64, 25, 3] + [D] * 18 + [None], [2, 48, 64, 0, 3] + [D] * 18 + [None]),
        "sr_cycle_loss_forward": (warp(15), warp(15, P=-1)),
        "sr_cycle_loss_backward": (warp(16), warp(16, M=0)),
        "sr_feature_rows_forward": (rows(13), rows(13, M=3)),
        "sr_feature_rows_backward": (rows(18), rows(18, Cf=27)),
        "sr_adam_flat": (adam(), adam(step=0)),
        "sr_surfel_compact": (compact(), compact(P_new=-1)),
        "sr_knn_mean_dist2": (knn(), knn(P=-1)),
        "sr_radius_outlier_mask": (outlier(), outlier(nb_points=-1)),
    }
    return lib, calls, keep


def test_adam_betas_are_double(built):
    """Both Adam entry points take torch's double betas (their 1 - beta and bias corrections are formed in double)."""
    from vidu4d_b200 import _capi
    for table, name in ((_capi.PROTOTYPES, "sr_adam_flat"), (_capi.OPTIM_PROTOTYPES, "sr_adam_flat_state")):
        assert table[name][1][3:5] == [C.c_double, C.c_double], name


def test_covers_every_int_entry_point(built):
    from vidu4d_b200 import _capi
    _, calls, _ = _calls()
    ints = {n for n, (res, _) in _capi.PROTOTYPES.items() if res is C.c_int and n != "sr_abi_version"}
    assert set(calls) == ints and len(ints) == 22


def test_bad_argument_sets_its_own_message(built):
    lib, calls, _keep = _calls()
    for name, (_, bad) in calls.items():
        # a sentinel message from a different failure, so that a stale message cannot pass for this call's
        if name == "sr_debug_view":
            assert lib.sr_mark_visible(-1, None, None, None, None, None) == -1
        else:
            assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        sentinel = lib.sr_last_error()
        assert sentinel
        rc = getattr(lib, name)(*bad)
        msg = lib.sr_last_error()
        assert rc == -1, (name, rc, msg)
        assert msg and msg != sentinel, (name, msg)


def _cuda_failures_child():
    """Run with no visible device: every entry point that reaches the device returns SR_ECUDA with the CUDA error's text."""
    import torch
    if torch.cuda.device_count() != 0:
        print("SKIP: a device is visible")
        return
    lib, calls, _keep = _calls()
    cudart = C.CDLL("libcudart.so.12")
    cudart.cudaGetErrorString.restype = C.c_char_p
    assert cudart.cudaGetDeviceCount(C.byref(C.c_int())) != 0
    # the runtime's own wording of each error code (cub reports the missing device as another code than the runtime)
    texts = {cudart.cudaGetErrorString(e) for e in range(1, 1000)} - {cudart.cudaGetErrorString(999999)}
    for name, (good, _) in calls.items():
        if name == "sr_debug_view":         # pure host arithmetic
            continue
        assert lib.sr_debug_view(0, 0, 0, 0, None) == -1
        rc = getattr(lib, name)(*good)
        msg = lib.sr_last_error()
        assert rc == -2, (name, rc, msg)
        assert b"CUDA error in" in msg and any(msg.endswith(b": " + t) for t in texts), (name, msg)
    print("OK")


def test_cuda_failure_sets_its_own_message(built):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", "import tests.test_abi_errors_cpu as t; t._cuda_failures_child()"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().splitlines()[-1] in ("OK", "SKIP: a device is visible"), r.stdout
