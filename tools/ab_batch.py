"""A/B of launch strategies on the headline frame set: F frames per step, forward+backward, device resident.
  streams : F single-frame calls alternating over S CUDA streams (round-1 harness)
  batch   : ONE batched call (sr_forward / sr_backward over F frames) on one stream
Each configuration runs in a child process."""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import json, os, sys, time
import numpy as np, torch
sys.path.insert(0, %r)
from vidu4d_b200 import rasterizer as R, _capi
from vidu4d_b200.synthetic import object_scene, orbit_view, projection_matrix
surfels, res, F, mode, S, steps = int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]), sys.argv[4], int(sys.argv[5]), int(sys.argv[6])
dev = torch.device("cuda:0")
sc = object_scene(surfels, seed=0, opacity="trained", center=(0, 0, 0)); t = sc.to_torch(dev)
e = torch.empty((0,), device=dev); bg = torch.zeros(3, device=dev)
g = torch.Generator(device=dev).manual_seed(1234)
dLc = torch.randn((F, 3, res, res), device=dev, generator=g); dLo = torch.randn((F, 8, res, res), device=dev, generator=g) * 0.1
P = projection_matrix(0.5, 0.5).astype(np.float64)
vms, pms, cps = [], [], []
for f in range(64):
    Rm, tt = orbit_view(f, 64); W2C = np.eye(4); W2C[:3, :3] = Rm; W2C[:3, 3] = tt
    vms.append(W2C.T.astype(np.float32)); pms.append((W2C.T @ P).astype(np.float32)); cps.append((-Rm.T @ tt).astype(np.float32))
vms = torch.from_numpy(np.stack(vms)).to(dev); pms = torch.from_numpy(np.stack(pms)).to(dev); cps = torch.from_numpy(np.stack(cps)).to(dev)
C = R._C
R.set_sync_mode(False)
side = [torch.cuda.Stream(device=dev) for _ in range(max(S, 1))]
flush = torch.empty((256 << 20,), dtype=torch.uint8, device=dev)
def step(s):
    v0 = (s * F) %% 64
    idx = [(v0 + f) %% 64 for f in range(F)]
    if mode == "split":      # S half-/quarter-batches on S streams
        main = torch.cuda.current_stream()
        for st in side: st.wait_stream(main)
        n = F // S
        for k in range(S):
            with torch.cuda.stream(side[k]):
                ii = idx[k * n:(k + 1) * n]
                o = C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms[ii], pms[ii], 0.5, 0.5, res, res, t["shs"], 3, cps[ii])
                gr = C.rasterize_gaussians_backward_batch(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, vms[ii], pms[ii], 0.5, 0.5, dLc[k * n:(k + 1) * n], dLo[k * n:(k + 1) * n], t["shs"], 3, cps[ii], o[4], o[5], o[6], sum_shared=True, want_transmat=False)
        for st in side: main.wait_stream(st)
        return o, gr
    if mode == "batchsum":
        o = C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms[idx], pms[idx], 0.5, 0.5, res, res, t["shs"], 3, cps[idx])
        gr = C.rasterize_gaussians_backward_batch(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, vms[idx], pms[idx], 0.5, 0.5, dLc, dLo, t["shs"], 3, cps[idx], o[4], o[5], o[6], sum_shared=True, want_transmat=False)
        return o, gr
    if mode == "batch":
        o = C.rasterize_gaussians_batch(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, vms[idx], pms[idx], 0.5, 0.5, res, res, t["shs"], 3, cps[idx])
        gr = C.rasterize_gaussians_backward_batch(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, vms[idx], pms[idx], 0.5, 0.5, dLc, dLo, t["shs"], 3, cps[idx], o[4], o[5], o[6])
        return o, gr
    main = torch.cuda.current_stream()
    for st in side: st.wait_stream(main)
    for f in range(F):
        with torch.cuda.stream(side[f %% S]):
            v = idx[f]
            o = C.rasterize_gaussians(bg, t["means3D"], e, t["opacities"], t["scales"], t["rotations"], 1.0, e, vms[v], pms[v], 0.5, 0.5, res, res, t["shs"], 3, cps[v], False, False)
            gr = C.rasterize_gaussians_backward(bg, t["means3D"], o[3], e, t["scales"], t["rotations"], 1.0, e, vms[v], pms[v], 0.5, 0.5, dLc[f], dLo[f], t["shs"], 3, cps[v], o[4], o[0], o[5], o[6], False)
    for st in side: main.wait_stream(st)
    return o, gr
# first call in sync mode to learn the capacity
R.set_sync_mode(True); step(0); R.set_sync_mode(False)
for s in range(3): step(s)
R.check_overflow(); torch.cuda.synchronize()
ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
for s in range(steps):
    flush.fill_(s & 255)
    ev[s][0].record(); o, gr = step(3 + s); ev[s][1].record()
torch.cuda.synchronize(); R.check_overflow()
ms = sorted(a.elapsed_time(b) for a, b in ev)
med = ms[len(ms) // 2]
out = {"ms_per_step_median": med, "ms_per_frame": med / F, "fps": F / med * 1e3, "min_ms": ms[0]}
# per-kernel timing of one more step, single stream
_capi.get_profile(); _capi.set_profiling(True)
for s in range(2): step(100 + s)
prof = _capi.get_profile(); _capi.set_profiling(False)
out["kernels_ms_per_frame"] = {k: round(v["ms"] / (2 * F), 5) for k, v in prof.items()}
out["checksum"] = [float(o[1].double().sum()), float(gr[2].double().abs().sum())]
print("RESULT " + json.dumps(out))
''' % ROOT

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--surfels", type=int, default=300000); ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--frames", type=int, default=8); ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--configs", default="streams:8;batch:1")
    ap.add_argument("--out", default="ab_batch.json")
    a = ap.parse_args()
    rows = {}
    for cfg in a.configs.split(";"):
        mode, S = cfg.split(":")
        r = subprocess.run([sys.executable, "-c", CHILD, str(a.surfels), str(a.res), str(a.frames), mode, S, str(a.steps)], capture_output=True, text=True)
        line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
        if not line:
            print(cfg, "FAILED", r.stderr[-3000:]); continue
        d = json.loads(line[0][7:]); rows[cfg] = d
        k = d["kernels_ms_per_frame"]
        print(cfg, "fps %.0f  ms/frame %.4f | fwd %.4f bwd %.4f sort %.4f pre %.4f sbwd %.4f gather %.4f" % (
            d["fps"], d["ms_per_frame"], k.get("composite_fwd", 0), k.get("composite_bwd", 0),
            k.get("onesweep_passes", 0) + k.get("sort_histogram", 0) + k.get("sort_plan", 0), k.get("preprocess_fwd", 0),
            k.get("surfel_bwd", 0), k.get("ranges_gather", 0)), d["checksum"], flush=True)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, "gpurun_out", a.out), "w"), indent=1)

if __name__ == "__main__":
    main()
