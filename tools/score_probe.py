"""Dev probe: time the scan/merge kernels on a shard-sized corpus generated on the device (not a bench line).

usage: python tools/score_probe.py ROWS DIM [mod] [streamed]
  mod       also time the score-modifier variant
  streamed  force the streamed-query scan kernel (the one dims above 1024 use) whatever DIM is
The JSON line reports the kernel that ran and search_stats(): queries the guard flagged and collect passes run."""
import sys, time, json
import numpy as np
import torch
sys.path.insert(0, ".")
from marqo_b200 import _native
from marqo_b200.engine import RowStore, debug_scan_kernel

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 1_250_000
d = int(sys.argv[2]) if len(sys.argv) > 2 else 768
nq, k = 64, 10
torch.cuda.set_device(0)
g = torch.Generator(device="cuda").manual_seed(0)
store = RowStore(d, capacity=n)
if "streamed" in sys.argv[3:]:
    debug_scan_kernel(store, force_streamed=True)
chunk = 125_000
for lo in range(0, n, chunk):
    m = min(chunk, n - lo)
    x = torch.randn(m, d, device="cuda", generator=g)
    x = torch.nn.functional.normalize(x, dim=1).contiguous()
    torch.cuda.synchronize()
    store.add_device(x.data_ptr(), m)
q = torch.nn.functional.normalize(torch.randn(nq, d, device="cuda", generator=g), dim=1).contiguous()
od = torch.empty(nq, k, dtype=torch.int32, device="cuda")
orow = torch.empty_like(od)
osc = torch.empty(nq, k, dtype=torch.float64, device="cuda")
torch.cuda.synchronize()
res = []
for it in range(8):
    store.search_device(q.data_ptr(), nq, k, od.data_ptr(), orow.data_ptr(), osc.data_ptr(), sync=True)
    res.append(store.last_timing())
scan = sorted(r[0] for r in res[2:])
merge = sorted(r[1] for r in res[2:])
bytes_ = n * d * 2
kernel = {_native.SCAN_RESIDENT_Q: "resident_q", _native.SCAN_STREAMED_Q: "streamed_q"}[debug_scan_kernel(store)]
out = {"n": n, "d": d, "kernel": kernel, "scan_ms_med": scan[len(scan)//2], "scan_ms_min": scan[0],
       "merge_ms_med": merge[len(merge)//2], "GBps_med": bytes_ / scan[len(scan)//2] / 1e6, "GBps_best": bytes_ / scan[0] / 1e6,
       "qps_med": nq * 1e3 / (scan[len(scan)//2] + merge[len(merge)//2]), "search_stats": store.search_stats(), "all": res}
print(json.dumps(out))
print(od[:2].tolist(), osc[:2].tolist())

# score modifiers (f3): same corpus, 3 attribute columns, the scan kernel's HAS_MOD variant through the host entry point
if "mod" in sys.argv[3:]:
    rng = np.random.default_rng(0)
    ids = np.arange(n, dtype=np.int32)
    for c in range(3):
        store.set_attributes(c, ids, rng.uniform(0.5, 2.0, size=n))
    qh = q.cpu().numpy()
    for nq_m in (1, 64):
        ts = []
        for it in range(6):
            t0 = time.perf_counter()
            store.search_modified(qh[:nq_m], k, [(0, 1.5), (1, 0.5)], [(2, 0.01)])
            wall = (time.perf_counter() - t0) * 1e3
            ts.append((store.last_timing()[0], wall))
        ts = sorted(ts[2:])
        print(json.dumps({"modified_search": True, "nq": nq_m, "scan_ms_med": ts[len(ts) // 2][0],
                          "GBps_med": bytes_ / ts[len(ts) // 2][0] / 1e6, "wall_ms_med": sorted(w for _, w in ts)[len(ts) // 2]}))
    for nq_m in (1, 64):
        ts = []
        for it in range(6):
            t0 = time.perf_counter()
            store.search(qh[:nq_m], k)
            ts.append((store.last_timing()[0], (time.perf_counter() - t0) * 1e3))
        ts = sorted(ts[2:])
        print(json.dumps({"modified_search": False, "nq": nq_m, "scan_ms_med": ts[len(ts) // 2][0],
                          "wall_ms_med": sorted(w for _, w in ts)[len(ts) // 2]}))
