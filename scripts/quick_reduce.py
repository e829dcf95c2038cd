# scratch: device-resident timing of tg_reduce_by_key (Zipf s=1, U=2^26) with the per-kernel-class profile
# usage: quick_reduce.py [n] [iters] [zipf|uniform] [sum_f64|min_f64|max_f64|sum_u64|min_u64|max_u64|first]
import ctypes as C
import os
import sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench
from thrill_b200 import capi
c = capi.Ctx(0)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 125000000
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
uniform = len(sys.argv) > 3 and sys.argv[3] == "uniform"
op = sys.argv[4] if len(sys.argv) > 4 else "sum_f64"
U = 1 << 26
d_cdf = c.to_device(bench.zipf_cdf_numpy(U))
d = c.alloc(n * 16)
kvd = capi.KVDesc(16, getattr(capi, "OP_" + op.upper()))
best = 1e9
for i in range(iters):
    if uniform:
        c.ck(c.L.tg_gen_reduce_uniform(c.h, d, 0, n, 42, U, 0))
    else:
        c.ck(c.L.tg_gen_reduce_zipf(c.h, d, 0, n, 42, d_cdf, U, 0))
    c.sync()
    if i == iters // 2: c.profile_enable(True)
    c.timer_start()
    rp, rc = C.c_void_p(), C.c_size_t()
    c.ck(c.L.tg_reduce_by_key(c.h, C.byref(kvd), d, n, C.byref(rp), C.byref(rc)))
    ms = c.timer_stop()
    best = min(best, ms)
names = ["hist", "partition", "merge", "preagg", "aggregate", "compact", "other", "fixup"]
parts = []
for k, nm in enumerate(names):
    t, cnt = c.profile_get(k)
    if cnt: parts.append("%s %.3f ms/%d" % (nm, t / cnt, cnt))
print("reduce %s %s n=%d best %.3f ms = %.2f Grec/s distinct=%d | %s" % (op, "uniform" if uniform else "zipf", n, best, n / best / 1e6, rc.value, " | ".join(parts)), flush=True)
# per-launch partition times in launch order (fastest of the profiled calls at each position)
profiled = iters - iters // 2
per = c.profile_list(capi.K_PARTITION)
k = len(per) // profiled if profiled else 0
if k:
    lst = [min(per[s * k + i] for s in range(profiled)) for i in range(k)]
    print("partition per launch: " + " ".join("%.4f" % t for t in lst) + " ms", flush=True)
