# scratch: quick device-resident timing of tg_radix_sort_local with the per-kernel-class profile (not the bench contract)
import ctypes as C
import os
import sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from thrill_b200 import capi
c = capi.Ctx(0)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 100000000
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 6
d = c.alloc(n * 8 + (4 << 20)); tmp = c.alloc(n * 8 + (4 << 20))
desc = capi.u64_desc()
c.ck(c.L.tg_gen_sort_uniform(c.h, d, 0, n, 42)); c.sync()
cs0 = c.checksum(d, n, 8)
best = 1e9
for i in range(iters):
    c.ck(c.L.tg_gen_sort_uniform(c.h, d, 0, n, 42)); c.sync()
    if i == iters // 2: c.profile_enable(True)
    c.timer_start()
    c.ck(c.L.tg_radix_sort_local(c.h, C.byref(desc), d, tmp, n))
    ms = c.timer_stop()
    best = min(best, ms)
pm, pc = c.profile_get(capi.K_PARTITION); hm, hc = c.profile_get(capi.K_RADIX_HIST)
fm, fc = c.profile_get(capi.K_FIXUP); sm, sc = c.profile_get(capi.K_SEGCOUNT)
ok = c.is_sorted(desc, d, n) and c.checksum(d, n, 8) == cs0
print("n=%d best %.3f ms = %.2f Gkeys/s | partition %.4f ms/launch (%d) = %.0f GB/s | hist %.4f ms | fixup %.4f ms (%d) | segcount %.4f ms (%d) | correct=%s"
      % (n, best, n / best / 1e6, pm / max(pc, 1), pc,
         16 * n / (pm / max(pc, 1)) / 1e6, hm / max(hc, 1), fm / max(fc, 1), fc, sm / max(sc, 1), sc, ok), flush=True)
# per-launch partition times in launch order (fastest of the profiled sorts at each position)
profiled = iters - iters // 2
per = c.profile_list(capi.K_PARTITION)
k = len(per) // profiled if profiled else 0
if k:
    lst = [min(per[s * k + i] for s in range(profiled)) for i in range(k)]
    print("partition per launch: " + " ".join("%.4f" % t for t in lst) + " ms", flush=True)
