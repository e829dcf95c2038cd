# Device-resident timing of the HyperLogLog action (tg_hyperloglog, one GPU), against what the stock action pays first:
#   u64 uniform / zipf      1e8 uint64_t: all distinct (consecutive integers), and a Zipf(1.1) draw over 2^20 values
#   pair uniform / zipf     5e7 pair<uint64_t, uint64_t>, the same two key distributions
#   each at p = 14 (a 16 KB register array per CTA in shared memory) and p = 18 (the 256 KB array in global memory)
#   fetch                   tg_dev_file_fetch of the same 1e8 x 8 B buffer into page-locked host memory (the D2H a GPU node
#                           makes before the stock HyperLogLogNode can hash anything)
# Calls are timed with CUDA events after warm-up (median and min); the kernel's share comes from a separate profiled call
# (TG_K_HLL).  The kernel is bound by integer instructions, not by HBM: the script reports items/s, the 64-bit operations of
# SipHash per second (14 per round, 8 rounds for 8-byte items, 10 for pairs) and the bytes/s only for comparison.  The registers
# of a 1e6-item prefix are checked against the numpy model (tests/hll_ref.py); the full model would take minutes.  Prints the
# card, its power limit and its SM clock (a read-only query).
#   python scripts/quick_hll.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import hll_ref as H  # noqa: E402

PREFIX = 1_000_000


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def timed(c, call, iters):
    times = []
    for it in range(iters + 2):
        c.timer_start()
        call()
        t = c.timer_stop()
        if it >= 2:
            times.append(t)
    return float(np.median(times)), min(times)


def run_case(c, name, words, ib, p, iters):
    n = len(words) // (ib // 8)
    d = c.to_device(words)
    out = np.zeros(1 << p, np.uint8)

    def call(count=n):
        c.ck(c.L.tg_hyperloglog(c.h, ib, p, d, count, out.ctypes.data))
    med, best = timed(c, call, iters)
    c.profile_enable(True)
    before = len(c.profile_list(capi.K_HLL))
    call()
    kern = c.profile_list(capi.K_HLL)[before]
    c.profile_enable(False)
    nonzero = int(np.count_nonzero(out))
    call(PREFIX)
    ok = np.array_equal(out, H.registers(words[:PREFIX * (ib // 8)], ib, p))
    ops = 14 * (8 if ib == 8 else 10)
    print("%-12s p=%-2d n=%.0e  %.3f ms (min %.3f); kernel %.3f ms = %.1f Gitems/s = %.2f T 64-bit SipHash ops/s (%.2f TB/s read); "
          "%d registers set; 1e6-item prefix %s"
          % (name, p, n, med, best, kern, n / kern / 1e6, n * ops / kern / 1e9, n * ib / kern / 1e9, nonzero,
             "equal to the model" if ok else "DIFFERENT from the model"), flush=True)
    c.free(d)
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    n = 100_000_000
    rng = np.random.default_rng(5)
    c = capi.Ctx(0)
    uniform = np.uint64(1 << 40) + np.arange(n, dtype=np.uint64)
    zipf = (rng.zipf(1.1, n) % (1 << 20)).astype(np.uint64)
    ok = True
    for p in (14, 18):
        ok = run_case(c, "u64 uniform", uniform, 8, p, iters) and ok
        ok = run_case(c, "u64 zipf", zipf, 8, p, iters) and ok
    pairs = np.empty(n, np.uint64)                  # 5e7 pairs: (key, position)
    for name, keys in (("pair uniform", uniform[:n // 2]), ("pair zipf", zipf[:n // 2])):
        pairs[0::2] = keys
        pairs[1::2] = np.arange(n // 2, dtype=np.uint64) & np.uint64(7)
        for p in (14, 18):
            ok = run_case(c, name, pairs, 16, p, iters) and ok
    del pairs, zipf
    # what the stock action pays first: the device File fetched to the host
    d = c.to_device(uniform)
    f = capi.DevFile(d, n, 8, 0)
    host = c.host_alloc(n * 8)
    blk = (capi.Block * 1)()
    blk[0].data, blk[0].bytes = host.ctypes.data, n * 8

    def fetch():
        c.ck(c.L.tg_dev_file_fetch(c.h, C.byref(f), blk, 1))
    med, best = timed(c, fetch, max(3, iters // 2))
    ok = ok and np.array_equal(host.view(np.uint64), uniform)
    print("%-12s n=%.0e  %.3f ms (min %.3f) = %.1f GB/s D2H into page-locked memory" % ("fetch", n, med, best, n * 8 / best / 1e6),
          flush=True)
    c.host_free(host)
    c.free(d)
    c.close()
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
