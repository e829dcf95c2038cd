# Device-resident timing of GroupByKey / GroupToIndex (tg_group_by_key, tg_group_to_index, one GPU) on 1e8 pairs with
# value = global index:
#   uniform:  keys uniform over 2^26                                    GroupByKey
#   zipf:     keys Zipf(1.1) folded into [0, 2^26)                      GroupByKey
#   index:    keys uniform over 2^26, result_size = 2^26                GroupToIndex
# Calls are timed with CUDA events after warm-up (median and min); the per-kernel-class profile comes from a separate profiled
# call, and the D2H of the grouped items (tg_fetch_output into page-locked memory, what GpuGroupNode::PushData pays before its
# host loop) from a _file call on a device File.  The output of the same run is checked against the numpy model
# (tests/group_ref.py: a stable sort by key) by tg_checksum and sampled positions.  Prints the card and its power limit.
#   python scripts/quick_group.py [iters]
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import group_ref as G  # noqa: E402

CLASSES = [("hist", capi.K_RADIX_HIST), ("partition", capi.K_PARTITION), ("fixup", capi.K_FIXUP),
           ("segcount", capi.K_SEGCOUNT), ("other", capi.K_OTHER)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run_case(c, name, arr, size, iters):
    n = len(arr)
    d = c.to_device(arr)

    def call():
        out, m, b, e = C.c_void_p(), C.c_size_t(), C.c_uint64(), C.c_uint64()
        if size is None:
            c.ck(c.L.tg_group_by_key(c.h, d, n, C.byref(out), C.byref(m)))
        else:
            c.ck(c.L.tg_group_to_index(c.h, d, n, size, C.byref(out), C.byref(m), C.byref(b), C.byref(e)))
        return out.value, m.value

    times = []
    for it in range(iters + 2):
        c.timer_start()
        call()
        t = c.timer_stop()
        if it >= 2:
            times.append(t)
    c.profile_enable(True)
    out, m = call()
    prof = [(k, c.profile_get(cls)) for k, cls in CLASSES]
    c.profile_enable(False)
    # the model: a stable sort by key; the multiset by checksum, the order at sampled positions
    ref = G.grouped(arr)
    dref = c.to_device(ref)
    ok = m == n and c.checksum(dref, n, 16) == c.checksum(out, m, 16)
    pos = np.unique(np.concatenate([np.arange(100), np.arange(n - 100, n), np.random.default_rng(1).integers(0, n, 300)]))
    for p_ in pos[::7]:
        ok = ok and c.download(out + int(p_) * 16, 16).view(G.KV).tolist() == ref[p_:p_ + 1].tolist()
    c.free(dref)
    del ref
    # the D2H of the grouped items into page-locked memory (a _file call on a device File, then tg_fetch_output)
    f = capi.DevFile(d, n, 16, 0)
    inp = capi.MergeInput(C.pointer(f), None, 0)
    host = c.host_alloc(n * 16)
    blocks = (capi.Block * 1)()
    blocks[0].data, blocks[0].bytes = host.ctypes.data, n * 16
    d2h = []
    for _ in range(3):
        cnt, b, e = C.c_size_t(), C.c_uint64(), C.c_uint64()
        if size is None:
            c.ck(c.L.tg_group_by_key_file(c.h, C.byref(inp), C.byref(cnt)))
        else:
            c.ck(c.L.tg_group_to_index_file(c.h, C.byref(inp), size, C.byref(cnt), C.byref(b), C.byref(e)))
        c.sync()
        t0 = time.perf_counter()
        c.ck(c.L.tg_fetch_output(c.h, blocks, 1))
        c.sync()
        d2h.append((time.perf_counter() - t0) * 1e3)
    c.host_free(host)
    med = float(np.median(times))
    print("%-8s n=%.0e  %s %.3f ms (min %.3f) = %.2f Gpairs/s | D2H of the result %.1f ms (%.1f GB/s)"
          % (name, n, "tg_group_by_key" if size is None else "tg_group_to_index", med, min(times), n / med / 1e6,
             min(d2h), n * 16 / min(d2h) / 1e6), flush=True)
    print("    profile: " + ", ".join("%s %.3f ms (%d)" % (k, ms, cnt) for k, (ms, cnt) in prof if cnt), flush=True)
    print("    checksum and sampled positions vs model: %s" % ("equal" if ok else "DIFFERENT"), flush=True)
    c.free(d)
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    rng = np.random.default_rng(5)
    n, u = 100_000_000, 1 << 26
    c = capi.Ctx(0)
    arr = np.empty(n, G.KV)
    arr["val"] = np.arange(n, dtype=np.uint64)
    arr["key"] = rng.integers(0, u, n, dtype=np.uint64)
    ok = run_case(c, "uniform", arr, None, iters)
    ok = run_case(c, "index", arr, u, iters) and ok
    arr["key"] = (rng.zipf(1.1, n) - 1).astype(np.uint64) % np.uint64(u)
    ok = run_case(c, "zipf", arr, None, iters) and ok
    c.close()
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
