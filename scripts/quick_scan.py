# Device-resident timing of PrefixSum and ZipWithIndex (tg_prefix_sum, tg_zip_with_index, one GPU):
#   u64:    PrefixSum std::plus<uint64_t> of 1e8 uint64_t                        model 24 B/item
#   pairs:  PrefixSum ScanSecond<MaxU64> of 1e8 pairs (prefix doubling's names)   model 48 B/item
#   zip:    ZipWithIndex(IndexFirst) of 1e8 uint64_t                              model 24 B/item
# Calls are timed with CUDA events after warm-up (median and min); the per-kernel times come from a separate profiled call
# (TG_K_SCAN launches in order: tile reduce, tile prefix, tile scan; or the one zip kernel), each with its achieved bytes/s at
# the model's bytes for that kernel.  The outputs of the same run are checked in full against the numpy model
# (tests/scan_ref.py).  Prints the card and its power limit.
#   python scripts/quick_scan.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import scan_ref as S  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run_case(c, name, arr, ib, call, kernel_bytes, ref_fn, iters):
    n = len(arr)
    d = c.to_device(arr)
    times = []
    for it in range(iters + 2):
        c.timer_start()
        call(d, n)
        t = c.timer_stop()
        if it >= 2:
            times.append(t)
    c.profile_enable(True)
    out, m = call(d, n)
    per = c.profile_list(capi.K_SCAN)
    c.profile_enable(False)
    res = c.download(out, m * ib).view(S.KV if ib == 16 else np.uint64)
    ok = m == n and np.array_equal(np.ascontiguousarray(res).view(np.uint64), np.ascontiguousarray(ref_fn(arr)).view(np.uint64))
    med = float(np.median(times))
    model = sum(b for _, b in kernel_bytes)
    print("%-6s n=%.0e  %.3f ms (min %.3f) = %.2f Gitems/s, %.2f TB/s at the model's %d B/item"
          % (name, n, med, min(times), n / med / 1e6, n * model / min(times) / 1e9, model), flush=True)
    for (k, b), ms in zip(kernel_bytes, per):
        extra = " = %.2f TB/s (%d B/item)" % (n * b / ms / 1e9, b) if b else ""
        print("    TG_K_SCAN %-8s %.3f ms%s" % (k, ms, extra), flush=True)
    print("    outputs vs model: %s" % ("equal" if ok else "DIFFERENT"), flush=True)
    c.free(d)
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    n = 100_000_000
    rng = np.random.default_rng(5)
    c = capi.Ctx(0)

    def prefix(desc, inclusive):
        def call(d, m):
            out, k = C.c_void_p(), C.c_size_t()
            c.ck(c.L.tg_prefix_sum(c.h, C.byref(desc), d, m, None, inclusive, C.byref(out), C.byref(k)))
            return out.value, k.value
        return call

    def zip_call(d, m):
        out, k = C.c_void_p(), C.c_size_t()
        c.ck(c.L.tg_zip_with_index(c.h, d, m, 1, C.byref(out), C.byref(k)))
        return out.value, k.value

    x = rng.integers(0, 1 << 62, n, dtype=np.uint64)
    ok = run_case(c, "u64", x, 8, prefix(capi.ScanDesc(8, capi.OP_SUM_U64), 1),
                  [("reduce", 8), ("prefix", 0), ("scan", 16)], lambda a: np.cumsum(a, dtype=np.uint64), iters)
    idx = np.arange(n, dtype=np.uint64)
    pairs = S.pairs(rng.integers(0, 1 << 62, n, dtype=np.uint64), np.where(rng.integers(0, 4, n) == 0, idx + np.uint64(1), 0))
    del idx

    def names(a):
        o = np.empty(len(a), S.KV)
        o["key"], o["val"] = a["key"], np.maximum.accumulate(a["val"])
        return o
    ok = run_case(c, "pairs", pairs, 16, prefix(capi.ScanDesc(16, capi.OP_MAX_U64), 1),
                  [("reduce", 16), ("prefix", 0), ("scan", 32)], names, iters) and ok
    del pairs
    ok = run_case(c, "zip", x, 16, zip_call, [("zip", 24)], lambda a: S.zip_with_index([a], True)[0], iters) and ok
    c.close()
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
