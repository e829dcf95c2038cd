# Device-resident timing of Sample and BernoulliSample (tg_sample / tg_bernoulli_sample, one GPU), against what the stock nodes
# pay first:
#   Sample(10), Sample(5e7)          of 1e8 uint64_t
#   Sample(10)                       of 5e7 pairs (16-byte items)
#   BernoulliSample(0.01), (0.5)     of 1e8 uint64_t
#   fetch                            tg_dev_file_fetch of the same 1e8 x 8 B buffer into page-locked host memory (the D2H the
#                                    stock nodes need before they sample anything)
# Calls are timed with CUDA events after warm-up (median of `iters`, and min); the kernels come from a separate profiled call
# (TG_K_SAMPLE): the hashing passes one by one (histogram, candidate gather, count, write) and the small kernels (candidate
# histograms, digit picks, tile scan) summed.  Every output is checked against tests/sample_ref.py in the same run.  Prints the
# card, its power limit and SM clock.
#   python scripts/quick_sample.py [iters]
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from thrill_b200 import capi  # noqa: E402
import sample_ref as S  # noqa: E402

SEED = 0x5EED


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


def run_case(c, name, d, n, ib, keys, bern, param, iters):
    out, m = C.c_void_p(), C.c_size_t()
    fn = c.L.tg_bernoulli_sample if bern else c.L.tg_sample

    def call():
        c.ck(fn(c.h, ib, d, n, param, SEED, C.byref(out), C.byref(m)))
    med, best = timed(c, call, iters)
    c.profile_enable(True)
    call()
    kern = c.profile_list(capi.K_SAMPLE)
    c.profile_enable(False)
    # launch order: Sample = histogram, pick, gather, (candidate histogram, pick) x 5, count, tile scan, write;
    # BernoulliSample = count, tile scan, write
    if bern:
        passes = {"count": kern[0], "write": kern[2]}
        small = kern[1]
    else:
        passes = {"hist": kern[0], "gather": kern[2], "count": kern[-3], "write": kern[-1]}
        small = sum(kern) - sum(passes.values())
    if bern:
        mask = (keys >> np.uint64(11)) < np.uint64(S.bernoulli_threshold(param))
    else:
        mask = keys <= np.partition(keys, param - 1)[param - 1]
    got = c.download(out.value, m.value * ib).view(np.uint64)
    pos = got[::ib // 8]                            # the first word of every item is its position
    ok = m.value == int(mask.sum()) and np.array_equal(pos, np.flatnonzero(mask).astype(np.uint64))
    moved = m.value * ib * 2                        # the write reads and writes s bytes per kept item
    print("%-22s n=%.0e  %.3f ms (min %.3f); kernels %.3f ms: %s, small kernels %.3f; write moves %.0f MB (%.2f TB/s); kept %d; %s"
          % (name, n, med, best, sum(kern), ", ".join("%s %.3f" % kv for kv in passes.items()), small, moved / 1e6,
             moved / passes["write"] / 1e9 if passes["write"] > 0 else 0.0, m.value,
             "equal to the model" if ok else "DIFFERENT from the model"), flush=True)
    return ok


def main():
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print("card: %s" % card(), flush=True)
    n = 100_000_000
    c = capi.Ctx(0)
    x = np.arange(n, dtype=np.uint64)
    keys = S.keys(SEED, x)
    d = c.to_device(x)
    ok = True
    ok = run_case(c, "Sample(10) u64", d, n, 8, keys, False, 10, iters) and ok
    ok = run_case(c, "Sample(5e7) u64", d, n, 8, keys, False, 50_000_000, iters) and ok
    ok = run_case(c, "BernoulliSample(0.01)", d, n, 8, keys, True, 0.01, iters) and ok
    ok = run_case(c, "BernoulliSample(0.5)", d, n, 8, keys, True, 0.5, iters) and ok
    # 5e7 pairs: the same 800 MB as (position, position + n) pairs
    h = n // 2
    pairs = np.stack([x[:h], x[:h] + np.uint64(n)], axis=1)
    dp = c.to_device(pairs)
    ok = run_case(c, "Sample(10) pairs", dp, h, 16, keys[:h], False, 10, iters) and ok
    c.free(dp)
    del pairs
    f = capi.DevFile(d, n, 8, 0)
    host = c.host_alloc(n * 8)
    blk = (capi.Block * 1)()
    blk[0].data, blk[0].bytes = host.ctypes.data, n * 8

    def fetch():
        c.ck(c.L.tg_dev_file_fetch(c.h, C.byref(f), blk, 1))
    med, best = timed(c, fetch, max(3, iters // 2))
    ok = ok and np.array_equal(host.view(np.uint64), x)
    print("%-22s n=%.0e  %.3f ms (min %.3f) = %.1f GB/s D2H into page-locked memory" % ("fetch", n, med, best, n * 8 / best / 1e6),
          flush=True)
    c.host_free(host)
    c.free(d)
    c.close()
    print("card: %s" % card(), flush=True)
    print("ALL_OK" if ok else "MISMATCH", flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
