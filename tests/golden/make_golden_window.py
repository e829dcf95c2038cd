#!/usr/bin/env python
"""Window fixtures (tests/golden/reference_outputs_window.npz): the UNMODIFIED reference's DIA::Window(k, WindowFold),
Window(k, WindowFold, WindowFold) and Window(DisjointTag, k, DisjointFold) (oracle/_ref/host/ref_window_driver,
tests/host/ref_window_driver.cpp) with every function on uint64_t, double and pairs, at 1, 2, 3, 4 and 8 workers.
Each worker's shard is placed with ConcatToDIA, so the per-worker sizes are chosen here: even, uneven, an empty first, middle or
last worker, one worker holding everything, and workers holding fewer than k - 1 items (the halo of the next ones spans several
predecessors).  Sizes per k: N < k - 1, N = k - 1, N = k, N mod k = 0 and N mod k != 0 (at k = 4096: k - 2, k - 1, k, k + 5 and
2k, N = 2k in the full and disjoint forms).  Every function at every k, with one deliberate gap to keep the file small: at
k = 4096 a partial Window emits about 4096 suffixes whatever N is, and an overlapping one at N = 2k about 4096 windows, so those
two are recorded for four functions only (BIG_K_MODES); the GPU tests cover every function there against the model.  One input
per item type, shared: a case takes its first N items.  The concatenation of the workers' outputs is the same for every worker count (checked here: a
difference would be a finding about the stock node), so it is stored once per case, with every worker count's per-worker
output counts.  The layout is described in tests/window_ref.py.
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_window_driver.mk):
    python tests/golden/make_golden_window.py"""
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import scan_ref as S  # noqa: E402
import window_ref as W  # noqa: E402

DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_window_driver")
SCHEMES = ["even", "uneven", "empty_first", "empty_mid", "empty_last", "one_holds_all", "small"]
KS = [2, 3, 5, 64, 4096]
QNAN = 0x7FF8000000000000
NAN_PAYLOAD = 0x7FF8000000012345
NMAX = 3 * 4096 + 7


def counts_for(scheme, n, p, k):
    if p == 1:
        return [n]
    if scheme == "even":
        return S.even_counts(n, p)
    if scheme == "uneven":
        w = [(r + 1) * (r + 1) for r in range(p)]
        c = [n * w[r] // sum(w) for r in range(p)]
        c[-1] += n - sum(c)
        return c
    if scheme == "empty_first":
        return [0] + S.even_counts(n, p - 1)
    if scheme == "empty_mid":
        c = S.even_counts(n, p - 1)
        return c[:p // 2] + [0] + c[p // 2:]
    if scheme == "empty_last":
        return S.even_counts(n, p - 1) + [0]
    if scheme == "one_holds_all":
        return [0, n] + [0] * (p - 2)
    if scheme == "small":                           # p - 1 workers of fewer than k - 1 items, the last one the rest
        s = min(max(1, (k - 1) // 3), n // p)
        return [s] * (p - 1) + [n - s * (p - 1)]
    raise ValueError(scheme)


def inputs():
    """one (NMAX, 2) word array per item type: u64, f64, pair_u64, pair_f64"""
    rng = np.random.RandomState(23)
    i = np.arange(NMAX, dtype=np.uint64)
    u = S.splitmix64(i) | np.uint64(1 << 63)        # sums wrap
    u[::5] = rng.randint(0, 1000, len(u[::5])).astype(np.uint64)
    mags = 10.0 ** rng.randint(-12, 13, NMAX)
    d = rng.standard_normal(NMAX) * mags
    d[3::29] = 0.0
    d[4::29] = -0.0
    d[5::31] = -0.0
    d[6::31] = 0.0
    f = S.f64_words(d)
    f[0] = NAN_PAYLOAD                              # the first window's first item
    f[[9, 70, 4100, 8200]] = NAN_PAYLOAD
    f[[40, 5000]] = QNAN
    f[[64, 127, 4096]] = S.f64_words(np.array([np.inf, -np.inf, np.inf]))
    keys = S.splitmix64(i + np.uint64(7))
    out = {}
    for name, vals in (("u64", u), ("f64", f)):
        out[name] = np.stack([np.zeros(NMAX, np.uint64), vals], axis=1)
        out["pair_" + name] = np.stack([keys, vals], axis=1)
    return out


def sizes(k):
    if k == KS[-1]:
        return [k - 2, k - 1, k, k + 5, 2 * k]
    return [max(0, k - 2), k - 1, k, 3 * k, 2 * k + 1 + k // 3]


# at k = 4096 a partial Window emits about 4096 suffixes whatever N is, and an overlapping one at N = 2k about 4096 windows:
# those two are recorded for a few functions only, to keep the file small
BIG_K_MODES = ("u64_sum", "f64_sum", "f64_max", "pair_f64_min")


def big_k_skip(mode, form, N, k):
    if mode in BIG_K_MODES:
        return form == "partial" and N not in (k - 1, k + 5)
    return form == "partial" or (form == "full" and N == 2 * k)


def cases():
    """(name, mode, form, k, input key, N, schemes for p = 2, 3, 4, 8)"""
    c = 0
    for mode in W.MODES:
        for form in W.FORMS:
            for k in KS:
                for N in sizes(k):
                    if k == KS[-1] and big_k_skip(mode, form, N, k):
                        continue
                    sch = [SCHEMES[(c + t) % len(SCHEMES)] for t in range(4)]
                    c += 1
                    yield "%s_%s_k%d_n%d" % (mode, form, k, N), mode, form, k, mode.split("_")[0] if not mode.startswith(
                        "pair_") else "pair_" + mode.split("_")[1], N, sch


def run_driver(workers, in_path, out_path, mode, form, k, cnt):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    args = [DRIVER, in_path, out_path, mode, form, str(k)] + [str(c) for c in cnt]
    res = subprocess.run(args, env=env, capture_output=True, text=True, timeout=600)
    if res.returncode != 0:
        raise RuntimeError("ref_window_driver failed: %s %s\n%s" % (args, res.returncode, res.stderr[-2000:]))
    return [np.fromfile("%s.%d" % (out_path, r), dtype=np.uint64).reshape(-1, 2) for r in range(workers)]


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_window_driver.mk"
    tmp = tempfile.mkdtemp()
    ins = inputs()
    keys = sorted(ins)
    paths = {}
    for key in keys:
        paths[key] = {}
    jobs, meta, names, shards = [], [], [], []
    for name, mode, form, k, key, N, sch in cases():
        if N not in paths[key]:
            p = os.path.join(tmp, "%s_%d.in" % (key, N))
            ins[key][:N].reshape(-1).tofile(p) if key.startswith("pair_") else ins[key][:N, 1].tofile(p)
            paths[key][N] = p
        c = len(names)
        names.append(name)
        meta.append([W.MODES.index(mode), W.FORMS.index(form), k, keys.index(key), N])
        sh = np.zeros((len(W.WORKERS), 8), np.int64)
        for w, p in enumerate(W.WORKERS):
            cnt = counts_for(sch[w - 1] if p > 1 else "even", N, p, k)
            sh[w, :p] = cnt
            jobs.append((c, w, paths[key][N], os.path.join(tmp, "%d.p%d.out" % (c, p)), mode, form, k, cnt))
        shards.append(sh)
    counts = np.zeros((len(names), len(W.WORKERS), 8), np.int64)
    outs = [None] * len(names)

    def run(job):
        c, w, ip, op, mode, form, k, cnt = job
        return c, w, run_driver(W.WORKERS[w], ip, op, mode, form, k, cnt)

    with ThreadPoolExecutor(12) as ex:
        for c, w, res in ex.map(run, jobs):
            counts[c, w, :len(res)] = [len(r) for r in res]
            cat = np.concatenate(res) if res else np.zeros((0, 2), np.uint64)
            if outs[c] is None:
                outs[c] = cat
            elif not np.array_equal(outs[c], cat):
                raise RuntimeError("finding: %s at %d workers differs from another worker count" % (names[c], W.WORKERS[w]))
    out_start = np.cumsum([0] + [len(o) for o in outs]).astype(np.int64)
    in_start = np.cumsum([0] + [2 * NMAX] * len(keys)).astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "reference_outputs_window.npz"), names=np.array(names), meta=np.array(meta, np.int64),
                        input_keys=np.array(keys), in_start=in_start, words=np.concatenate([ins[key].reshape(-1) for key in keys]),
                        out_start=out_start, outputs=np.concatenate(outs), counts=counts, shards=np.array(shards))
    print("wrote reference_outputs_window.npz: %d cases, %d driver runs" % (len(names), len(jobs)))


if __name__ == "__main__":
    main()
