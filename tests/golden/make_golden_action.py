#!/usr/bin/env python
"""Sum / Min / Max / AllReduce fixtures (tests/golden/reference_outputs_action.npz): the UNMODIFIED reference's DIA::Sum, Min, Max
and AllReduce (oracle/_ref/host/ref_action_driver, tests/host/ref_action_driver.cpp) on fixed inputs at 1, 2, 3, 4 and 8 workers,
with and without an initial value.  Each worker's shard is placed with ConcatToDIA, so the per-worker sizes are chosen here:
even, uneven, an empty first, middle or last worker, or one worker holding everything.
The inputs are shared: one array per dataset and item type, whatever the function, initial value or placement.  The layout
(a few arrays, not one entry per case) is described in tests/action_ref.py.
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_action_driver.mk):
    python tests/golden/make_golden_action.py"""
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import action_ref as A  # noqa: E402
import scan_ref as S  # noqa: E402

WORKERS = A.WORKERS
SCHEMES = ["even", "uneven", "empty_first", "empty_mid", "empty_last", "one_holds_all"]
DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_action_driver")
U64 = (1 << 64) - 1
NEG0 = 0x8000000000000000
QNAN = 0x7FF8000000000000
NAN_PAYLOAD = 0x7FF8000000012345             # a NaN with a payload: which NaN comes out is visible in the bits


def counts_for(scheme, n, p):
    if p == 1:
        return [n]
    if scheme == "even":
        return S.even_counts(n, p)
    if scheme == "uneven":                          # sizes growing with the rank, the last worker takes the rest
        w = [(r + 1) * (r + 1) for r in range(p)]
        c = [n * w[r] // sum(w) for r in range(p)]
        c[-1] += n - sum(c)
        return c
    if scheme == "empty_first":
        return [0] + S.even_counts(n, p - 1)
    if scheme == "empty_mid":                       # worker p // 2 holds nothing
        c = S.even_counts(n, p - 1)
        return c[:p // 2] + [0] + c[p // 2:]
    if scheme == "empty_last":
        return S.even_counts(n, p - 1) + [0]
    if scheme == "one_holds_all":                   # worker 1 holds everything, the others nothing
        return [0, n] + [0] * (p - 2)
    raise ValueError(scheme)


def f64(x):
    return S.f64_words(x)


def datasets(kind, rng):
    """(name, value words) of one value type"""
    if kind == "u64":
        i = np.arange(300, dtype=np.uint64)
        yield "wrap", S.splitmix64(i) | np.uint64(1 << 63)                   # sums wrap many times
        yield "small", (rng.randint(1, 1000, 250)).astype(np.uint64)      # positive: an empty worker's T() = 0 is the Min
        return
    mags = 10.0 ** rng.randint(-12, 13, 300)
    mixed = rng.standard_normal(300) * mags
    mixed[::97] = 0.0
    mixed[5::101] = -0.0
    yield "mixed", f64(mixed)
    pos = rng.uniform(1.0, 100.0, 150)
    a = f64(pos)
    a[0] = NAN_PAYLOAD
    yield "nan_first", a
    b = f64(pos)
    b[[7, 70, 149]] = [QNAN, NAN_PAYLOAD, QNAN]
    yield "nan_later", b
    z = f64(np.concatenate([pos[:40], [0.0, -0.0], pos[40:90], [-0.0, 0.0], -pos[90:120], [0.0, -0.0]]))
    yield "zeros_pos_neg", z                        # +-0 ties in both orders among positives and negatives
    z2 = f64(np.concatenate([pos[:30], [-0.0, 0.0, -0.0], pos[30:70]]))
    yield "zeros_neg_first", z2
    w = rng.standard_normal(200)
    w[[30, 130]] = [np.inf, -np.inf]
    yield "inf_both", f64(w)
    w2 = rng.standard_normal(200)
    w2[100] = -np.inf
    yield "inf_neg", f64(w2)
    yield "all_negzero", f64(np.full(100, -0.0))


def cases():
    """(name, mode, initial words (first, value) or None, input key, input words, schemes)"""
    rng = np.random.RandomState(17)
    data = {kind: list(datasets(kind, rng)) for kind in ("u64", "f64")}
    keys = S.splitmix64(np.arange(1000, dtype=np.uint64) + np.uint64(99))          # the .first of pair items
    k = 0
    for mode in A.MODES:
        op, pair = A.mode_op(mode)
        kind = "f64" if op in A.F64_OPS else "u64"
        for dname, vals in data[kind]:
            if pair and dname not in ("wrap", "small", "mixed", "nan_first", "zeros_pos_neg", "all_negzero"):
                continue
            if not pair and kind == "f64" and op == A.OP_SUM_F64 and dname.startswith("zeros"):
                continue
            inits = [None, (77, 12345 if kind == "u64" else int(f64([2.5])[0]))]
            if kind == "u64":
                inits.append((5, U64 - 3))
            elif op != A.OP_SUM_F64 or dname == "all_negzero":
                inits.append((5, NEG0))
            if kind == "f64" and op != A.OP_SUM_F64 and dname in ("mixed", "zeros_pos_neg"):
                inits.append((9, NAN_PAYLOAD))
            words = S.pairs(keys[:len(vals)], vals).view(np.uint64) if pair else vals
            in_key = "%s%s_%s" % ("pair_" if pair else "", kind, dname)
            for init in inits:
                schemes = [SCHEMES[k % len(SCHEMES)], SCHEMES[(k + 3) % len(SCHEMES)]]
                k += 1
                tag = "none" if init is None else "init%d" % inits.index(init)
                yield ("%s_%s_%s" % (mode, dname, tag), mode, init, in_key, np.ascontiguousarray(words, np.uint64), pair,
                       schemes)


def run_driver(workers, in_path, out_path, mode, init, counts):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    i = init or (0, 0)
    args = [DRIVER, in_path, out_path, mode, "init" if init else "none", str(i[0]), str(i[1])] + [str(c) for c in counts]
    res = subprocess.run(args, env=env, capture_output=True, text=True, timeout=600)
    if res.returncode != 0:
        raise RuntimeError("ref_action_driver failed: %s\n%s" % (res.returncode, res.stderr[-2000:]))
    return np.fromfile(out_path, dtype=np.uint64)


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_action_driver.mk"
    tmp = tempfile.mkdtemp()
    jobs, names, meta, inputs = [], [], [], {}
    for name, mode, init, in_key, words, pair, schemes in cases():
        if in_key not in inputs:
            inputs[in_key] = (len(inputs), words)
            words.tofile(os.path.join(tmp, in_key + ".in"))
        n = len(words) // 2 if pair else len(words)
        for scheme in schemes:
            names.append("%s_%s" % (name, scheme))
            meta.append([A.MODES.index(mode), init is not None] + list(init or (0, 0)) + [inputs[in_key][0]])
            for k, p in enumerate(WORKERS):
                jobs.append((len(names) - 1, k, os.path.join(tmp, in_key + ".in"),
                             os.path.join(tmp, "%d.p%d.out" % (len(names) - 1, p)), mode, init, counts_for(scheme, n, p)))
    counts = np.zeros((len(names), len(WORKERS), 8), np.int64)
    results = np.zeros((len(names), len(WORKERS), 2), np.uint64)

    def run(job):
        c, k, ip, op, mode, init, cnt = job
        return c, k, cnt, run_driver(WORKERS[k], ip, op, mode, init, cnt)

    with ThreadPoolExecutor(8) as ex:
        for c, k, cnt, res in ex.map(run, jobs):
            assert len(res) == 2, (names[c], WORKERS[k])
            counts[c, k, :len(cnt)] = cnt
            results[c, k] = res
    order = sorted(inputs.values())
    in_start = np.cumsum([0] + [len(w) for _, w in order]).astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "reference_outputs_action.npz"), names=np.array(names), meta=np.array(meta, np.uint64),
                        in_start=in_start, words=np.concatenate([w for _, w in order]), counts=counts, results=results)
    print("wrote reference_outputs_action.npz: %d cases, %d inputs, %d driver runs" % (len(names), len(order), len(jobs)))


if __name__ == "__main__":
    main()
