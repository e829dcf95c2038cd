#!/usr/bin/env python
"""HyperLogLog fixtures (tests/golden/reference_outputs_hll.npz): the UNMODIFIED reference's core::HyperLogLogRegisters<p>
(oracle/_ref/host/ref_hll_driver, tests/host/ref_hll_driver.cpp) on fixed inputs at p = 4, 8, 12, 14, 16 and 18: the registers (a)
of an object that is dense from the first item on, and the natural path (every worker starts sparse, operator + in rank order)
at 1, 2, 3, 4 and 8 workers with even, uneven and empty shards: whether it ends dense, whether its registers equal (a), and the
stock result() of both.  Inputs are stored once; the large all-distinct inputs are consecutive integers, kept as (start, words)
only.  Registers are kept whole where at most 1024 are non-zero, and as a SHA-256 digest always.  The layout is described in
tests/hll_ref.py.  Prints every case where the natural path's registers differ from (a).
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_hll_driver.mk):
    python tests/golden/make_golden_hll.py"""
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import hll_ref as H  # noqa: E402

DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_hll_driver")
KEEP_NONZERO = 1024


def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        z = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def inputs():
    """(name, mode, words or None, (start, nwords) of a range input)"""
    rng = np.random.RandomState(23)
    for mode, wpi in (("u64", 1), ("pair", 2)):
        def items(n, seed):
            return splitmix64(np.arange(n * wpi, dtype=np.uint64) + np.uint64(seed << 32))
        yield mode + "_empty", mode, np.zeros(0, np.uint64), None
        yield mode + "_one", mode, items(1, 1), None
        yield mode + "_all_equal", mode, np.tile(items(1, 2), 5000), None
        pool = items(50, 3).reshape(50, wpi)
        yield mode + "_few_distinct", mode, pool[rng.randint(0, 50, 4000)].reshape(-1), None
        yield mode + "_range_3000", mode, None, (1 << 20, 3000 * wpi)
        # all distinct, and enough of them that the stock sparse list outgrows 2^p bytes at every p
        n = 200000 if mode == "u64" else 150000
        yield mode + "_range_%d" % n, mode, None, (1 << 40, n * wpi)
    d = rng.randint(-4000, 4000, 2000) / 8.0              # doubles are hashed as their bits: +0.0 and -0.0 are two items
    d[::50] = 0.0
    d[7::50] = -0.0
    yield "u64_doubles", "u64", np.ascontiguousarray(d).view(np.uint64), None
    # hashes given to insert_hash directly: for every p some whose low 64 - p bits are all zero (w == 0), some with a single
    # low bit, and random ones
    h = [rng.randint(0, 1 << 62, 300, dtype=np.uint64) * np.uint64(4) + rng.randint(0, 4, 300, dtype=np.uint64)]
    for p in H.PRECISIONS:
        idx = rng.randint(0, 1 << p, 6, dtype=np.uint64)
        h.append(idx << np.uint64(64 - p))
        h.append((idx[:3] << np.uint64(64 - p)) | np.uint64(1))
        h.append((idx[3:] << np.uint64(64 - p)) | (np.uint64(1) << np.uint64(63 - p)))
    h.append(np.array([0, H.M64, 1, 1 << 63], np.uint64))
    yield "hash_edges", "hash", np.concatenate(h), None


def layouts(n):
    """per-worker item counts at 1, 2, 3, 4 and 8 workers: even, uneven, empty shards first, in the middle and last"""
    def even(m, p):
        return [m // p + (1 if r < m % p else 0) for r in range(p)]
    w = [(r + 1) * (r + 1) for r in range(7)]
    un = [n * x // sum(w) for x in w]
    un[0] += n - sum(un)
    return [[n], even(n, 2), [n - n // 3, 0, n // 3], [0] + even(n, 3), un + [0]]


def run_driver(in_path, out_path, mode, counts):
    res = subprocess.run([DRIVER, in_path, out_path, mode] + [str(c) for c in counts], capture_output=True, text=True, timeout=600)
    if res.returncode != 0:
        raise RuntimeError("ref_hll_driver failed: %s\n%s" % (res.returncode, res.stderr[-2000:]))
    raw = open(out_path, "rb").read()
    out, off = [], 0
    for p in H.PRECISIONS:
        m = 1 << p
        a = np.frombuffer(raw, np.uint8, m, off)
        b = np.frombuffer(raw, np.uint8, m, off + m)
        dense = int(np.frombuffer(raw, np.uint64, 1, off + 2 * m)[0])
        est = np.frombuffer(raw, np.float64, 2, off + 2 * m + 8)
        out.append((a, b, dense, float(est[0]), float(est[1])))
        off += 2 * m + 24
    assert off == len(raw)
    return out


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_hll_driver.mk"
    tmp = tempfile.mkdtemp()
    ins = list(inputs())
    jobs = []
    for i, (name, mode, words, rng_) in enumerate(ins):
        if words is None:
            words = np.uint64(rng_[0]) + np.arange(rng_[1], dtype=np.uint64)
        path = os.path.join(tmp, "%d.in" % i)
        words.tofile(path)
        n = len(words) // (2 if mode == "pair" else 1)
        for counts in layouts(n):
            jobs.append((i, path, os.path.join(tmp, "%d.out" % len(jobs)), mode, counts))
    with ThreadPoolExecutor(8) as ex:
        results = list(ex.map(lambda j: run_driver(j[1], j[2], j[3], j[4]), jobs))
    np_ = len(H.PRECISIONS)
    arrays = {}
    digest = np.zeros((len(ins), np_, 32), np.uint8)
    est_a = np.zeros((len(ins), np_))
    lay_counts = np.full((len(jobs), 8), -1, np.int64)
    lay_dense = np.zeros((len(jobs), np_), np.uint8)
    lay_equal = np.zeros((len(jobs), np_), np.uint8)
    lay_est = np.zeros((len(jobs), np_))
    differ = 0
    for j, (job, res) in enumerate(zip(jobs, results)):
        i = job[0]
        lay_counts[j, :len(job[4])] = job[4]
        for k, (a, b, dense, ea, eb) in enumerate(res):
            d = H.digest(a)
            assert not digest[i, k].any() or np.array_equal(digest[i, k], d), "(a) depends on nothing but the items"
            digest[i, k] = d
            est_a[i, k] = ea
            if np.count_nonzero(a) <= KEEP_NONZERO:
                arrays["regs_%d_%d" % (i, H.PRECISIONS[k])] = a
            lay_dense[j, k], lay_equal[j, k], lay_est[j, k] = dense, np.array_equal(a, b), eb
            if not np.array_equal(a, b):
                differ += 1
                at = np.flatnonzero(a != b)
                print("DIFFERS %s p=%d counts=%s: %d registers, first at %d: direct %d, natural %d"
                      % (ins[i][0], H.PRECISIONS[k], job[4], len(at), at[0], a[at[0]], b[at[0]]))
    stored = [w if w is not None else np.zeros(0, np.uint64) for _, _, w, _ in ins]
    np.savez_compressed(
        os.path.join(HERE, "reference_outputs_hll.npz"), precisions=np.array(H.PRECISIONS, np.int64),
        in_names=np.array([x[0] for x in ins]), in_mode=np.array([H.MODES.index(x[1]) for x in ins], np.int64),
        in_start=np.cumsum([0] + [len(w) for w in stored]).astype(np.int64), words=np.concatenate(stored),
        in_range=np.array([x[3] or (0, 0) for x in ins], np.uint64), digest=digest, est_a=est_a,
        lay_input=np.array([j[0] for j in jobs], np.int64), lay_counts=lay_counts, lay_dense=lay_dense, lay_equal=lay_equal,
        lay_est=lay_est, **arrays)
    print("wrote reference_outputs_hll.npz: %d inputs, %d driver runs, %d register sets kept whole; the natural path's registers "
          "differ from the direct ones in %d of %d results" % (len(ins), len(jobs), len(arrays), differ, len(jobs) * np_))


if __name__ == "__main__":
    main()
