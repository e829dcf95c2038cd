#!/usr/bin/env python
"""PrefixSum / ExPrefixSum / ZipWithIndex fixtures (tests/golden/reference_outputs_scan.npz): the UNMODIFIED reference's
DIA::PrefixSum, DIA::ExPrefixSum and DIA::ZipWithIndex (oracle/_ref/host/ref_scan_driver, tests/host/ref_scan_driver.cpp) on fixed
inputs at 1, 2, 3, 4 and 8 workers.  Each worker's shard is placed with ConcatToDIA, so the per-worker sizes are chosen here:
even, uneven, an empty worker in the middle, or one worker holding everything.
For each case it stores
    <case>/in          the input words (uint64; pairs as (first, second) words, doubles as their bits)
    <case>/meta        [mode index into MODES, inclusive, init_first, init_second, pair]
    <case>/p<p>/counts the items of each worker
    <case>/p<p>/rows   the outputs in worker order: n x 2 uint64 (first word, second word) of pairs, n uint64 of 8-byte items
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_scan_driver.mk):
    python tests/golden/make_golden_scan.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import scan_ref as S  # noqa: E402

WORKERS = (1, 2, 3, 4, 8)
MODES = ["sum_u64", "min_u64", "max_u64", "sum_f64", "pair_max", "pair_sum_f64", "zip_first", "zip_second"]
DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_scan_driver")
U64 = (1 << 64) - 1
NEG0 = 0x8000000000000000


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
    if scheme == "empty_mid":                       # worker p // 2 holds nothing
        c = S.even_counts(n, p - 1)
        return c[:p // 2] + [0] + c[p // 2:]
    if scheme == "one_holds_all":                   # worker 1 holds everything, the others nothing
        return [0, n] + [0] * (p - 2)
    raise ValueError(scheme)


def cases():
    """(name, mode, inclusive, (init_first, init_second), input words, scheme)"""
    rng = np.random.RandomState(11)
    i = np.arange(1000, dtype=np.uint64)
    big = S.splitmix64(i) | np.uint64(1 << 63)                     # wraps many times
    yield "sum_u64_wrap_incl", "sum_u64", 1, (0, 12345), big, "uneven"
    yield "sum_u64_wrap_excl", "sum_u64", 0, (0, U64 - 7), big, "empty_mid"
    small = rng.randint(0, 1000, 1200).astype(np.uint64)
    yield "sum_u64_default_excl", "sum_u64", 0, (0, 0), small, "one_holds_all"
    desc = (np.uint64(1 << 40) - S.splitmix64(i) % np.uint64(1 << 20) * i)
    yield "min_u64_init_max_incl", "min_u64", 1, (0, U64), desc, "even"
    yield "min_u64_init_max_excl", "min_u64", 0, (0, U64), desc, "empty_mid"
    yield "max_u64_incl", "max_u64", 1, (0, 0), S.splitmix64(i + np.uint64(5)) >> np.uint64(rng.randint(0, 40)), "uneven"
    yield "max_u64_init_excl", "max_u64", 0, (0, 1 << 62), S.splitmix64(i + np.uint64(9)), "even"
    mags = 10.0 ** rng.randint(-12, 13, 1500)
    mixed = rng.standard_normal(1500) * mags
    mixed[::97] = 0.0
    mixed[5::101] = -0.0
    yield "sum_f64_mixed_incl", "sum_f64", 1, (0, 0), S.f64_words(mixed), "uneven"
    yield "sum_f64_mixed_excl", "sum_f64", 0, (0, int(S.f64_words([2.5])[0])), S.f64_words(mixed), "empty_mid"
    negz = S.f64_words(np.full(700, -0.0))
    yield "sum_f64_negzero_incl", "sum_f64", 1, (0, NEG0), negz, "even"
    yield "sum_f64_negzero_excl", "sum_f64", 0, (0, NEG0), negz, "one_holds_all"
    yield "sum_f64_negzero_default_incl", "sum_f64", 1, (0, 0), negz, "even"
    special = rng.standard_normal(900)
    special[300] = np.inf
    special[600] = -np.inf
    special[750] = np.nan
    yield "sum_f64_inf_nan_incl", "sum_f64", 1, (0, 0), S.f64_words(special), "uneven"
    special2 = rng.standard_normal(900)
    special2[450] = np.inf
    yield "sum_f64_inf_excl", "sum_f64", 0, (0, 0), S.f64_words(special2), "even"
    # prefix doubling's names: (index, rank) pairs; rank = 0 where a new name starts, else the position in a run
    idx = np.arange(1400, dtype=np.uint64)
    names = np.where(rng.randint(0, 4, 1400) == 0, idx + np.uint64(1), np.uint64(0))
    pw = np.stack([S.splitmix64(idx) % np.uint64(1 << 32), names], axis=1).reshape(-1)
    yield "pair_max_names_incl", "pair_max", 1, (0, 0), pw, "empty_mid"
    yield "pair_max_names_excl", "pair_max", 0, (77, 3), pw, "empty_mid"
    yield "pair_max_names_all_excl", "pair_max", 0, (0, 0), pw, "one_holds_all"
    pv = rng.standard_normal(1100) * 10.0 ** rng.randint(-6, 7, 1100)
    pf = np.stack([S.splitmix64(np.arange(1100, dtype=np.uint64)), S.f64_words(pv)], axis=1).reshape(-1)
    yield "pair_sum_f64_incl", "pair_sum_f64", 1, (0, 0), pf, "empty_mid"
    yield "pair_sum_f64_excl", "pair_sum_f64", 0, (5, int(S.f64_words([-1.25])[0])), pf, "empty_mid"
    zw = S.splitmix64(np.arange(1300, dtype=np.uint64) + np.uint64(3))
    yield "zip_first_uneven", "zip_first", 1, (0, 0), zw, "uneven"
    yield "zip_second_uneven", "zip_second", 1, (0, 0), zw, "uneven"
    yield "zip_first_empty_mid", "zip_first", 1, (0, 0), zw[:500], "empty_mid"


def run_driver(workers, in_path, out_path, mode, inclusive, init, counts):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    args = [DRIVER, in_path, out_path, mode, "incl" if inclusive else "excl", str(init[0]), str(init[1])] + [str(c) for c in counts]
    res = subprocess.run(args, env=env, capture_output=True, text=True, timeout=600)
    if res.returncode != 0:
        raise RuntimeError("ref_scan_driver failed: %s\n%s" % (res.returncode, res.stderr[-2000:]))
    return np.fromfile(out_path, dtype=np.uint64).reshape(-1, 3)


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_scan_driver.mk"
    tmp = tempfile.mkdtemp()
    ip, op = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    g = {}
    for name, mode, inclusive, init, words, scheme in cases():
        words = np.ascontiguousarray(words, np.uint64)
        pair = mode.startswith("pair_")
        n = len(words) // 2 if pair else len(words)
        words.tofile(ip)
        g[name + "/in"] = words
        g[name + "/meta"] = np.array([MODES.index(mode), inclusive, init[0], init[1], int(pair)], np.uint64)
        for p in WORKERS:
            counts = counts_for(scheme, n, p)
            rows = run_driver(p, ip, op, mode, inclusive, init, counts)
            assert len(rows) == n and np.array_equal(rows[:, 0], np.repeat(np.arange(p), counts).astype(np.uint64)), (name, p)
            g["%s/p%d/counts" % (name, p)] = np.array(counts, np.int64)
            # (the rank column follows from the counts, and an 8-byte output's first word is 0: neither is stored)
            g["%s/p%d/rows" % (name, p)] = rows[:, 1:] if pair or mode.startswith("zip_") else rows[:, 2]
            print(name, p, counts, flush=True)
    np.savez_compressed(os.path.join(HERE, "reference_outputs_scan.npz"), **g)
    print("wrote reference_outputs_scan.npz")


if __name__ == "__main__":
    main()
