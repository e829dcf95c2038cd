#!/usr/bin/env python
"""GroupByKey / GroupToIndex fixtures (tests/golden/reference_outputs_group.npz): the UNMODIFIED reference's DIA::GroupByKey and
DIA::GroupToIndex (oracle/_ref/host/ref_group_driver, tests/host/ref_group_driver.cpp) on fixed inputs, at 1, 2, 3, 4 and 8
workers.  The group functions are those of group_ref.py (stats, and the partial function for GroupByKey); their rows carry the
worker's rank and come in worker order, so the placement is recorded too.
For each shape it stores the input (<name>/in: pair<u64, u64>) and, per case and worker count p:
    <name>/<case>_p<p>          the rows (n x 7 uint64), or the sha256 of their bytes (uint8) for the larger outputs
    <name>/<case>_p<p>_counts   the rows of each worker
<case> is key_stats, key_partial or index_<size>.
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_group_driver.mk):
    python tests/golden/make_golden_group.py"""
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import group_ref as G  # noqa: E402

DIGEST_ABOVE = 500            # rows
WORKERS = (1, 2, 3, 4, 8)
DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_group_driver")


def run_driver(workers, in_path, out_path, args):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([DRIVER, in_path, out_path] + args, env=env, capture_output=True, text=True, timeout=1800)
    if res.returncode != 0:
        raise RuntimeError("ref_group_driver failed: %s\n%s" % (res.returncode, res.stderr[-2000:]))
    return np.fromfile(out_path, dtype=np.uint64).reshape(-1, 7)


def shapes():
    """(name, input, cases): a case is ("key", fn) or ("index", size)"""
    by_key = [("key", G.STATS), ("key", G.PARTIAL)]
    i = np.arange(5000, dtype=np.uint64)
    vals = G.splitmix64(i + np.uint64(77))
    yield "identity_5000", G.pairs(i, vals), by_key + [("index", 5000)]
    j = np.arange(8000, dtype=np.uint64)
    yield "mod7_8000", G.pairs(j % np.uint64(7), G.splitmix64(j)), by_key + [("index", 7)]
    yield "splitmix_2000", G.pairs(G.splitmix64(j) % np.uint64(2000), j * np.uint64(3)), by_key + [("index", 2000)]
    yield "key0", G.pairs(np.zeros(1000), i[:1000] + np.uint64(5)), by_key + [("index", 1)]
    yield "one_key", G.pairs(np.full(3000, 123456789), G.splitmix64(i[:3000])), by_key
    yield "empty", G.pairs([], []), by_key + [("index", 10)]
    yield "multiples_of_8", G.pairs((G.splitmix64(i) % np.uint64(500)) * np.uint64(8), i), by_key
    yield "bit63", G.pairs((G.splitmix64(i + np.uint64(1)) % np.uint64(300)) | np.uint64(1 << 63), i * np.uint64(5)), by_key
    # GroupToIndex: missing indices, a size not divisible by p, a size below p (empty ranges) and size 1
    k = G.splitmix64(i[:3000] + np.uint64(9)) % np.uint64(1003)
    k = k[(k % np.uint64(3)) != 0]
    yield "index_missing_1003", G.pairs(k, np.arange(len(k))), [("index", 1003), ("index", 1009)]
    yield "index_small", G.pairs([0, 2, 2, 0, 2], [1, 2, 3, 4, 5]), [("index", 3), ("index", 5)]
    yield "index_size1", G.pairs(np.zeros(7), np.arange(7)), [("index", 1)]
    # a small PageRank-like edge list (src, dst), grouped by source into link lists
    rng = np.random.RandomState(5)
    nodes = 300
    src = (rng.zipf(1.5, 2500) - 1) % nodes
    dst = rng.randint(0, nodes, 2500)
    yield "pagerank_edges", G.pairs(src, dst), [("index", nodes)] + by_key


def case_name(case):
    return "key_" + case[1] if case[0] == "key" else "index_%d" % case[1]


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_group_driver.mk"
    tmp = tempfile.mkdtemp()
    ip, op = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
    g = {}
    for name, inp, cases in shapes():
        inp.tofile(ip)
        g[name + "/in"] = inp.view(np.uint64)
        for case in cases:
            args = ["key", case[1]] if case[0] == "key" else ["index", "stats", str(case[1])]
            for p in WORKERS:
                rows = run_driver(p, ip, op, args)
                counts = np.bincount(rows[:, 0].astype(np.int64), minlength=p).astype(np.int64)
                assert np.all(np.diff(rows[:, 0].astype(np.int64)) >= 0), (name, case, p)
                key = "%s/%s_p%d" % (name, case_name(case), p)
                g[key + "_counts"] = counts
                if len(rows) > DIGEST_ABOVE:
                    g[key] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest(), np.uint8)
                else:
                    g[key] = rows
                print(name, case_name(case), p, len(rows), flush=True)
    np.savez_compressed(os.path.join(HERE, "reference_outputs_group.npz"), **g)
    print("wrote reference_outputs_group.npz")


if __name__ == "__main__":
    main()
