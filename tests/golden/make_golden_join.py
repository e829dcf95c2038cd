#!/usr/bin/env python
"""InnerJoin fixtures (tests/golden/reference_outputs_join.npz): the UNMODIFIED reference's api::InnerJoin with the
(key, l.second, r.second) join function (oracle/_ref/host/ref_join_driver, tests/host/ref_join_driver.cpp) on fixed inputs, at 1
and at 3 workers.
For each shape it stores the inputs (<name>/left, <name>/right: pair<u64, u64>) and, per worker count p, the output multiset
(<name>/out_p<p>): the (key, v1, v2) rows sorted, or the sha256 of those rows' bytes (uint8) for the larger shapes.
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_join_driver.mk):
    python tests/golden/make_golden_join.py"""
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import join_ref as J  # noqa: E402

DIGEST_ABOVE = 4000           # rows
DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_join_driver")


def run_driver(workers, left_path, right_path, out_path):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([DRIVER, left_path, right_path, out_path], env=env, capture_output=True, text=True, timeout=1800)
    if res.returncode != 0:
        raise RuntimeError("ref_join_driver failed: %s\n%s" % (res.returncode, res.stderr[-2000:]))


def pairs(keys, vals):
    out = np.empty(len(keys), J.KV)
    out["key"], out["val"] = np.asarray(keys, np.uint64), np.asarray(vals, np.uint64)
    return out


def shapes():
    i = np.arange(9999, dtype=np.uint64)
    yield "identity_9999", pairs(i, i * np.uint64(3)), pairs(i, i + np.uint64(1000000))
    j = np.arange(333, dtype=np.uint64)
    yield "one_key_333x333", pairs(np.full(333, 1), j), pairs(np.full(333, 1), j * np.uint64(2))
    yield "small_100x333", pairs(np.arange(100) % 10, np.arange(100)), pairs(np.arange(333) % 7, np.arange(333) + 500)
    yield "disjoint", J.make_side(3000, 1000, 1), pairs(np.arange(3000) + 5000, np.arange(3000))
    yield "key0", pairs(np.arange(500) % 4, np.arange(500)), pairs(np.arange(300) % 3, np.arange(300) * 11)
    yield "empty_right", J.make_side(1000, 100, 2), np.zeros(0, J.KV)
    fk = J.make_side(20000, 1000, 3, zipf=1.0)
    yield "foreign_key_zipf", fk, pairs(np.arange(1, 1001), np.arange(1000) * 7 + 1)
    yield "zipf_many_to_many", J.make_side(2000, 100, 4, zipf=1.0), J.make_side(2000, 100, 5, zipf=1.0)


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_join_driver.mk"
    tmp = tempfile.mkdtemp()
    lp, rp, op = (os.path.join(tmp, x) for x in ("l.bin", "r.bin", "o.bin"))
    g = {}
    for name, left, right in shapes():
        left.tofile(lp)
        right.tofile(rp)
        g[name + "/left"], g[name + "/right"] = left.view(np.uint64), right.view(np.uint64)
        for p in (1, 3):
            run_driver(p, lp, rp, op)
            rows = np.fromfile(op, dtype=np.uint64).reshape(-1, 3)
            rows = rows[np.lexsort(rows.T[::-1])]
            assert len(rows) == J.output_counts(left, right), (name, p, len(rows))
            if len(rows) > DIGEST_ABOVE:
                g["%s/out_p%d" % (name, p)] = np.frombuffer(hashlib.sha256(np.ascontiguousarray(rows).tobytes()).digest(), np.uint8)
            else:
                g["%s/out_p%d" % (name, p)] = rows
            print(name, p, len(rows), flush=True)
    np.savez_compressed(os.path.join(HERE, "reference_outputs_join.npz"), **g)
    print("wrote reference_outputs_join.npz")


if __name__ == "__main__":
    main()
