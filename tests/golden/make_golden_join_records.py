#!/usr/bin/env python
"""InnerJoin-on-records fixtures (tests/golden/reference_outputs_join_records.npz): the UNMODIFIED reference's api::InnerJoin with
a key field extractor on each side and (l, r) -> std::make_pair(l, r) (oracle/_ref/host/ref_join_records_driver,
tests/host/ref_join_records_driver.cpp), at 1, 2, 3 and 4 workers on the mock network.
The inputs are generated, not stored: each case records the driver's shape, and per side (left, then right) the item size, the key
(offset, bytes), the item count, the record seed and the key draw (uniform over a universe, Zipf over a universe with skew, or
one key), all in <name>/params; the records come from join_records_ref.make_records and set_keys, and <name>/inputs holds the
digest (join_records_ref.digest) of each side so a change of the generator is caught.  Per worker count p, <name>/out_p<p>
holds the output multiset: the rows sorted (join_records_ref.multiset) where they take at most 64 KiB, the order-independent
digest (count, sum, xor) as uint64 for the larger ones.
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_join_records_driver.mk):
    python tests/golden/make_golden_join_records.py"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import join_records_ref as J  # noqa: E402

ROW_BYTES_ABOVE_DIGEST = 64 << 10
DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_join_records_driver")
UNIFORM, ZIPF, ONE_KEY = J.UNIFORM, J.ZIPF, J.ONE_KEY

# name: (driver shape, left side, right side); side = (item bytes, key offset, key bytes, n, seed, draw, universe, skew x 100)
CASES = {
    "w4_uniform": ("w4", (4, 0, 4, 3000, 1, UNIFORM, 1000, 0), (4, 0, 4, 2000, 2, UNIFORM, 1000, 0)),
    "r12x24_zipf": ("r12x24", (12, 5, 2, 4000, 3, ZIPF, 500, 100), (24, 3, 5, 3000, 4, ZIPF, 500, 100)),
    "r24x8_key_at_end": ("r24x8", (24, 3, 5, 2500, 5, UNIFORM, 4000, 0), (8, 3, 5, 2500, 6, UNIFORM, 4000, 0)),
    "r24x8_many_to_many": ("r24x8", (24, 3, 5, 3000, 7, UNIFORM, 300, 0), (8, 3, 5, 1000, 8, UNIFORM, 300, 0)),
    "tpch_176x152": ("r176x152", (176, 0, 8, 6000, 9, UNIFORM, 1500, 0), (152, 0, 8, 1500, 10, UNIFORM, 1500, 0)),
    "pair8": ("pair8", (16, 0, 8, 5000, 11, ZIPF, 2000, 110), (16, 0, 8, 4000, 12, UNIFORM, 2000, 0)),
    "pair24": ("pair24", (16, 0, 8, 3000, 13, UNIFORM, 1000, 0), (32, 0, 8, 2000, 14, UNIFORM, 1000, 0)),
    "empty_left": ("r12x24", (12, 5, 2, 0, 15, UNIFORM, 100, 0), (24, 3, 5, 500, 16, UNIFORM, 100, 0)),
    "empty_both": ("w4", (4, 0, 4, 0, 17, UNIFORM, 100, 0), (4, 0, 4, 0, 18, UNIFORM, 100, 0)),
    "one_hot_key": ("r24x8", (24, 3, 5, 150, 19, ONE_KEY, 0, 0), (8, 3, 5, 120, 20, ONE_KEY, 0, 0)),
    "self24": ("self24", (24, 3, 5, 3000, 21, UNIFORM, 800, 0), (24, 3, 5, 3000, 21, UNIFORM, 800, 0)),
}


def run_driver(shape, workers, lp, rp, op):
    env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(workers), THRILL_LOG="")
    res = subprocess.run([DRIVER, shape, lp, rp, op], env=env, capture_output=True, text=True, timeout=1800)
    if res.returncode != 0:
        raise RuntimeError("ref_join_records_driver failed: %s\n%s" % (res.returncode, res.stderr[-2000:]))


def main():
    assert os.access(DRIVER, os.X_OK), "build the driver first: make -C oracle ref && make -C tests/host -f ref_join_records_driver.mk"
    tmp = tempfile.mkdtemp()
    lp, rp, op = (os.path.join(tmp, x) for x in ("l.bin", "r.bin", "o.bin"))
    g = {}
    for name, (shape, ls, rs) in CASES.items():
        left, right = J.side_from_params(ls), J.side_from_params(rs)
        left.tofile(lp)
        right.tofile(rp)
        g[name + "/params"] = np.array(list(ls) + list(rs), np.uint64)
        g[name + "/inputs"] = np.array(J.digest(left) + J.digest(right), np.uint64)
        s = ls[0] + rs[0]
        m = J.output_count(J.keys_of(left, ls[1], ls[2]), J.keys_of(right, rs[1], rs[2]))
        for p in (1, 2, 3, 4):
            run_driver(shape, p, lp, rp, op)
            rows = np.fromfile(op, dtype=np.uint8).reshape(-1, s)
            assert len(rows) == m, (name, p, len(rows), m)
            if rows.size > ROW_BYTES_ABOVE_DIGEST:
                g["%s/out_p%d" % (name, p)] = np.array(J.digest(rows), np.uint64)
            else:
                g["%s/out_p%d" % (name, p)] = J.multiset(rows)
            print(name, p, len(rows), flush=True)
    np.savez_compressed(os.path.join(HERE, "reference_outputs_join_records.npz"), **g)
    print("wrote reference_outputs_join_records.npz")


if __name__ == "__main__":
    main()
