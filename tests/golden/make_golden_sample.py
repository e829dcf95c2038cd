#!/usr/bin/env python
"""Sample / BernoulliSample fixtures (tests/golden/reference_outputs_sample.npz): the UNMODIFIED reference's DIA::Sample and
DIA::BernoulliSample (oracle/_ref/host/ref_sample_driver, tests/host/ref_sample_driver.cpp) at 1 to 4 workers, with the global
positions as items so that a sample names its positions.  Three parts:
  det_*   the deterministic cases: s >= N (everything, in input order, on its worker), N = 0, BernoulliSample(1) and (0), and
          Sample(s < n) on one worker, whose items are the reservoir's (random) but whose count is s.  det_exact says whether the
          items are deterministic; det_items holds every case's outputs, worker after worker, from det_offsets[c].
  sub_*   20 000 frozen runs of Sample(4) of 12 items, 5000 at each sharding of sub_sizes (the first sub_workers entries): the
          subset (sorted positions) and the per-worker counts of every run.
  bern_*  5000 frozen runs of BernoulliSample(p) of 64 items for p = 0.05 (the stock geometric skip path) and 0.3 (the
          Bernoulli path), at 1 and 3 workers: the kept positions of every run as a packed 64-bit mask.
Checks while generating that every worker emits a BernoulliSample's kept items in input order.
Needs the reference library and the driver (make -C oracle ref && make -C tests/host -f ref_sample_driver.mk):
    python tests/golden/make_golden_sample.py"""
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DRIVER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle", "_ref", "host", "ref_sample_driver")
OUT = os.path.join(HERE, "reference_outputs_sample.npz")

# (sizes, mode, param, exact): mode 0 Sample(param), 1 BernoulliSample(param)
DET = [
    ([0], 0, 5, True), ([12], 0, 12, True), ([12], 0, 100, True), ([12], 0, 4, False), ([100], 0, 99, False),
    ([0, 0], 0, 3, True), ([6, 6], 0, 12, True), ([0, 12], 0, 20, True), ([5, 7], 1, 1.0, True), ([5, 7], 1, 0.0, True),
    ([5, 0, 7], 0, 12, True), ([5, 0, 7], 0, 13, True), ([0, 0, 0], 0, 1, True), ([5, 0, 7], 1, 1.0, True),
    ([3, 3, 3, 3], 0, 12, True), ([0, 12, 0, 0], 0, 1000, True), ([0, 0, 0, 0], 0, 2, True), ([3, 0, 3, 6], 1, 1.0, True),
    ([3, 0, 3, 6], 1, 0.0, True), ([64], 1, 1.0, True), ([64], 1, 0.0, True),
]
SUB_SIZES = [[12], [6, 6], [5, 0, 7], [3, 3, 3, 3]]
SUB_REPS = 5000
BERN = [(0.05, [64]), (0.05, [20, 0, 44]), (0.3, [64]), (0.3, [20, 0, 44])]
BERN_REPS = 5000


def run_driver(sizes, mode, param, reps):
    """per rep, the outputs of every worker in its emit order: a list of reps lists of W arrays"""
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "out")
        env = dict(os.environ, THRILL_NET="mock", THRILL_LOCAL="1", THRILL_WORKERS_PER_HOST=str(len(sizes)), THRILL_LOG="")
        args = [DRIVER, out, "bernoulli" if mode else "sample", repr(float(param)) if mode else str(int(param)), str(reps)]
        res = subprocess.run(args + [str(s) for s in sizes], env=env, capture_output=True, text=True, timeout=600)
        if res.returncode != 0:
            raise RuntimeError(res.stdout[-2000:] + res.stderr[-2000:])
        per = [np.fromfile(out + ".%d" % r, np.uint64) for r in range(len(sizes))]
    runs = [[None] * len(sizes) for _ in range(reps)]
    for w, raw in enumerate(per):
        i = 0
        for rep in range(reps):
            c = int(raw[i])
            runs[rep][w] = raw[i + 1:i + 1 + c].astype(np.int64)
            i += 1 + c
        assert i == len(raw)
    return runs


def main():
    det_sizes = np.zeros((len(DET), 4), np.int64)
    det_workers, det_mode, det_param, det_exact = [], [], [], []
    det_counts = np.zeros((len(DET), 4), np.int64)
    items, offsets = [], [0]
    for c, (sizes, mode, param, exact) in enumerate(DET):
        run = run_driver(sizes, mode, param, 1)[0]
        det_sizes[c, :len(sizes)] = sizes
        det_workers.append(len(sizes))
        det_mode.append(mode)
        det_param.append(float(param))
        det_exact.append(exact)
        for w, o in enumerate(run):
            det_counts[c, w] = len(o)
            items.append(o)
        offsets.append(offsets[-1] + sum(len(o) for o in run))
    sub_subsets, sub_counts, sub_config = [], [], []
    for k, sizes in enumerate(SUB_SIZES):
        for run in run_driver(sizes, 0, 4, SUB_REPS):
            sub_subsets.append(np.sort(np.concatenate(run)))
            cnt = np.zeros(4, np.int64)
            cnt[:len(sizes)] = [len(o) for o in run]
            sub_counts.append(cnt)
            sub_config.append(k)
    sub_sizes = np.zeros((len(SUB_SIZES), 4), np.int64)
    for k, sizes in enumerate(SUB_SIZES):
        sub_sizes[k, :len(sizes)] = sizes
    bern_masks, bern_p, bern_sizes = [], [], np.zeros((len(BERN), 4), np.int64)
    for b, (p, sizes) in enumerate(BERN):
        bern_sizes[b, :len(sizes)] = sizes
        bern_p.append(p)
        m = np.zeros((BERN_REPS, 64), bool)
        for rep, run in enumerate(run_driver(sizes, 1, p, BERN_REPS)):
            for o in run:
                if np.any(np.diff(o) <= 0):
                    raise RuntimeError("finding: the stock BernoulliSample emitted %s out of input order" % o)
                m[rep, o] = True
        bern_masks.append(np.packbits(m, axis=1, bitorder="little"))
    np.savez_compressed(
        OUT,
        det_sizes=det_sizes, det_workers=np.array(det_workers, np.int64), det_mode=np.array(det_mode, np.int64),
        det_param=np.array(det_param), det_exact=np.array(det_exact), det_counts=det_counts,
        det_items=np.concatenate(items).astype(np.int64), det_offsets=np.array(offsets, np.int64),
        sub_sizes=sub_sizes, sub_workers=np.array([len(x) for x in SUB_SIZES], np.int64),
        sub_subsets=np.array(sub_subsets, np.uint8), sub_counts=np.array(sub_counts, np.uint8), sub_config=np.array(sub_config, np.uint8),
        bern_p=np.array(bern_p), bern_sizes=bern_sizes, bern_workers=np.array([len(x) for _, x in BERN], np.int64),
        bern_masks=np.array(bern_masks, np.uint8))
    print("wrote %s: %d deterministic cases, %d Sample(4) runs, %d BernoulliSample runs" %
          (OUT, len(DET), len(sub_config), len(BERN) * BERN_REPS))


if __name__ == "__main__":
    main()
