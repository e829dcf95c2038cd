"""Window model (DIA::Window, api/window.hpp:140-246 and :387-503; include/thrill_gpu.h states the contract).

Items are words: an (n, 2) uint64 array of (first, value) per item (8-byte items have first = 0; doubles are their bits).
Every output is the left fold of a run of consecutive items by global position, from the run's first item, with the stock
function; pairs take .first from the run's last item (ScanSecond<F>).  The concatenation of the workers' outputs does not
depend on the sharding:
    FULL      the windows [i, i+k-1], i = 0 .. N-k                    worker r gets those whose last item it holds
    PARTIAL   FULL, then the suffixes [j, N-1], j = max(0, N-k+1) .. N-1, on the last worker
    DISJOINT  the blocks [bk, bk+k-1] with bk+k-1 < N, then the trailing N mod k items on the last worker
so `outputs` gives the concatenation and `counts` the share of each worker.

`emulate_sum` restates the kernel's bracketing of double sums (tg_window.cu): blocks of k from position 0, runs of R items,
D = min(k - 1, R + J - 1) (`depth`).

Fixture layout (tests/golden/reference_outputs_window.npz, written by tests/golden/make_golden_window.py):
    names[c]            case name
    meta[c]             (mode index into MODES, form index into FORMS, k, input index, N)
    in_start, words     input i is words[in_start[i]:in_start[i+1]] (2 words per item for pairs); a case takes its first N items
    out_start, outputs  case c's concatenated outputs are outputs[out_start[c]:out_start[c+1]], (first, value) rows
    counts[c, w, r]     the outputs worker r emitted with WORKERS[w] workers
    shards[c, w, r]     the items worker r held
"""
import numpy as np

OP_SUM_F64, OP_SUM_U64, OP_MIN_U64, OP_MAX_U64, OP_MIN_F64, OP_MAX_F64 = range(6)
F64_OPS = (OP_SUM_F64, OP_MIN_F64, OP_MAX_F64)
FULL, PARTIAL, DISJOINT = range(3)
FORMS = ["full", "partial", "disjoint"]
WORKERS = [1, 2, 3, 4, 8]
MODES = ["%s%s_%s" % (pre, t, fn) for pre in ("", "pair_") for t in ("u64", "f64") for fn in ("sum", "min", "max")]
U = 2.0 ** -53


def mode_op(mode):
    """(op, pair) of a driver mode such as pair_f64_min"""
    pair = mode.startswith("pair_")
    t, fn = mode[5:].split("_") if pair else mode.split("_")
    ops = {("u64", "sum"): OP_SUM_U64, ("u64", "min"): OP_MIN_U64, ("u64", "max"): OP_MAX_U64,
           ("f64", "sum"): OP_SUM_F64, ("f64", "min"): OP_MIN_F64, ("f64", "max"): OP_MAX_F64}
    return ops[(t, fn)], pair


def stock_fn(op, a, b):
    """the stock function on value words (uint64 arrays), elementwise"""
    if op == OP_SUM_U64:
        return a + b
    if op == OP_MIN_U64:
        return np.where(b < a, b, a)
    if op == OP_MAX_U64:
        return np.where(a < b, b, a)
    x, y = a.view(np.float64), b.view(np.float64)
    if op == OP_SUM_F64:
        with np.errstate(all="ignore"):
            return (x + y).view(np.uint64)
    with np.errstate(invalid="ignore"):
        return np.where(y < x, b, a) if op == OP_MIN_F64 else np.where(x < y, b, a)


def fold_runs(vals, op, starts, lengths):
    """the left fold with the stock function of vals[s : s + l] for every (s, l), vectorised over the runs"""
    starts = np.asarray(starts, np.int64)
    lengths = np.asarray(lengths, np.int64)
    if not len(starts):
        return np.zeros(0, np.uint64)
    acc = vals[starts].copy()
    for t in range(1, int(lengths.max())):
        act = np.nonzero(t < lengths)[0]
        acc[act] = stock_fn(op, acc[act], vals[starts[act] + t])
    return acc


def runs(N, k, form):
    """(start, length) of every output in concatenation order"""
    if form == DISJOINT:
        s = np.arange(N // k, dtype=np.int64) * k
        ln = np.full(len(s), k, np.int64)
        if N % k:
            s, ln = np.append(s, N - N % k), np.append(ln, N % k)
        return s, ln
    s = np.arange(max(N - k + 1, 0), dtype=np.int64)
    ln = np.full(len(s), k, np.int64)
    if form == PARTIAL:
        j = np.arange(max(0, N - k + 1), N, dtype=np.int64)
        s, ln = np.concatenate([s, j]), np.concatenate([ln, N - j])
    return s, ln


def counts(form, k, shard_sizes):
    """the outputs of each worker"""
    N = int(sum(shard_sizes))
    out, f = [], 0
    for r, n in enumerate(shard_sizes):
        L, last = f + n, r == len(shard_sizes) - 1
        if form == DISJOINT:
            c = L // k - f // k + (1 if last and N % k else 0)
        else:
            c = max(0, L - max(f, k - 1))
            if form == PARTIAL and last:
                c += min(N, k - 1)
        out.append(c)
        f = L
    return out


def outputs(items, op, k, form):
    """the concatenated outputs, (first, value) rows, of the stock fold"""
    items = np.asarray(items, np.uint64).reshape(-1, 2)
    s, ln = runs(len(items), k, form)
    out = np.zeros((len(s), 2), np.uint64)
    out[:, 1] = fold_runs(items[:, 1].copy(), op, s, ln)
    out[:, 0] = items[s + ln - 1, 0] if len(s) else 0
    return out


def run_shape(k):
    """(R, J): the run length of the kernel's in-block folds and the runs per block"""
    lg = (k - 1).bit_length()
    R = 1 << max(4, (lg + 1) // 2)
    return R, -(-k // R)


def depth(k):
    """D, the longest chain of additions a summand of a window goes through in the kernel's bracketing: k - 1 for one run per
    block (the block folded sequentially).  With J >= 2 runs of R: R - 1 inside its run's aggregate, J - 2 along the aggregates'
    fold (E or F), 1 to join the run prefix / suffix, 1 for the output's combine of S and P: R + J - 1 at most, and never more
    than the k - 1 additions of a k-item sum."""
    R, J = run_shape(k)
    return k - 1 if J == 1 else min(k - 1, R + J - 1)


def emulate_sum(vals, k, form):
    """the kernel's double sums (value words) for the items `vals` (uint64 words of doubles), concatenated outputs"""
    N = len(vals)
    R, J = run_shape(k)
    nb = -(-N // k) + 1
    x = np.full(nb * k, -0.0)
    x[:N] = np.asarray(vals, np.uint64).view(np.float64)
    blk = np.full((nb, J * R), -0.0)
    blk[:, :k] = x.reshape(nb, k)
    r = blk.reshape(nb, J, R)
    lens = [min(R, k - j * R) for j in range(J)]
    with np.errstate(all="ignore"):
        inpre = np.empty_like(r)
        acc = r[:, :, 0].copy()
        inpre[:, :, 0] = acc
        for t in range(1, R):
            acc = acc + r[:, :, t]
            inpre[:, :, t] = acc
        A = np.stack([inpre[:, j, lens[j] - 1] for j in range(J)], axis=1)
        E = np.empty((nb, J))
        F = np.empty((nb, J))
        if J > 1:
            e = A[:, 0].copy()
            E[:, 1] = e
            for j in range(2, J):
                e = e + A[:, j - 1]
                E[:, j] = e
            s = A[:, J - 1].copy()
            F[:, J - 2] = s
            for j in range(J - 3, -1, -1):
                s = A[:, j + 1] + s
                F[:, j] = s
        P = inpre.copy()
        for j in range(1, J):
            P[:, j, :] = E[:, j:j + 1] + inpre[:, j, :]
        S = np.empty_like(r)
        for j in range(J):
            acc = r[:, j, lens[j] - 1].copy()
            S[:, j, lens[j] - 1] = acc
            for t in range(lens[j] - 2, -1, -1):
                acc = r[:, j, t] + acc
                S[:, j, t] = acc
            if j + 1 < J:
                S[:, j, :lens[j]] = S[:, j, :lens[j]] + F[:, j:j + 1]
        P = P.reshape(nb, J * R)[:, :k].reshape(-1)
        S = S.reshape(nb, J * R)[:, :k].reshape(-1)
        s, ln = runs(N, k, form)
        e = s + ln - 1
        out = S[s].copy()
        join = (s // k) != (e // k)
        out[join] = S[s[join]] + P[e[join]]
    return out.view(np.uint64)


def bound_violations(got_words, vals, k, form):
    """the outputs (indices) with |got - exact| > gamma_D A + u |exact| among those whose window is finite and in the safe range
    (1 + gamma_D) A < DBL_MAX; exact sums in fixed point (scan_exact.to_fixed: x * 2^1074 as an int)"""
    from fractions import Fraction
    import scan_exact as X
    D = depth(k)
    g, u = Fraction(D, 2 ** 53 - D), Fraction(1, 2 ** 53)
    x = np.asarray(vals, np.uint64).view(np.float64)
    fin = np.isfinite(x)
    cs, ca, cn = [0], [0], np.concatenate([[0], np.cumsum(~fin)])
    for v in x:
        f = X.to_fixed(v) if np.isfinite(v) else 0
        cs.append(cs[-1] + f)
        ca.append(ca[-1] + abs(f))
    top = X.to_fixed(np.finfo(np.float64).max)
    s, ln = runs(len(x), k, form)
    got = np.asarray(got_words, np.uint64).view(np.float64)
    bad = []
    for o, (a, l) in enumerate(zip(s, ln)):
        if cn[a + l] - cn[a]:
            continue
        ex, A = cs[a + l] - cs[a], ca[a + l] - ca[a]
        if (1 + g) * A >= top:
            continue
        if not np.isfinite(got[o]) or abs(X.to_fixed(got[o]) - ex) > g * A + u * abs(ex):
            bad.append(o)
    return bad


def emulate_worker_sum(vals, f, n, k, form):
    """the kernel's double sums as ONE worker computes them: it sees only positions [max(f - k + 1, 0), f + n) (its halo and its
    items), the rest is the identity -0.0; returns the concatenated outputs of the whole sequence computed from that view (the
    caller takes the worker's slice)"""
    x = np.asarray(vals, np.uint64).copy()
    lo, L = max(f - k + 1, 0), f + n
    x[:lo] = 0x8000000000000000
    x[L:] = 0x8000000000000000
    return emulate_sum(x, k, form)


def load_fixtures(path):
    """the cases of reference_outputs_window.npz: dicts with name, op, pair, form, k, items ((N, 2) words), out ((m, 2) words),
    and per worker count p: shards[p] (items per worker) and counts[p] (outputs per worker)"""
    z = np.load(path)
    out = []
    for c, name in enumerate(z["names"]):
        mode, form, k, inp, N = (int(v) for v in z["meta"][c])
        op, pair = mode_op(MODES[mode])
        words = z["words"][z["in_start"][inp]:z["in_start"][inp + 1]].reshape(-1, 2)[:N]
        case = dict(name=str(name), op=op, pair=pair, form=form, k=k, items=words,
                    out=z["outputs"][z["out_start"][c]:z["out_start"][c + 1]], shards={}, counts={})
        for w, p in enumerate(WORKERS):
            case["shards"][p] = [int(v) for v in z["shards"][c, w, :p]]
            case["counts"][p] = [int(v) for v in z["counts"][c, w, :p]]
        out.append(case)
    return out


def same(got, ref, op):
    """(first, value) rows equal bit for bit; for double sums two NaNs are equal whatever their payloads (the contract leaves a
    sum's NaN payload open)"""
    got, ref = np.asarray(got, np.uint64), np.asarray(ref, np.uint64)
    if got.shape != ref.shape:
        return False
    eq = got == ref
    if op == OP_SUM_F64:
        both = np.isnan(got[..., -1].view(np.float64)) & np.isnan(ref[..., -1].view(np.float64))
        eq[..., -1] |= both
    return bool(eq.all())
