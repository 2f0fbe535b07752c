"""PAF files with values no synthetic generator writes: a pafgen set of which about 15 % of the lines carry one mutation each,
tagged with its class.

The reference reads every numeric column with strtol into a uint32 (paf.c:34-56), ml into a 31-bit field, and takes a read's
length from its first line (hit.c:88, sd_put).  So a PAF can hand the selection and the graph build negative columns, values
of 2^31 and more, starts past ends, ends past lengths, lengths that disagree between lines and reads longer than 2^31; the
classes below produce each of them.  Whole-read classes ("long_read", "near_2^32") mutate several lines of one read:
a read is long only if its first line says so, and the second ma_hit_sub (end_clip = min_span / 2) only opens an interval
below zero when min_dp of its query starts sit within end_clip of 2^32.

    make(base, out, seed) -> {class: number of lines}

is seeded and deterministic.
"""
import numpy as np

LINE_CLASSES = ["negative", "ge2^31", "ge2^32_same", "ge2^32_small", "strtol", "qs>qe", "ts>te", "end_past_len",
                "len_disagree", "ml>bl", "bl=0", "ml_big", "10_fields", "strand"]
EXTRA_CLASSES = ["self", "self_pal"]
READ_CLASSES = ["long_read", "near_2^32"]
CLASSES = LINE_CLASSES + EXTRA_CLASSES + READ_CLASSES
NUM_COLS = [1, 2, 3, 6, 7, 8, 9, 10]            # ql qs qe . . tl ts te ml bl


def _line(f, rng, cls, i):
    """Mutates the fields f of line i in place by class cls; False if the class does not apply to this line."""
    c = int(rng.choice(NUM_COLS))
    if cls == "negative":
        f[c] = str(-int(f[c]) if int(f[c]) else -int(rng.integers(1, 5000)))
    elif cls == "ge2^31":
        f[c] = str(int(f[c]) + 2**31)
    elif cls == "ge2^32_same":                       # the same low 32 bits
        f[c] = str(int(f[c]) + 2**32 * int(rng.integers(1, 4)))
    elif cls == "ge2^32_small":                      # wraps to a small value
        f[c] = str(2**32 + int(rng.integers(0, 3000)))
    elif cls == "strtol":
        k = int(rng.integers(0, 4))
        f[c] = ["+" + f[c], "  00" + f[c], f[c] + "x7", "9" * int(rng.integers(19, 24))][k]
    elif cls == "qs>qe":
        f[2], f[3] = f[3], f[2]
    elif cls == "ts>te":
        f[7], f[8] = f[8], f[7]
    elif cls == "end_past_len":
        j = 3 if rng.random() < 0.5 else 8
        f[j] = str(int(f[j - 2]) + int(rng.integers(1, 4000)))
    elif cls == "len_disagree":
        j = 1 if rng.random() < 0.5 else 6
        f[j] = str(max(int(f[j]) + int(rng.integers(-3000, 3000)), 1))
    elif cls == "ml>bl":
        f[9] = str(int(f[10]) + int(rng.integers(1, 3000)))
    elif cls == "bl=0":
        f[10] = "0"
    elif cls == "ml_big":
        f[9] = str(int(f[9]) + 2**31)
    elif cls == "10_fields":
        if i == 0:                                   # (the first record's stale bl would be uninitialised memory)
            return False
        del f[10:]
    elif cls == "strand":
        f[4] = str(rng.choice(["*", "x", "-junk", "", "+-"]))
    return True


def make(base, out, seed, frac=0.15):
    rng = np.random.default_rng(seed)
    lines = [ln.split("\t") for ln in open(base).read().splitlines() if ln]
    n = len(lines)
    counts = {c: 0 for c in CLASSES}
    touched = np.zeros(n, dtype=bool)
    by_q = {}
    for i, f in enumerate(lines):
        by_q.setdefault(f[0], []).append(i)
    names = sorted(by_q)
    pick = rng.permutation(len(names))
    # reads longer than 2^31: every length column of theirs (the first appearance decides, hit.c:88)
    long_reads = {names[k] for k in pick[:3]}
    for i, f in enumerate(lines):
        for j, c in ((0, 1), (5, 6)):
            if f[j] in long_reads:
                f[c] = str(int(f[c]) + 2**31)
                touched[i] = True
                counts["long_read"] += 1
    # min_dp + 1 query starts within end_clip of 2^32 on each of three reads (qe - qs stays >= min_span in 32 bits)
    for k in pick[3:6]:
        for i in by_q[names[k]][:4]:
            f = lines[i]
            f[2] = str(2**32 - int(rng.integers(1, 1000)))
            f[3] = str(max(int(f[3]), 2500))
            touched[i] = True
            counts["near_2^32"] += 1
    # one class per line on the rest, about frac of all lines in total
    budget = int(frac * n) - int(touched.sum())
    cand = rng.permutation(np.flatnonzero(~touched))[:max(budget, 0)]
    for t, i in enumerate(cand):
        cls = LINE_CLASSES[t % len(LINE_CLASSES)]
        if _line(lines[i], rng, cls, int(i)):
            counts[cls] += 1
    # self lines and palindromic self lines (asm.c:27), inserted among the others
    extra = []
    for k in range(60):
        src = lines[int(rng.integers(0, n))]
        if len(src) < 12:
            continue
        f = list(src)
        f[5], f[6] = f[0], f[1]
        if k % 2:
            f[7], f[8], f[4] = f[2], f[3], "-"
            counts["self_pal"] += 1
        else:
            counts["self"] += 1
        extra.append((int(rng.integers(1, n)), f))
    for pos, f in sorted(extra, key=lambda x: -x[0]):
        lines.insert(pos, f)
    with open(out, "w") as fo:
        fo.writelines("\t".join(f) + "\n" for f in lines)
    return counts
