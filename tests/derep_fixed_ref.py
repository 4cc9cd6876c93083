"""Plain-Python restatement of sk_dereplicate_fixed's waves (skani_b200/csrc/derep.cu): the genomes of rank < n_fixed are
representatives before the first wave and their markers are in the index; the waves cover the other genomes.  Driven by a
pair oracle as tests/derep_ref.py is (the pairs that pass the triangle's screen and the ANI of every such pair's chained
row).  It returns what the library returns plus every pair it chained, in order, the number of pairs that passed a screen
(the library's pairs_screened) and the number of waves, so that tests can hold it against tests/cluster_ref.py's greedy
clusters of the triangle's rows without the rows between two fixed genomes, and against the library's stats."""
import numpy as np

UNDECIDED, REP, MEMBER = 0, 1, 2
FIRST_WAVE, MAX_WAVE = 64, 4096     # the library's default wave sizes (wave = 0)


def pair(a, b):
    return (min(a, b), max(a, b))


def wave_bounds(n, n_fixed, wave):
    """the [w0, w1) rank ranges of the waves: from rank n_fixed, `wave` genomes each, or 64 doubling up to 4096 when 0"""
    out, w0, size = [], n_fixed, wave or FIRST_WAVE
    while w0 < n:
        out.append((w0, min(n, w0 + size)))
        w0 += size
        size = wave or min(2 * size, MAX_WAVE)
    return out


def dereplicate(n, screen, ani, min_ani, rank, wave, n_fixed=0):
    """screen: set of pairs (i, j), i < j, that pass the screen; ani: dict pair -> float32 ANI of its chained row.  wave = 0
    is the library's default schedule.  Returns (rep, cluster, join, chained, screened, waves): join[g] = the pair joining
    member g to rep[g] (None for a representative); chained lists the chained pairs in chaining order.  Raises if a pair
    would be chained twice or a pair of two fixed genomes would be screened."""
    rank = [int(r) for r in rank]
    order = sorted(range(n), key=lambda g: rank[g])
    fixed = set(order[:n_fixed])
    min_ani = np.float32(min_ani)
    state = [UNDECIDED] * n
    for g in fixed:
        state[g] = REP
    reps = list(order[:n_fixed])
    chained, done = [], set()
    screened = 0

    def passes(p):
        nonlocal screened
        assert not (p[0] in fixed and p[1] in fixed), p
        if p in screen:
            screened += 1
            return True
        return False

    def chain(p):
        assert p in screen and p not in done, p
        done.add(p)
        chained.append(p)

    def edge(p):
        a = np.float32(ani[p])
        return bool(a > np.float32(0.1) and a >= min_ani)

    bounds = wave_bounds(n, n_fixed, wave)
    for w0, w1 in bounds:
        w = order[w0:w1]
        # 1. the wave against the representatives so far, the fixed ones included: an edge to one makes a member
        for g in w:
            for r in reps:
                p = pair(g, r)
                if passes(p):
                    chain(p)
                    if edge(p):
                        state[g] = MEMBER
        # 2. the undecided genomes of the wave against each other, then the greedy rule in rank order
        u = [g for g in w if state[g] == UNDECIDED]
        adj = {g: [] for g in u}
        for i, g in enumerate(u):
            for h in u[i + 1:]:
                p = pair(g, h)
                if passes(p):
                    chain(p)
                    if edge(p):
                        adj[g].append(h)
                        adj[h].append(g)
        for g in u:
            state[g] = MEMBER if any(state[h] == REP and rank[h] < rank[g] for h in adj[g]) else REP
        # 3. the new representatives join the index
        reps += [g for g in u if state[g] == REP]
    # every member against every representative, the pairs not chained yet
    for g in order:
        if state[g] == MEMBER:
            for r in reps:
                p = pair(g, r)
                if passes(p) and p not in done:
                    chain(p)
    rep = np.arange(n, dtype=np.uint32)
    join = [None] * n
    for g in range(n):
        if state[g] != MEMBER:
            continue
        best = None
        for r in reps:
            p = pair(g, r)
            if p in done and edge(p):
                key = (-float(np.float32(ani[p])), rank[r])
                if best is None or key < best[0]:
                    best = (key, r, p)
        assert best is not None, g
        rep[g], join[g] = best[1], best[2]
    is_rep = np.array([s == REP for s in state], bool)
    pos = np.cumsum(is_rep[order]) - 1
    cid = np.empty(n, np.int64)
    cid[order] = pos
    cluster = cid[rep].astype(np.uint32) if n else np.zeros(0, np.uint32)
    return rep, cluster, join, chained, screened, len(bounds)
