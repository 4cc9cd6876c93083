"""Plain-Python restatement of sk_dereplicate's wave algorithm (skani_b200/csrc/derep.cu), driven by a pair oracle: the set
of pairs that pass the triangle's screen and the ANI of every such pair's chained row.  It returns what the library returns
(rep, cluster, the pair joining each member to its representative) plus every pair it chained, in order, so that tests can
hold it against tests/cluster_ref.py's greedy clusters of the triangle's rows."""
import numpy as np

UNDECIDED, REP, MEMBER = 0, 1, 2


def pair(a, b):
    return (min(a, b), max(a, b))


def dereplicate(n, screen, ani, min_ani, rank, wave):
    """screen: set of pairs (i, j), i < j, that pass the screen; ani: dict pair -> float32 ANI of its chained row (every pair of
    screen has one).  Returns (rep, cluster, join, chained): join[g] = the pair joining member g to rep[g] (None for a
    representative); chained lists the chained pairs in chaining order.  Raises if a pair would be chained twice."""
    rank = [int(r) for r in rank]
    order = sorted(range(n), key=lambda g: rank[g])
    min_ani = np.float32(min_ani)
    state = [UNDECIDED] * n
    reps = []
    chained, done = [], set()

    def chain(p):
        assert p in screen and p not in done, p
        done.add(p)
        chained.append(p)

    def edge(p):
        a = np.float32(ani[p])
        return bool(a > np.float32(0.1) and a >= min_ani)

    for w0 in range(0, n, wave):
        w = order[w0:w0 + wave]
        # 1. the wave against the representatives chosen so far: an edge to one makes a member
        for g in w:
            for r in reps:
                p = pair(g, r)
                if p in screen:
                    chain(p)
                    if edge(p):
                        state[g] = MEMBER
        # 2. the undecided genomes of the wave against each other, then the greedy rule in rank order
        u = [g for g in w if state[g] == UNDECIDED]
        adj = {g: [] for g in u}
        for i, g in enumerate(u):
            for h in u[i + 1:]:
                p = pair(g, h)
                if p in screen:
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
                if p in screen and p not in done:
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
    is_rep = np.array([s == REP for s in state])
    pos = np.cumsum(is_rep[order]) - 1
    cid = np.empty(n, np.int64)
    cid[order] = pos
    cluster = cid[rep].astype(np.uint32) if n else np.zeros(0, np.uint32)
    return rep, cluster, join, chained
