"""Exact numpy restatement of sk_neighbor_joining (include/skani_b200.h), a naive textbook NJ, and the Newick and patristic
helpers the tree tests use.

nj(D) follows the contract step by step: float64 throughout, every operation rounded on its own (numpy never fuses), live
nodes ordered by id, the dead row and column removed after each join.  np.argmin over the row-major upper triangle returns
the first minimum, which is exactly the tie rule (smallest (i, j)), and it compares doubles, so -0 equals +0."""
import math

import numpy as np

NJ_JOIN_DTYPE = np.dtype([("a", np.uint32), ("b", np.uint32), ("len_a", np.float64), ("len_b", np.float64)])


def matrix(n, a, b, ani):
    """the initial distances: 1 - (double)ani for every row with ani > 0.1, 1.0 for pairs without one, 0 on the diagonal"""
    D = np.ones((n, n))
    np.fill_diagonal(D, 0.0)
    ani = np.asarray(ani, np.float32)
    with np.errstate(invalid="ignore"):
        keep = ani > np.float32(0.1)
    a = np.asarray(a, np.int64)[keep]; b = np.asarray(b, np.int64)[keep]
    d = 1.0 - ani[keep].astype(np.float64)
    D[a, b] = d
    D[b, a] = d
    return D


def nj(D):
    """the join table (NJ_JOIN_DTYPE, n - 1 rows) of the dense distance matrix D"""
    D = np.array(D, np.float64)
    n = len(D)
    joins = np.zeros(max(n - 1, 0), NJ_JOIN_DTYPE)
    if n < 2:
        return joins
    R = D.sum(axis=1)          # exact: every term is a multiple of 2^-27 (or of the caller's grid) and the sum < 2^26
    node = list(range(n))
    low = np.tril(np.ones((n, n), bool))
    m, t = n, 0
    while m > 2:
        Q = ((m - 2) * D - R[:, None]) - R[None, :]
        Q[low[:m, :m]] = np.inf
        i, j = divmod(int(np.argmin(Q)), m)
        dij, ri, rj = D[i, j], R[i], R[j]
        di = 0.5 * dij + (ri - rj) / (2.0 * (m - 2))
        joins[t] = (node[i], node[j], di, dij - di)
        duk = 0.5 * ((D[i] + D[j]) - dij)
        R = ((R - D[i]) - D[j]) + duk
        R[i] = 0.5 * ((ri + rj) - m * dij)
        D[i, :] = duk
        D[:, i] = duk
        D[i, i] = 0.0
        node[i] = n + t
        keep = np.arange(m) != j
        D = D[keep][:, keep]
        R = R[keep]
        del node[j]
        m -= 1
        t += 1
    h = 0.5 * D[0, 1]
    joins[n - 2] = (node[0], node[1], h, h)
    return joins


def nj_results(n, a, b, ani):
    return nj(matrix(n, a, b, ani))


def nj_textbook(D):
    """textbook neighbour joining over Python lists: row sums recomputed with math.fsum every step, the new node appended at
    the end.  Returns (a, b, len_a, len_b) rows with the scipy node numbering."""
    D = [list(map(float, r)) for r in D]
    n = len(D)
    node = list(range(n))
    out = []
    while len(node) > 2:
        m = len(node)
        R = [math.fsum(r) for r in D]
        best = None
        for i in range(m):
            for j in range(i + 1, m):
                q = (m - 2) * D[i][j] - R[i] - R[j]
                if best is None or q < best[0]:
                    best = (q, i, j)
        _, i, j = best
        di = 0.5 * D[i][j] + (R[i] - R[j]) / (2 * (m - 2))
        out.append((node[i], node[j], di, D[i][j] - di))
        du = [0.5 * (D[i][k] + D[j][k] - D[i][j]) for k in range(m)]
        keep = [k for k in range(m) if k not in (i, j)]
        D = [[D[x][y] for y in keep] + [du[x]] for x in keep] + [[du[y] for y in keep] + [0.0]]
        node = [node[k] for k in keep] + [n + len(out) - 1]
    if n >= 2:
        h = 0.5 * D[0][1]
        out.append((node[0], node[1], h, h))
    return out


# ---- trees as (parent, length) per node: leaves 0..n-1, join row t creates n + t
def tree_of_joins(n, joins):
    parent = [-1] * (2 * n - 1 if n else 0)
    length = [0.0] * len(parent)
    for t, r in enumerate(joins):
        for c, ln in ((int(r["a"]), float(r["len_a"])), (int(r["b"]), float(r["len_b"]))):
            parent[c] = n + t
            length[c] = ln
    return parent, length


def patristic(n_leaves, parent, length):
    """leaf x leaf path lengths of a tree given as parent / branch length per node (leaves are nodes 0..n_leaves-1), built
    bottom up: at each internal node, every leaf pair that meets there gets (leaf-to-node distance) + (leaf-to-node
    distance).  Exact whenever the lengths are multiples of a power of two and the sums stay below 1."""
    kids = {}
    for c, p in enumerate(parent):
        if p >= 0:
            kids.setdefault(p, []).append(c)
    order, stack = [], [v for v, p in enumerate(parent) if p < 0]
    while stack:
        v = stack.pop()
        order.append(v)
        stack.extend(kids.get(v, []))
    P = np.zeros((n_leaves, n_leaves))
    below = {}                     # node -> (leaves under it, their distances to it)
    for v in reversed(order):
        if v < n_leaves and v not in kids:
            below[v] = (np.array([v]), np.zeros(1))
            continue
        parts = []
        for c in kids[v]:
            leaves, dist = below.pop(c)
            parts.append((leaves, dist + length[c]))
        for x in range(len(parts)):
            for y in range(x + 1, len(parts)):
                (la, da), (lb, db) = parts[x], parts[y]
                blk = da[:, None] + db[None, :]
                P[np.ix_(la, lb)] = blk
                P[np.ix_(lb, la)] = blk.T
        below[v] = (np.concatenate([q[0] for q in parts]), np.concatenate([q[1] for q in parts]))
    return P


def splits(n_leaves, parent):
    """the non-trivial bipartitions of the unrooted tree, each as the frozenset of leaves on the side without leaf 0"""
    kids = {}
    for c, p in enumerate(parent):
        if p >= 0:
            kids.setdefault(p, []).append(c)
    out = set()
    clade = {}
    order = sorted(kids, key=lambda v: v)          # children before parents: ids only grow towards the root
    for v in range(n_leaves):
        clade[v] = frozenset([v])
    for v in order:
        clade[v] = frozenset().union(*(clade[c] for c in kids[v]))
    full = frozenset(range(n_leaves))
    for v, s in clade.items():
        side = s if 0 not in s else full - s
        if 1 < len(side) < n_leaves - 1:
            out.add(side)
    return out


# ---- Newick
def parse_newick(text):
    """(labels, parent, length): leaves first in order of appearance (node k is labels[k]), internal nodes after them, the
    root with parent -1.  Quoted labels ('' is a quote) are unquoted.  Iterative, so deep caterpillars parse."""
    s = text.strip()
    assert s.endswith(";"), "Newick must end with ';'"
    s = s[:-1]
    nodes = []          # (label or None, parent index, length)
    stack = []
    pos = 0
    cur = None          # index of the node whose label / length come next

    def read_label(p):
        if p < len(s) and s[p] == "'":
            out = []
            p += 1
            while True:
                q = s.index("'", p)
                out.append(s[p:q])
                if q + 1 < len(s) and s[q + 1] == "'":
                    out.append("'")
                    p = q + 2
                else:
                    return "".join(out), q + 1
        q = p
        while q < len(s) and s[q] not in "(),:;":
            q += 1
        return s[p:q], q

    while pos < len(s):
        ch = s[pos]
        if ch == "(":
            nodes.append([None, stack[-1] if stack else -1, 0.0])
            stack.append(len(nodes) - 1)
            pos += 1
            cur = None
        elif ch == ",":
            pos += 1
            cur = None
        elif ch == ")":
            cur = stack.pop()
            pos += 1
            lab, pos = read_label(pos)
            if lab:
                nodes[cur][0] = lab
        elif ch == ":":
            q = pos + 1
            while q < len(s) and s[q] not in "(),;":
                q += 1
            nodes[cur][2] = float(s[pos + 1:q])
            pos = q
        else:
            lab, pos = read_label(pos)
            nodes.append([lab, stack[-1] if stack else -1, 0.0])
            cur = len(nodes) - 1
    assert not stack, "unbalanced parentheses"
    has_kids = {nd[1] for nd in nodes}
    leaves = [k for k in range(len(nodes)) if k not in has_kids]
    inner = [k for k in range(len(nodes)) if k in has_kids]
    new = {k: i for i, k in enumerate(leaves + inner)}
    labels = [nodes[k][0] for k in leaves]
    parent = [-1] * len(nodes)
    length = [0.0] * len(nodes)
    for k, nd in enumerate(nodes):
        parent[new[k]] = new[nd[1]] if nd[1] >= 0 else -1
        length[new[k]] = nd[2]
    return labels, parent, length


def newick_splits(labels, parent, names):
    """splits() of a parsed Newick tree, with leaves renumbered by their index in `names`"""
    idx = [names.index(x) for x in labels]
    n = len(labels)
    kids = {}
    for c, p in enumerate(parent):
        if p >= 0:
            kids.setdefault(p, []).append(c)
    clade = {}
    stack = [k for k, p in enumerate(parent) if p < 0]
    order = []
    while stack:
        v = stack.pop()
        order.append(v)
        stack.extend(kids.get(v, []))
    for v in reversed(order):
        clade[v] = frozenset([idx[v]]) if v < n else frozenset().union(*(clade[c] for c in kids[v]))
    full = frozenset(range(n))
    out = set()
    for v, s in clade.items():
        side = s if 0 not in s else full - s
        if 1 < len(side) < n - 1:
            out.add(side)
    return out


# ---- random additive trees: branch lengths multiples of 2^-24, so every 1 - d is an exact float32 above 0.1
def random_additive(rng, n, max_diameter=0.9):
    """(D, parent, length) of a random binary tree on n leaves whose patristic matrix D has diameter < max_diameter"""
    parent = [-1] * (2 * n - 1)
    length = [0.0] * (2 * n - 1)
    live = list(range(n))
    nxt = n
    while len(live) > 1:
        x, y = rng.choice(len(live), 2, replace=False)
        for c in (live[x], live[y]):
            parent[c] = nxt
        live = [v for k, v in enumerate(live) if k not in (x, y)] + [nxt]
        nxt += 1
    depth = max(1, _height(n, parent))
    cap = int(max_diameter / (2 * depth) * 2 ** 24)        # every root-to-leaf path < max_diameter / 2
    for v in range(2 * n - 2):
        length[v] = int(rng.integers(1, max(cap, 2))) / 2 ** 24
    return patristic(n, parent, length), parent, length


def _height(n, parent):
    best = 0
    for x in range(n):
        h = 0
        while parent[x] >= 0:
            x = parent[x]
            h += 1
        best = max(best, h)
    return best
