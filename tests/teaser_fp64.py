"""An independent fp64 evaluator of the TEASER++ refiner's stages (row f13), written from the definitions rather than
the kernel's operation order: farthest-point sampling in fp64, the maximum clique by Bron-Kerbosch enumeration, the
weighted rotation by np.linalg.svd (Kabsch with a proper rotation), and the voted translation by a brute force over
every consensus set.  numpy only."""
import numpy as np


def fps(src, M):
    p = src.astype(np.float64)
    mind = np.full(len(p), np.inf)
    idx = [0]
    gaps = []                                          # how far the winner was ahead of the runner-up, per step
    for _ in range(1, M):
        mind = np.minimum(mind, ((p - p[idx[-1]]) ** 2).sum(1))
        order = np.argsort(-mind, kind="stable")
        idx.append(int(order[0]))
        gaps.append(float(mind[order[0]] - mind[order[1]]) if len(order) > 1 else np.inf)
    return np.asarray(idx), np.asarray(gaps)


def clique_size(adj):
    """The clique number by Bron-Kerbosch with Tomita's pivot over every maximal clique (no bound, no ordering)."""
    nbr = [int.from_bytes(np.packbits(row, bitorder="little").tobytes(), "little") for row in np.asarray(adj, bool)]
    best = 0

    def expand(size, P, X):
        nonlocal best
        if not P and not X:
            best = max(best, size)
            return
        u = max(_bits(P | X), key=lambda w: bin(P & nbr[w]).count("1"))
        for v in _bits(P & ~nbr[u]):
            expand(size + 1, P & nbr[v], X & nbr[v])
            P &= ~(1 << v)
            X |= 1 << v
    expand(0, (1 << len(nbr)) - 1, 0)
    return best


def _bits(x):
    out = []
    while x:
        low = x & -x
        out.append(low.bit_length() - 1)
        x ^= low
    return out


def is_clique(adj, members):
    sub = adj[np.ix_(members, members)]
    return bool((sub | np.eye(len(members), dtype=bool)).all())


def colouring_bound(adj):
    """Colours of a largest-first greedy colouring (each vertex, by degree descending, takes the smallest colour no
    neighbour has): an upper bound on the clique number."""
    adj = np.asarray(adj, bool)
    colour = np.full(len(adj), -1)
    for v in np.argsort(-adj.sum(1), kind="stable"):
        used = set(colour[adj[v]].tolist())
        colour[v] = next(c for c in range(len(adj) + 1) if c not in used)
    return int(colour.max()) + 1


def kabsch(w, s, t):
    H = (w[:, None] * s).T @ t
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1, 1, np.sign(np.linalg.det(Vt.T @ U.T))])
    return Vt.T @ D @ U.T


def gnc_weights(r, mu, eps2):
    th1, th2 = (mu + 1) / mu * eps2, mu / (mu + 1) * eps2
    w = np.sqrt(eps2 * mu * (mu + 1) / np.maximum(r, 1e-300)) - mu
    return np.where(r >= th1, 0.0, np.where(r <= th2, 1.0, w))


def vote(x, r, upm):
    """Every interval between consecutive endpoints has one consensus set; the TLS cost of its mean."""
    ends = np.sort(np.concatenate([x - r, x + r]))
    best, est = np.inf, None
    for a, b in zip(ends[:-1], ends[1:]):
        c = (a + b) / 2
        inside = np.abs(x - c) <= r
        if not inside.any():
            continue
        mean = x[inside].mean()
        cost = ((x[inside] - mean) ** 2).sum() + upm * r * (~inside).sum()
        if cost < best:
            best, est = cost, mean
    return est
