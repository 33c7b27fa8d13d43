"""TEST INFRASTRUCTURE: a float64 numpy restatement of probreg's GMMTree (probreg/cc/gmmtree.cc, probreg/gmmtree.py), function by
function, with the line numbers it restates.  It takes the same explicit leaf seeds as the library (the reference draws them with
Eigen's std::rand and, for tree_level >= 2, reads beyond the 8 L indices it drew) and the same per-level iteration cap.

It is not pinned to outputs of the reference: the reference's C++ needs the Eigen submodule and its Python needs open3d.  It is
pinned by cases with known answers (tests/test_zz_gmmtree.py) and by review against the cited lines.  probreg_b200 never imports it.
"""
import numpy as np

N_NODE = 8
EPS = 1.0e-15                       # gmmtree.cc:9


def level(l):                       # gmmtree.cc:44
    return N_NODE * (N_NODE ** l - 1) // (N_NODE - 1)


def child(j):                       # gmmtree.cc:42
    return (j + 1) * N_NODE


def n_total(tree_level):            # gmmtree.cc:100
    return level(tree_level)


def gaussian_pdf(x, mu, cov):
    """gmmtree.cc:11-18 for the rows of x: 0 when det < 1e-15, else c exp(-d^T cov^-1 d / 2)"""
    det = np.linalg.det(cov)
    if det < EPS:
        return np.zeros(len(x))
    c = 1.0 / (det ** 0.5 * (2.0 * np.pi) ** 1.5)
    d = x - mu
    ep = -0.5 * np.einsum("ni,ij,nj->n", d, np.linalg.inv(cov), d)
    return c * np.exp(ep)


def log_likelihood(nodes, points, j0, jn):
    """gmmtree.cc:20-33"""
    tmp = np.zeros(len(points))
    for j in range(j0, jn):
        pi, mu, cov = nodes[j]
        if pi < EPS:
            continue
        tmp += pi * gaussian_pdf(points, mu, cov)
    return float(np.sum(np.log(np.maximum(tmp, EPS))))


def complexity(cov):
    """gmmtree.cc:35-40: smallest eigenvalue / sum of the eigenvalues"""
    lmds = np.sort(np.linalg.eigvalsh(cov))[::-1]
    return lmds[2] / lmds.sum()


def initialize_nodes(points, tree_level, leaf_seeds):
    """gmmtree.cc:46-73, the leaves seeded from leaf_seeds (8^L point indices)"""
    nodes = [None] * n_total(tree_level)
    lf = level(tree_level - 1)
    n = len(points)
    for j in range(N_NODE ** tree_level):
        y = points[leaf_seeds[j]]
        diff = points - y
        nodes[lf + j] = (1.0 / N_NODE, y.copy(), diff.T.dot(diff) / n)
    for l in range(tree_level - 2, -1, -1):
        pidx, cidx = level(l), level(l + 1)
        for j in range(N_NODE ** (l + 1)):
            mu, cov = np.zeros(3), np.zeros((3, 3))
            for k in range(N_NODE):
                _, cm, cc = nodes[cidx + j * N_NODE + k]
                mu += cm
                cov += cc + np.outer(cm, cm)
            mu /= N_NODE
            cov /= N_NODE
            nodes[pidx + j] = (1.0 / N_NODE, mu, cov - np.outer(mu, mu))
    return nodes


def _gamma(points, nodes, j0):
    """gmmtree.cc:141-152 for points that share the first child j0: (normalised gamma (n, 8), argmax)"""
    g = np.stack([nodes[j][0] * gaussian_pdf(points, nodes[j][1], nodes[j][2]) for j in range(j0, j0 + N_NODE)], axis=1)
    den = g.sum(axis=1)
    ok = den > EPS
    g = np.where(ok[:, None], g / np.where(ok, den, 1.0)[:, None], 0.0)
    return g, np.argmax(g, axis=1)          # the first maximum, as Eigen's maxCoeff


def _moments(g, z):
    return (g.sum(), g.dot(z), np.einsum("n,ni,nj->ij", g, z, z))


def build_estep(points, nodes, parent_idx):
    """gmmTreeEstep (gmmtree.cc:125-163): moments {node: (m0, m1, m2)} and the argmax node of every point"""
    moments = {}
    current = np.zeros(len(points), dtype=np.int64)
    for p in np.unique(parent_idx):
        sel = np.nonzero(parent_idx == p)[0]
        j0 = child(p)
        g, best = _gamma(points[sel], nodes, j0)
        for c in range(N_NODE):
            moments[j0 + c] = _moments(g[:, c], points[sel])
        current[sel] = j0 + best
    return moments, current


def ml_estimator(m, n_points, lambda_d):
    """gmmtree.cc:81-96"""
    m0, m1, m2 = m
    if m0 < lambda_d:
        return (0.0, np.zeros(3), np.identity(3))
    mu = m1 / m0
    return (m0 / n_points, mu, m2 / m0 - np.outer(mu, mu))


def build(points, tree_level, lambda_s, lambda_d, leaf_seeds, maxiter=1000):
    """buildGmmTree (gmmtree.cc:98-123) with a cap of maxiter EM iterations per level.
    Returns (nodes [(pi, mu, cov)], iterations per level, argmax node of every point in the last E-step, q trace per level)."""
    points = np.asarray(points, dtype=np.float64)
    nodes = initialize_nodes(points, tree_level, leaf_seeds)
    parent = -np.ones(len(points), dtype=np.int64)
    current = np.zeros(len(points), dtype=np.int64)
    iters, qs = [], []
    for l in range(tree_level):
        prev_q, it, trace = 0.0, 0, []
        while True:
            moments, current = build_estep(points, nodes, parent)
            for j in range(level(l), level(l + 1)):              # gmmTreeMstep, gmmtree.cc:166-173
                nodes[j] = ml_estimator(moments.get(j, (0.0, np.zeros(3), np.zeros((3, 3)))), len(points), lambda_d)
            q = log_likelihood(nodes, points, level(l), level(l + 1))
            trace.append(q)
            it += 1
            if abs(q - prev_q) < lambda_s or it >= maxiter:
                break
            prev_q = q
        iters.append(it)
        qs.append(trace)
        parent = current
    return nodes, iters, current, qs


def reg_estep(points, nodes, tree_level, lambda_c):
    """gmmTreeRegEstep (gmmtree.cc:175-215): [(m0, m1, m2)] per node"""
    points = np.asarray(points, dtype=np.float64)
    n = len(points)
    search = -np.ones(n, dtype=np.int64)
    gsel = np.zeros(n)
    active = np.ones(n, dtype=bool)
    cplx = {}
    for l in range(tree_level):
        j0s = child(search)
        for j0 in np.unique(j0s[active]):
            sel = np.nonzero(active & (j0s == j0))[0]
            g, best = _gamma(points[sel], nodes, j0)
            search[sel] = j0 + best
            gsel[sel] = g[np.arange(len(sel)), best]
        for j in np.unique(search[active]):
            if j not in cplx:
                cplx[j] = complexity(nodes[j][2])
        stop = np.array([cplx[j] <= lambda_c for j in search])
        active &= ~stop
    out = [(0.0, np.zeros(3), np.zeros((3, 3))) for _ in range(len(nodes))]
    for j in np.unique(search):
        sel = search == j
        out[j] = _moments(gsel[sel], points[sel])
    return out


def _skew(x):
    return np.array([[0.0, -x[2], x[1]], [x[2], 0.0, -x[0]], [-x[1], x[0], 0.0]])


def twist_mul(tw, rot, t):
    """se3_op.py: twist_trans + twist_mul (non-linear)"""
    twd = np.linalg.norm(tw[:3])
    if twd == 0.0:
        tr = np.identity(3)
    else:
        ntw = tw[:3] / twd
        c, s = np.cos(twd), np.sin(twd)
        tr = c * np.identity(3) + (1.0 - c) * np.outer(ntw, ntw) + s * _skew(ntw)
    return tr.dot(rot), t.dot(tr.T) + tw[3:]


def mstep(moments, nodes, rot, t):
    """gmmtree.py:64-83, node by node as the reference writes it; returns (rot, t, residual or NaN)"""
    n = len(moments)
    amat, bmat = np.zeros((n * 3, 6)), np.zeros(n * 3)
    for i, m in enumerate(moments):
        if m[0] < np.finfo(np.float32).eps:
            continue
        lmd, nn = np.linalg.eigh(nodes[i][2])
        s = m[1] / m[0]
        nn = np.multiply(nn, np.sqrt(m[0] / lmd))
        sl = slice(3 * i, 3 * (i + 1))
        bmat[sl] = np.dot(nn.T, nodes[i][1]) - np.dot(nn.T, s)
        amat[sl, :3] = np.cross(s, nn.T)
        amat[sl, 3:] = nn.T
    x, q, _, _ = np.linalg.lstsq(amat, bmat, rcond=-1)
    rot, t = twist_mul(x, rot, t)
    return rot, t, float(q[0]) if q.size else float("nan")


def registration(nodes, target, tree_level, lambda_c=0.01, maxiter=20, tol=1.0e-4):
    """gmmtree.py:85-96 on a built tree: (inverse rot, inverse t, q of the last iteration, q per iteration)"""
    rot, t = np.identity(3), np.zeros(3)
    q, trace = None, []
    for _ in range(maxiter):
        moments = reg_estep(np.asarray(target).dot(rot.T) + t, nodes, tree_level, lambda_c)
        rot, t, qn = mstep(moments, nodes, rot, t)
        trace.append(qn)
        if q is not None and abs(qn - q) < tol:
            break
        q = qn
    return rot.T, -rot.T.dot(t), trace[-1], trace
