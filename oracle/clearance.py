"""TEST INFRASTRUCTURE — float64 reference of rda_plan_clearance (include/rda_b200.h, DESIGN.md §9).

The signed distance of convex sets P (robot body at a pose) and Q (obstacle),

    sd(P, Q) = max over unit w of ( min_{x in P} w.x - max_{y in Q} w.y ),

is the Euclidean distance of disjoint sets and minus the penetration depth of overlapping ones.  Computed here in
numpy, in world coordinates, from the same H-rep rows the kernels read: polygon obstacles are canonical closed rows
(row i joins vertices i and i+1, the first zero-norm row ends the polygon), discs rows [[1,0],[0,1],[0,0]] with
b = (cx, cy, -r).  Bodies are taken as the kernels hold them (body_from_halfspaces: the float32 vertices of
robot_geom_from_halfspaces, or the float32 centre and radius of a disc).
"""
import numpy as np

from .cell_geo import poly_vertices

OBS_POLYGON, OBS_CIRCLE = 0, 1


def body_from_halfspaces(G, h, disc=False):
    """The body of canonical rows (G, h) as rda_create / rda_set_robot_classes store it: dict with 'disc' and either
    'V' (float32 vertices, vertex j joining rows j-1 and j) or 'c', 'r' (float32 centre and radius)."""
    G = np.asarray(G, np.float32).astype(float)
    h = np.asarray(h, np.float32).astype(float).ravel()
    if disc:
        return {'disc': True, 'c': h[:2].copy(), 'r': -h[2]}
    return {'disc': False, 'V': poly_vertices(G, h).astype(np.float32).astype(float)}


def _normals(V):
    """Unit outward normals of the edges i -> i+1 of a counter-clockwise polygon."""
    e = np.roll(V, -1, axis=0) - V
    n = np.stack([e[:, 1], -e[:, 0]], 1)
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def _seg_d2(q, a, e):
    e2 = e @ e
    t = np.clip((q - a) @ e / e2, 0.0, 1.0) if e2 > 0 else 0.0
    d = q - a - t * e
    return d @ d


def point_polygon(q, V, n=None):
    """Signed distance of the point q to the convex polygon V (counter-clockwise)."""
    n = _normals(V) if n is None else n
    gap = np.max(np.sum(n * (q[None, :] - V), 1))
    if gap <= 0:
        return float(gap)
    E = np.roll(V, -1, axis=0) - V
    return float(np.sqrt(min(_seg_d2(q, V[i], E[i]) for i in range(len(V)))))


def polygons(P, Q, nP=None, nQ=None):
    """Signed distance of convex polygons P and Q (counter-clockwise vertex arrays [n, 2]): the largest gap over the
    edge normals of both when it is <= 0 (minus the penetration depth), else the nearest vertex-to-edge distance."""
    nP = _normals(P) if nP is None else nP
    nQ = _normals(Q) if nQ is None else nQ
    gap = max(np.max(np.min((P @ nQ.T) - np.sum(nQ * Q, 1)[None, :], 0)),
              np.max(np.min((Q @ nP.T) - np.sum(nP * P, 1)[None, :], 0)))
    if gap <= 0:
        return float(gap)
    best = np.inf
    for X, Y in ((P, Q), (Q, P)):
        E = np.roll(Y, -1, axis=0) - Y
        for x in X:
            for i in range(len(Y)):
                best = min(best, _seg_d2(x, Y[i], E[i]))
    return float(np.sqrt(best))


def obstacle_polygon(A, b):
    """(vertices, unit row normals) of canonical polygon rows, up to the first zero-norm row; None below three rows."""
    A = np.asarray(A, np.float32).astype(float)
    b = np.asarray(b, np.float32).astype(float).ravel()
    nrm = np.linalg.norm(A, axis=1)
    ne = int(np.argmin(nrm > 0)) if not np.all(nrm > 0) else len(nrm)
    if ne < 3:
        return None
    return poly_vertices(A[:ne], b[:ne]), A[:ne] / nrm[:ne, None]


def cell(body, pose, kind, A, b):
    """sd of `body` (body_from_halfspaces) placed at pose (x, y, heading) and one obstacle (kind, rows A [E, 2], b [E])."""
    x, y, th = (float(v) for v in np.asarray(pose, np.float32))
    p = np.array([x, y])
    Rm = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    b = np.asarray(b, np.float32).astype(float).ravel()
    if kind == OBS_CIRCLE:
        oc, orad = b[:2], -b[2]
        if body['disc']:
            return float(np.linalg.norm(p + Rm @ body['c'] - oc) - orad - body['r'])
        V = p + body['V'] @ Rm.T
        return point_polygon(oc, V) - orad
    poly = obstacle_polygon(A, b)
    if poly is None:
        return np.inf
    Q, nQ = poly
    if body['disc']:
        return point_polygon(p + Rm @ body['c'], Q, nQ) - body['r']
    return polygons(p + body['V'] @ Rm.T, Q, None, nQ)


def plan_clearance(bodies, s, obs_A, obs_b, obs_kind, obs_count, time_varying=False):
    """The whole call: bodies (one body, or a list of B), s [B, 3, T+1], obstacle inputs as rda_inputs
    (obs_A [B, N, Tc, E, 2], ...).  Returns (dist [B, N, T+1] float64, +inf past min(obs_count, N))."""
    s = np.asarray(s)
    B, _, T1 = s.shape
    N = 0 if obs_kind is None else np.asarray(obs_kind).shape[1]
    dist = np.full((B, N, T1), np.inf)
    for bb in range(B):
        body = bodies[bb] if isinstance(bodies, (list, tuple)) else bodies
        for o in range(min(max(int(obs_count[bb]), 0), N)):
            for t in range(T1):
                c = t if time_varying else 0
                dist[bb, o, t] = cell(body, s[bb, :, t], int(obs_kind[bb][o]), obs_A[bb][o][c], obs_b[bb][o][c])
    return dist
