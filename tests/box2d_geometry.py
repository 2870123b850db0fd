"""Float64 geometry for the Box2D building blocks of csrc/b2probe.cuh, and the case generators and checks that
tests/test_box2d_geometry_cpu.py (host build) and tests/test_gpu_box2d_geometry.py (device) both run.

A probe is any function `probe(op, records) -> out` over float32 records (n, 16): `hostsim.sim.box2d_probe` or the
device entry point b200gym_selftest_box2d.  Each check returns the indices of the cases that break the stated bound,
so that a failing test names them.

The references see exactly the float32 inputs the probe sees (vertices as the device constants hold them, the float32
rotation (s, c) as given, not re-derived from an angle) and evaluate the geometry in float64.  The bounds count
float32 roundings: u = 2^-24 is the unit roundoff, L the magnitude of the coordinates involved.
"""
import numpy as np

U = 2.0 ** -24
POLYGON_RADIUS = 0.01
RADIUS = 2 * POLYGON_RADIUS           # the contact radius of two polygons (edges are polygons of radius too)
LINEAR_SLOP = 0.005

OP_ROT, OP_EDGE_POLYGON, OP_BOX_POLYGON, OP_EDGE_RAYCAST, OP_BOX_RAYCAST, OP_GJK, OP_TOI, OP_SOLVE22, OP_SOLVE33 = range(9)
FIXTURES = {0: "lander hull", 1: "lander leg", 2: "walker hull", 3: "walker upper leg", 4: "walker lower leg"}

# rot_of's Cody-Waite constants (csrc/b2lite.cuh)
CW1 = float(np.float32(1.5707963705062866))
CW2 = float(np.float32(4.371139000186241e-08))
TWO_OVER_PI = np.float32(0.636619772367581343)


def records(n):
    return np.zeros((n, 16), dtype=np.float32)


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def ulp32(x):
    """Spacing of float32 at |x| (the smallest subnormal at 0)."""
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


def fixture_polygons():
    """{fixture: float32 vertices (n, 2)} as the device constants hold them."""
    from hostsim import sim
    return {f: sim.shape_verts(f)[0] for f in FIXTURES}


# ---------------------------------------------------------------------------------------------------------------------
# brute-force helpers (also used by test_oracle_box2d.py)
# ---------------------------------------------------------------------------------------------------------------------
def seg_dist(p, a, b):
    """Distance from point p to segment a-b."""
    ab, ap = b - a, p - a
    t = np.clip(np.dot(ap, ab) / np.dot(ab, ab), 0.0, 1.0)
    return float(np.linalg.norm(ap - t * ab))


def intersects(p1, p2, q1, q2):
    """Segments p1-p2 and q1-q2 cross (proper crossing)."""
    def orient(a, b, c):
        return (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0])
    return (orient(p1, p2, q1) * orient(p1, p2, q2) < 0) and (orient(q1, q2, p1) * orient(q1, q2, p2) < 0)


def inside(poly, p):
    """p lies in the counter-clockwise convex polygon (boundary included)."""
    n = len(poly)
    return all(((poly[(i + 1) % n][0] - poly[i][0]) * (p[1] - poly[i][1]) - (poly[(i + 1) % n][1] - poly[i][1]) * (p[0] - poly[i][0])) >= 0
               for i in range(n))


def polygon_segment_distance(world, v1, v2):
    """Distance between a convex polygon (world vertices, CCW) and the segment v1-v2; 0 when they overlap."""
    n = len(world)
    if inside(world, v1) or inside(world, v2) or any(intersects(world[i], world[(i + 1) % n], v1, v2) for i in range(n)):
        return 0.0
    return min(min(seg_dist(p, v1, v2) for p in world),
               min(seg_dist(q, world[i], world[(i + 1) % n]) for q in (v1, v2) for i in range(n)))


def outward_normals(world):
    e = np.roll(world, -1, axis=0) - world
    n = np.stack([e[:, 1], -e[:, 0]], axis=1)
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def sat_separation(wa, wb):
    """Largest separation of two convex polygons over both polygons' face normals (SAT)."""
    best = -np.inf
    for P, Q in ((wa, wb), (wb, wa)):
        for i, n in enumerate(outward_normals(P)):
            best = max(best, float(np.min((Q - P[i]) @ n)))
    return best


def transform(verts, p, q):
    """World vertices of float32 local vertices under the float32 pose (p, q = (s, c)), evaluated in float64."""
    s, c = float(q[0]), float(q[1])
    v = np.asarray(verts, dtype=np.float64)
    return np.stack([c * v[:, 0] - s * v[:, 1] + p[0], s * v[:, 0] + c * v[:, 1] + p[1]], axis=1)


def box_verts(x0, ylo, x1, yhi):
    """static_box's vertex order: from the right-most lowest corner, counter-clockwise."""
    return np.array([(x1, ylo), (x1, yhi), (x0, yhi), (x0, ylo)], dtype=np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# rot_of
# ---------------------------------------------------------------------------------------------------------------------
def rot_cases(seed=1):
    """Float32 angles: dense over |x| <= 2 pi, random up to |x| <= 1024, odd multiples of pi/4 +- 2 ulp (where rintf
    switches quadrant), +-0 and tiny |x|."""
    rng = np.random.default_rng(seed)
    parts = [np.linspace(-2 * np.pi, 2 * np.pi, 100001), rng.uniform(-1024, 1024, 100000), rng.uniform(-8, 8, 50000)]
    m = np.arange(-1303, 1304, 2)
    centre = (m * (np.pi / 4)).astype(np.float32)
    near = [centre]
    lo = hi = centre
    for _ in range(2):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        near += [lo, hi]
    parts += near
    tiny = np.array([0.0, 1e-45, 1e-40, 1e-38, 1e-30, 2.0 ** -30, 1e-7, 2.0 ** -12], dtype=np.float32)
    parts += [tiny, -tiny]
    return np.concatenate([np.asarray(p, dtype=np.float32) for p in parts])


def rot_records(x):
    r = records(len(x))
    r[:, 0] = x
    return r


def rot_bound(x):
    """The error bound of rot_of(x) for each of sin and cos, from its construction:
      k = rintf(x * 2/pi) in float32; r1 = fmaf(k, -C1, x) and r = fmaf(k, C2, r1) are each rounded once
      (<= ulp(r1) / 2 + ulp(r) / 2, carried to the result with a slope <= 1); C1 - C2 misses pi/2 by
      |pi/2 - (C1 - C2)| = 1.8e-15, which k multiplies; the minimax polynomials and their float32 evaluation are
      within 1 ulp of the result (the "~1 ulp" of the comment in b2lite.cuh)."""
    x = np.asarray(x, dtype=np.float32)
    k = np.rint((x * TWO_OVER_PI).astype(np.float32)).astype(np.float64)
    xd = x.astype(np.float64)
    r1 = xd - k * CW1                  # exact in float64: |k| < 2^11, C1 has 24 bits
    r = r1 + k * CW2
    red = np.abs(k) * abs(np.pi / 2 - (CW1 - CW2))
    return k, 0.5 * ulp32(r1) + 0.5 * ulp32(r) + red


def check_rot(x, out):
    """Indices where rot_of(x) = (out[:, 0], out[:, 1]) is further from float64 (sin x, cos x) than rot_bound allows."""
    x = np.asarray(x, dtype=np.float32)
    _, red = rot_bound(x)
    xd = x.astype(np.float64)
    bad = np.zeros(len(x), dtype=bool)
    for j, f in ((0, np.sin), (1, np.cos)):
        want = f(xd)
        got = out[:, j].astype(np.float64)
        bad |= ~(np.abs(got - want) <= ulp32(want) + red)
    return np.flatnonzero(bad)


# ---------------------------------------------------------------------------------------------------------------------
# manifolds
# ---------------------------------------------------------------------------------------------------------------------
def unpack_manifold(o):
    ids = o[8:12:3].view(np.uint32)
    return {"type": int(o[0]), "count": int(o[1]), "ln": o[2:4].astype(np.float64), "lp": o[4:6].astype(np.float64),
            "pts": [o[6:8].astype(np.float64), o[9:11].astype(np.float64)], "ids": [int(ids[0]), int(ids[1])]}


def split_id(i):
    """(indexA, indexB, typeA, typeB) of a b2ContactFeature key; type 0 = vertex, 1 = face."""
    return i & 0xff, (i >> 8) & 0xff, (i >> 16) & 0xff, (i >> 24) & 0xff


def random_pose(rng):
    a = rng.uniform(-np.pi, np.pi)
    return np.array([np.sin(a), np.cos(a)], dtype=np.float32)


def edge_polygon_cases(polys, n_random=600, seed=2):
    """(records, kinds) of edge-vs-polygon cases for every fixture: random poses near contact (the deepest vertex at
    -0.04 .. 0.05 from the edge's line, projecting anywhere from before v1 to past v2, on either side of the edge) and
    constructed ones: a face parallel to the edge and overlapping it, a vertex on the edge, the polygon past an edge
    end, behind the edge (front = false), and the deepest vertex at 2 kPolygonRadius +- a few ulp."""
    rng = np.random.default_rng(seed)
    recs, kinds = [], []

    def place(f, v1, v2, q, side, s, sep, vertex=None, kind="random"):
        v1, v2 = np.asarray(v1, dtype=np.float32), np.asarray(v2, dtype=np.float32)
        e = v2.astype(np.float64) - v1
        n1 = np.array([e[1], -e[0]]) / np.linalg.norm(e)
        nf = side * n1
        wl = transform(polys[f], (0.0, 0.0), q)
        j = int(np.argmin(wl @ nf)) if vertex is None else vertex
        p = (v1 + s * e + sep * nf - wl[j]).astype(np.float32)
        r = np.zeros(16, dtype=np.float32)
        r[0] = f; r[1:3] = v1; r[3:5] = v2; r[5:7] = p; r[7:9] = q
        recs.append(r)
        kinds.append(kind)

    for f in FIXTURES:
        for _ in range(n_random):
            th = rng.uniform(-np.pi, np.pi) if rng.random() < 0.5 else rng.uniform(-0.6, 0.6)
            length = rng.uniform(0.3, 3.0)
            c = rng.uniform(-3, 3, 2)
            d = length / 2 * np.array([np.cos(th), np.sin(th)])
            place(f, c - d, c + d, random_pose(rng), rng.choice([-1.0, 1.0]), rng.uniform(-0.3, 1.3),
                  rng.uniform(-0.04, 0.05))
        # a face parallel to the edge and overlapping it
        m = len(polys[f])
        for k in range(m):
            vk, vk1 = polys[f][k].astype(np.float64), polys[f][(k + 1) % m].astype(np.float64)
            t = vk1 - vk
            ang = -np.arctan2(t[1], t[0])      # rotates face k onto +x: its outward normal points down
            q = np.array([np.sin(ang), np.cos(ang)], dtype=np.float32)
            flen = np.linalg.norm(t)
            for sep in (-0.005, 0.0, 0.005, 0.015):
                x0 = rng.uniform(-2, 2)
                y0 = rng.uniform(-1, 1)
                v1, v2 = (x0 - 2 * flen, y0), (x0 + 2 * flen, y0)
                # edge left to right: normal1 points down, the polygon above it is behind (front = false)
                place(f, v2, v1, q, 1.0, 0.5, sep, vertex=k, kind="parallel")
                place(f, v1, v2, q, -1.0, 0.5, sep, vertex=k, kind="parallel")
        # a vertex on the edge (generic angle), and the polygon past an edge end
        for _ in range(40):
            q = random_pose(rng)
            place(f, (-1.0, 0.3), (1.5, 0.3), q, rng.choice([-1.0, 1.0]), rng.uniform(0.3, 0.7), 0.0, kind="vertex")
            place(f, (-1.0, 0.3), (1.5, 0.3), q, rng.choice([-1.0, 1.0]), rng.uniform(1.4, 2.0), rng.uniform(-0.01, 0.01),
                  kind="past_end")
        # the deepest vertex at the contact radius, +- 4 ulp
        for _ in range(40):
            q = random_pose(rng)
            for dk in range(-4, 5):
                sep = float(np.float32(RADIUS)) + dk * float(ulp32(RADIUS))
                place(f, (-1.0, 0.0), (1.5, 0.0), q, rng.choice([-1.0, 1.0]), rng.uniform(0.3, 0.7), sep, kind="radius")
    return np.stack(recs), np.array(kinds)


def box_polygon_cases(polys, n_random=500, seed=3):
    """(records, kinds) of box-vs-polygon cases for every fixture: random poses near the boxes BipedalWalkerHardcore
    builds with static_box (a stump 1 x 1 step, a stair step 4 x 0.5 steps, a pit wall 0.47 wide and 4 deep), the
    polygon's deepest vertex at -0.04 .. 0.05 from one of the box's faces."""
    rng = np.random.default_rng(seed)
    step = 14 / 30.0
    boxes = [(0.0, 0.0, step, step), (0.0, 0.0, 4 * step, 0.5 * step), (0.0, -4 * step, step, 0.0)]
    recs, kinds = [], []
    for f in FIXTURES:
        for i in range(n_random):
            bx = boxes[i % 3]
            ox, oy = rng.uniform(10, 60), rng.uniform(2, 6)
            box = np.array([bx[0] + ox, bx[1] + oy, bx[2] + ox, bx[3] + oy], dtype=np.float32)
            bv = box_verts(*box.astype(np.float64))
            face = rng.integers(0, 4)
            a, b = bv[face], bv[(face + 1) % 4]
            nrm = outward_normals(bv)[face]
            q = random_pose(rng)
            wl = transform(polys[f], (0.0, 0.0), q)
            j = int(np.argmin(wl @ nrm))
            s = rng.uniform(-0.2, 1.2)
            p = (a + s * (b - a) + rng.uniform(-0.04, 0.05) * nrm - wl[j]).astype(np.float32)
            r = np.zeros(16, dtype=np.float32)
            r[0] = f; r[1:5] = box; r[5:7] = p; r[7:9] = q
            recs.append(r)
            kinds.append("random")
    return np.stack(recs), np.array(kinds)


def _scale(*pts):
    return 1.0 + max(float(np.max(np.abs(p))) for p in pts)


def _clip_point(face_a, face_b, t, plane):
    """The point of line face_a-face_b where t . x = plane."""
    d = face_b - face_a
    den = float(t @ d)
    return face_a + (plane - float(t @ face_a)) / den * d


def check_edge_polygon(rec, out, polys):
    """Indices of edge-polygon manifolds that break one of:
      * no points when the float64 distance between the segment and the polygon exceeds 2 kPolygonRadius + bound
        (every manifold point lies inside the reference face's slab within the radius of it);
      * at least one point when the polygon's deepest vertex (along the edge normal on the centroid's side) projects
        at least 0.02 inside the edge and lies no further than 2 kPolygonRadius - bound from it;
      * the world normal is a unit vector from the edge to the polygon;
      * every point, turned into a world point and separation by b2WorldManifold::Initialize's rules, agrees with the
        same rules applied to the float64 feature its id names (a polygon vertex, or the point of a polygon face on the
        edge's side plane; an edge end or the point of the edge on a polygon face's side plane), within bound.
    bound = 32 u L: every float32 quantity here passes through at most 16 roundings of magnitude <= u L, doubled."""
    bad = []
    for i in range(len(rec)):
        r = rec[i].astype(np.float64)
        f = int(r[0])
        v1, v2, p, q = r[1:3], r[3:5], r[5:7], r[7:9]
        W = transform(polys[f], p, q)
        m = unpack_manifold(out[i])
        L = _scale(v1, v2, W)
        bound = 32 * U * L
        e = v2 - v1
        elen = np.linalg.norm(e)
        eh = e / elen
        n1 = np.array([eh[1], -eh[0]])
        cen = W.mean(axis=0)
        side = 1.0 if float((cen - v1) @ n1) >= 0 else -1.0
        nf = side * n1
        dist = polygon_segment_distance(W, v1, v2)
        if m["count"] > 0 and dist > RADIUS + bound:
            bad.append((i, "points beyond the radius", dist))
            continue
        depth = (W - v1) @ nf
        j = int(np.argmin(depth))
        s = float((W[j] - v1) @ eh)
        if (m["count"] == 0 and 0.02 <= s <= elen - 0.02 and depth[j] <= RADIUS - bound
                and abs(float((cen - v1) @ n1)) > 0.02):
            bad.append((i, "no point for a vertex inside the radius", depth[j]))
            continue
        if m["count"] == 0:
            continue
        if m["type"] == 0:
            nw = m["ln"]
        else:
            nw = -np.array([q[1] * m["ln"][0] - q[0] * m["ln"][1], q[0] * m["ln"][0] + q[1] * m["ln"][1]])
        foot = v1 + np.clip(float((cen - v1) @ eh), 0.0, elen) * eh
        if abs(np.linalg.norm(nw) - 1.0) > 8 * U or float(nw @ (cen - foot)) <= 0.0:
            bad.append((i, "normal", nw))
            continue
        nPoly = outward_normals(W)
        for k in range(m["count"]):
            lp = m["pts"][k]
            ia, ib, ta, tb = split_id(m["ids"][k])
            if m["type"] == 0:
                # Initialize, e_faceA: clip = xfB * lp, plane = localPoint, normal = localNormal
                clip = transform(lp[None, :], p, q)[0]
                plane, nrm = m["lp"], m["ln"]
                if tb == 0:
                    want = W[ib]
                else:
                    want = _clip_point(W[ib], W[(ib + 1) % len(W)], eh, float(eh @ (v1 if ia == 0 else v2)))
                want_plane, want_n = (v1, nf)
            else:
                # e_faceB: clip = lp (the edge's frame is the world), plane = xfB * localPoint, normal = q * localNormal
                clip = lp
                plane = transform(m["lp"][None, :], p, q)[0]
                nrm = -nw
                tf = np.array([nPoly[ia][1], -nPoly[ia][0]])
                cands = [v1, v2] + [_clip_point(v1, v2, tf, float(tf @ W[c])) for c in (ia, (ia + 1) % len(W))
                                    if abs(float(tf @ e)) > 1e-9]
                want = min(cands, key=lambda c: np.linalg.norm(c - clip))
                want_plane, want_n = W[ia], nPoly[ia]
            sep = float((clip - plane) @ nrm) - RADIUS
            want_sep = float((want - want_plane) @ want_n) - RADIUS
            if np.linalg.norm(clip - want) > bound or abs(sep - want_sep) > bound:
                bad.append((i, "point", k, clip, want, sep, want_sep))
                break
    return bad


def check_box_polygon(rec, out, polys):
    """Indices of box-polygon manifolds (b2CollidePolygons) that break one of:
      * no points when the float64 SAT separation of the box and the polygon exceeds 2 kPolygonRadius + bound;
      * at least one point when the polygon's deepest vertex along a box face's normal projects at least 0.02 inside
        that face and lies within 2 kPolygonRadius - bound of it, and no other box face separates more;
      * the world normal is a unit vector from the box to the polygon;
      * every point agrees with the float64 feature its id names: a vertex of the incident polygon, or the point of
        the incident face on the reference face's side plane, which Box2D moves out by the contact radius;
        its Initialize separation agrees with the float64 one.  bound = 32 u L as for the edge."""
    bad = []
    for i in range(len(rec)):
        r = rec[i].astype(np.float64)
        f = int(r[0])
        box, p, q = r[1:5], r[5:7], r[7:9]
        A = box_verts(*box)
        B = transform(polys[f], p, q)
        m = unpack_manifold(out[i])
        L = _scale(A, B)
        bound = 32 * U * L
        sep = sat_separation(A, B)
        if m["count"] > 0 and sep > RADIUS + bound:
            bad.append((i, "points beyond the radius", sep))
            continue
        nA = outward_normals(A)
        face_sep = [float(np.min((B - A[k]) @ nA[k])) for k in range(4)]
        kf = int(np.argmax(face_sep))
        j = int(np.argmin((B - A[kf]) @ nA[kf]))
        t = A[(kf + 1) % 4] - A[kf]
        s = float((B[j] - A[kf]) @ t) / float(np.linalg.norm(t))
        if (m["count"] == 0 and 0.02 <= s <= np.linalg.norm(t) - 0.02 and face_sep[kf] <= RADIUS - bound
                and face_sep[kf] >= sep - 1e-3):
            bad.append((i, "no point for a vertex inside the radius", face_sep[kf]))
            continue
        if m["count"] == 0:
            continue
        ln, lpl = m["ln"], m["lp"]
        if m["type"] == 0:
            nw, planew = ln, lpl
            ref, inc = A, B
        else:
            nb = np.array([q[1] * ln[0] - q[0] * ln[1], q[0] * ln[0] + q[1] * ln[1]])
            nw, planew = -nb, transform(lpl[None, :], p, q)[0]
            ref, inc = B, A
        cB = B.mean(axis=0)
        if abs(np.linalg.norm(nw) - 1.0) > 8 * U or float(nw @ (cB - A.mean(axis=0))) <= 0.0:
            bad.append((i, "normal", nw))
            continue
        nref = nw if m["type"] == 0 else -nw
        for k in range(m["count"]):
            lp = m["pts"][k]
            clip = transform(lp[None, :], p, q)[0]          # localPoint is in B's frame (xf2 = xfB or identity)
            if m["type"] == 1:
                clip = lp
            ia, ib, ta, tb = split_id(m["ids"][k])
            # the reference face's index: the one whose plane is localPoint's face
            inc_vertex, inc_kind, ref_vertex = (ib, tb, ia) if m["type"] == 0 else (ia, ta, ib)
            if inc_kind == 0:
                want = inc[inc_vertex]
            else:
                # side planes: t . x = t . v11 - r (at the reference face's first vertex), t . v12 + r (its second)
                nr = len(ref)
                rf = next(c for c in range(nr) if np.allclose(outward_normals(ref)[c], nref, atol=1e-4)
                          and abs(float((ref[c] - planew) @ nref)) < 1e-4)
                v11, v12 = ref[rf], ref[(rf + 1) % nr]
                tg = (v12 - v11) / np.linalg.norm(v12 - v11)
                plane = float(tg @ v11) - RADIUS if ref_vertex == rf else float(tg @ v12) + RADIUS
                want = _clip_point(inc[inc_vertex], inc[(inc_vertex + 1) % len(inc)], tg, plane)
            s_got = float((clip - planew) @ nref) - RADIUS
            s_want = float((want - planew) @ nref) - RADIUS
            if np.linalg.norm(clip - want) > bound or abs(s_got - s_want) > bound:
                bad.append((i, "point", k, clip, want))
                break
    return bad


def perturbed(rec, rng, ulps=1):
    """The records with the pose (p, q) moved by up to `ulps` float32 steps per component."""
    out = rec.copy()
    for c in range(5, 9):
        col = out[:, c]
        for _ in range(ulps):
            step = rng.choice([-1, 0, 1], size=len(col))
            col = np.where(step > 0, np.nextafter(col, np.float32(np.inf)),
                           np.where(step < 0, np.nextafter(col, np.float32(-np.inf)), col))
        out[:, c] = col
    return out


# ---------------------------------------------------------------------------------------------------------------------
# ray casts
# ---------------------------------------------------------------------------------------------------------------------
def edge_ray_cases(seed=4, n=20000):
    """Rays against edges: random, through the edge's ends (s = 0, 1), parallel to it (denominator 0), starting on it
    (t = 0), and with maxFraction below 1."""
    rng = np.random.default_rng(seed)
    r = records(n)
    v1 = rng.uniform(-3, 3, (n, 2))
    v2 = v1 + rng.uniform(-1, 1, (n, 2))
    p1 = rng.uniform(-3, 3, (n, 2))
    p2 = p1 + rng.uniform(-4, 4, (n, 2))
    mf = np.where(rng.random(n) < 0.3, rng.uniform(0.2, 1.0, n), 1.0)
    kind = rng.integers(0, 5, n)
    # through an end: aim p2 beyond v1 or v2 along p1 -> end
    end = np.where(rng.random((n, 1)) < 0.5, v1, v2)
    p2 = np.where((kind == 1)[:, None], p1 + (end - p1) * rng.uniform(1.1, 3.0, (n, 1)), p2)
    # parallel to a horizontal edge
    y = rng.uniform(-2, 2, n)
    hz = kind == 2
    v1[hz, 1] = y[hz]; v2[hz, 1] = y[hz]
    p2[hz, 1] = p1[hz, 1]
    # starting on a horizontal edge
    st = kind == 3
    v1[st, 1] = y[st]; v2[st, 1] = y[st]
    p1[st] = np.stack([v1[st, 0] + rng.uniform(0.2, 0.8, st.sum()) * (v2[st, 0] - v1[st, 0]), y[st]], axis=1)
    r[:, 0:2], r[:, 2:4], r[:, 4:6], r[:, 6:8], r[:, 8] = v1, v2, p1, p2, mf
    return r


def segment_params(v1, v2, p1, p2):
    """float64 (t along p1 -> p2, s along v1 -> v2, the denominator n . d with the unit edge normal)."""
    d, e, w = p2 - p1, v2 - v1, v1 - p1
    n = np.stack([e[:, 1], -e[:, 0]], axis=1) / np.linalg.norm(e, axis=1, keepdims=True)
    den = np.sum(n * d, axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.sum(n * w, axis=1) / den
        q = p1 + t[:, None] * d
        s = np.sum((q - v1) * e, axis=1) / np.sum(e * e, axis=1)
    return t, s, den


def ray_t_bound(w, d, t, den):
    """|t - t*| for t = (n . w) / (n . d) in float32 with n normalised in float32: the numerator and denominator each
    carry <= 8 roundings relative to |w| and |d| (n: 4, differences and dot: 4), the quotient one more."""
    return 8 * U * (np.linalg.norm(w, axis=1) + np.abs(t) * np.linalg.norm(d, axis=1)) / np.abs(den) + 2 * U * np.abs(t)


def check_edge_ray(rec, out):
    """Indices where edge_raycast disagrees with the float64 segment intersection: a hit must be a float64 hit with
    |t - t*| <= ray_t_bound, and a float64 hit must be found, except in a band around the decisions -- s within
    the bound of 0 or 1, t within the bound of 0 or maxFraction, or a near-parallel ray (|n . d| < 1e-6 |d|)."""
    r = rec.astype(np.float64)
    v1, v2, p1, p2, mf = r[:, 0:2], r[:, 2:4], r[:, 4:6], r[:, 6:8], r[:, 8]
    t, s, den = segment_params(v1, v2, p1, p2)
    d = p2 - p1
    hit = out[:, 0] == 1.0
    got = out[:, 1].astype(np.float64)
    with np.errstate(invalid="ignore"):
        tb = ray_t_bound(v1 - p1, d, t, den)
        sb = (tb * np.linalg.norm(d, axis=1) + 16 * U * _scale(v1, v2, p1, p2)) / np.linalg.norm(v2 - v1, axis=1)
        grazing = np.abs(den) < 1e-6 * np.linalg.norm(d, axis=1)
        want = (t >= 0) & (t <= mf) & (s >= 0) & (s <= 1) & ~grazing
        clear_hit = want & (t >= tb) & (t <= mf - tb) & (s >= sb) & (s <= 1 - sb)
        clear_miss = ~grazing & ~((t >= -tb) & (t <= mf + tb) & (s >= -sb) & (s <= 1 + sb))
        bad = (clear_hit & ~hit) | (clear_miss & hit) | (hit & ~grazing & ~(np.abs(got - t) <= tb))
        # an exactly parallel ray has no hit
        bad |= (den == 0) & hit
    return np.flatnonzero(bad)


def box_ray_cases(seed=5, n=20000):
    """Rays against hardcore boxes: random, horizontal and vertical (denominators 0), through corners, from inside
    the box, with maxFraction below 1."""
    rng = np.random.default_rng(seed)
    r = records(n)
    x0 = rng.uniform(10, 60, n)
    w = rng.choice([14 / 30.0, 4 * 14 / 30.0], n)
    h = rng.choice([14 / 30.0, 0.5 * 14 / 30.0, 4 * 14 / 30.0], n)
    ylo = rng.uniform(2, 6, n)
    box = np.stack([x0, ylo, x0 + w, ylo + h], axis=1).astype(np.float32).astype(np.float64)
    c = (box[:, 0:2] + box[:, 2:4]) / 2
    p1 = c + rng.uniform(-3, 3, (n, 2))
    p2 = c + rng.uniform(-3, 3, (n, 2))
    kind = rng.integers(0, 5, n)
    hz, vt, cor = kind == 1, kind == 2, kind == 3
    p2[hz, 1] = p1[hz, 1]
    p2[vt, 0] = p1[vt, 0]
    corner = np.stack([box[:, 0], box[:, 3]], axis=1)
    p2[cor] = p1[cor] + (corner[cor] - p1[cor]) * rng.uniform(1.1, 2.0, (cor.sum(), 1))
    mf = np.where(rng.random(n) < 0.3, rng.uniform(0.2, 1.0, n), 1.0)
    r[:, 0:4], r[:, 4:6], r[:, 6:8], r[:, 8] = box, p1, p2, mf
    return r


def slab(box, p1, p2):
    """float64 slab intersection of segments p1 -> p2 with boxes: (entry t, exit t, the entry's margin to the
    other slab's edges: how far the entry point is from leaving the face it enters)."""
    d = p2 - p1
    lo, hi = box[:, 0:2], box[:, 2:4]
    with np.errstate(divide="ignore", invalid="ignore"):
        ta, tb = (lo - p1) / d, (hi - p1) / d
    tmin = np.where(d == 0, np.where((p1 >= lo) & (p1 <= hi), -np.inf, np.inf), np.minimum(ta, tb))
    tmax = np.where(d == 0, np.where((p1 >= lo) & (p1 <= hi), np.inf, -np.inf), np.maximum(ta, tb))
    enter, leave = tmin.max(axis=1), tmax.min(axis=1)
    return enter, leave


def check_box_ray(rec, out):
    """Indices where static_box_raycast disagrees with the float64 slab test: a segment that starts outside the box
    and enters it at t in [0, maxFraction] is a hit at that t (Box2D reports no hit for a segment starting inside);
    a band of the bound around t = 0, t = maxFraction and entry = exit (corners, faces grazed) is not decided."""
    r = rec.astype(np.float64)
    box, p1, p2, mf = r[:, 0:4], r[:, 4:6], r[:, 6:8], r[:, 8]
    enter, leave = slab(box, p1, p2)
    d = p2 - p1
    L = _scale(box, p1, p2)
    dn = np.linalg.norm(d, axis=1)
    tb = 16 * U * L / np.maximum(dn, 1e-30) + 2 * U
    hit = out[:, 0] == 1.0
    got = out[:, 1].astype(np.float64)
    with np.errstate(invalid="ignore"):
        want = (enter > 0) & (enter <= leave) & (enter <= mf)
        clear_hit = want & (enter >= tb) & (enter <= leave - tb) & (enter <= mf - tb)
        clear_miss = ~((enter >= -tb) & (enter <= leave + tb) & (enter <= mf + tb))
        bad = (clear_hit & ~hit) | (clear_miss & hit) | (hit & want & ~(np.abs(got - enter) <= tb))
    return np.flatnonzero(bad)


def nearest_hit_cases(seed=6, rays=2000, edges=8):
    """A ray crossing a zig-zag polyline of `edges` edges several times, the edges visited in a shuffled order."""
    rng = np.random.default_rng(seed)
    xs = np.linspace(0.0, 4.0, edges + 1)
    ys = rng.uniform(-0.5, 0.5, (rays, edges + 1))
    order = np.stack([rng.permutation(edges) for _ in range(rays)])
    p1 = np.stack([rng.uniform(-0.5, 0.5, rays), rng.uniform(-2.5, -1.0, rays)], axis=1)
    p2 = np.stack([rng.uniform(3.5, 4.5, rays), rng.uniform(1.0, 2.5, rays)], axis=1)
    return xs, ys.astype(np.float32), order, p1.astype(np.float32), p2.astype(np.float32)


def fold_nearest(probe, xs, ys, order, p1, p2):
    """env_post's loop: maxFraction starts at 1 and drops to every hit; the fraction is the last hit's t."""
    rays = len(p1)
    frac = np.ones(rays, dtype=np.float32)
    for k in range(order.shape[1]):
        e = order[:, k]
        r = records(rays)
        r[:, 0] = xs[e]; r[:, 1] = ys[np.arange(rays), e]; r[:, 2] = xs[e + 1]; r[:, 3] = ys[np.arange(rays), e + 1]
        r[:, 4:6], r[:, 6:8], r[:, 8] = p1, p2, frac
        o = probe(OP_EDGE_RAYCAST, r)
        frac = np.where(o[:, 0] == 1.0, o[:, 1], frac)
    return frac


def nearest_hit_reference(xs, ys, p1, p2):
    """float64 nearest t over every edge of the polyline, 1 when none is hit."""
    rays, edges = ys.shape[0], ys.shape[1] - 1
    best = np.ones(rays)
    for e in range(edges):
        v1 = np.stack([np.full(rays, xs[e]), ys[:, e]], axis=1).astype(np.float64)
        v2 = np.stack([np.full(rays, xs[e + 1]), ys[:, e + 1]], axis=1).astype(np.float64)
        t, s, den = segment_params(v1, v2, p1.astype(np.float64), p2.astype(np.float64))
        ok = (t >= 0) & (t <= 1) & (s >= 0) & (s <= 1)
        best = np.where(ok & (t < best), t, best)
    return best


# ---------------------------------------------------------------------------------------------------------------------
# solve22 / solve33
# ---------------------------------------------------------------------------------------------------------------------
def solve_cases(seed=7, n=4000):
    """(records, kinds): symmetric K as b2RevoluteJoint builds it (masses 0.5 .. 20, inertias, anchors up to 1.5 m),
    the same with one body's inverse inertia 1e-5 .. 1e-3 of the other's (near singular), general non-symmetric
    well-conditioned K (so that every entry's orientation is pinned), and exactly singular K."""
    rng = np.random.default_rng(seed)
    recs, kinds = [], []
    for i in range(n):
        kind = ("joint", "near_singular", "general", "singular")[i % 4]
        if kind in ("joint", "near_singular"):
            mA, mB = 1 / rng.uniform(0.5, 20), 1 / rng.uniform(0.5, 20)
            iA, iB = 1 / rng.uniform(0.05, 5), 1 / rng.uniform(0.05, 5)
            if kind == "near_singular":
                mA, iA = 0.0, iA * rng.uniform(1e-5, 1e-3)
                mB = mB * rng.uniform(1e-5, 1e-3)
            rA, rB = rng.uniform(-1.5, 1.5, 2), rng.uniform(-1.5, 1.5, 2)
            K = np.zeros((3, 3))
            K[0, 0] = mA + mB + rA[1] ** 2 * iA + rB[1] ** 2 * iB
            K[1, 0] = -rA[1] * rA[0] * iA - rB[1] * rB[0] * iB
            K[2, 0] = -rA[1] * iA - rB[1] * iB
            K[1, 1] = mA + mB + rA[0] ** 2 * iA + rB[0] ** 2 * iB
            K[2, 1] = rA[0] * iA + rB[0] * iB
            K[2, 2] = iA + iB
            K = K + np.tril(K, -1).T
        elif kind == "general":
            K = rng.normal(size=(3, 3)) + 3 * np.eye(3)
        else:
            a = rng.integers(1, 5, 3).astype(np.float64)
            K = np.outer(a, a) if i % 8 == 3 else np.zeros((3, 3))
        b = rng.normal(size=3) * 10
        r = np.zeros(16, dtype=np.float32)
        r[0:9] = K.ravel()          # K[c][r] = in[3 c + r]
        r[9:12] = b
        recs.append(r)
        kinds.append(kind)
    return np.stack(recs), np.array(kinds)


def _permanent(M):
    if len(M) == 2:
        return M[0, 0] * M[1, 1] + M[0, 1] * M[1, 0]
    return sum(M[0, j] * _permanent(np.delete(np.delete(M, 0, 0), j, 1)) for j in range(3))


def check_solve(rec, out, dim, kinds):
    """Indices where solve22 / solve33 (Cramer's rule in float32) misses numpy.linalg.solve of the same float32 K and
    b by more than the running error bound of Cramer's rule, or where a K whose float32 determinant is 0 does not
    give x = 0 (Box2D's `det != 0` guard).  A determinant or numerator evaluated by cofactors in float32 is within
    gamma * per(|M|) of the exact one (per: the permanent, the same sum with every product taken positive;
    gamma = 3 (dim - 1) u covers the 2 roundings in a row of a 2 x 2 and the 5 of a 3 x 3), so
    |x_i - x*_i| <= gamma (per(|M_i|) + per(|M|) |x*_i|) / (|det M| - gamma per(|M|)) + 2 u |x*_i| (the reciprocal
    and the product).  Near-singular K make the bound wide; that is what the condition of K implies."""
    bad = []
    for i in range(len(rec)):
        M = rec[i, 0:9].astype(np.float64).reshape(3, 3).T[:dim, :dim]     # M[r][c] = K[c][r]
        b = rec[i, 9:9 + dim].astype(np.float64)
        x = out[i, 0:dim].astype(np.float64)
        if kinds[i] == "singular":
            if not np.all(x == 0.0):
                bad.append(i)
            continue
        want = np.linalg.solve(M, b)
        det = np.linalg.det(M)
        gamma = 3 * (dim - 1) * U
        slack = abs(det) - gamma * _permanent(np.abs(M))
        for c in range(dim):
            Mi = M.copy()
            Mi[:, c] = b
            tol = (gamma * (_permanent(np.abs(Mi)) + _permanent(np.abs(M)) * abs(want[c])) / slack if slack > 0 else np.inf) \
                + 2 * U * abs(want[c])
            if not abs(x[c] - want[c]) <= tol:
                bad.append(i)
                break
    return bad
