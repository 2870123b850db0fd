"""Float64 references for the Box2D solver steps of csrc/b2lite.cuh (the contact and joint constraints, integration,
the host-computed mass properties), through the probe ops of csrc/b2probe.cuh, and the case generators and checks that
tests/test_box2d_solvers_cpu.py (host build) and tests/test_gpu_box2d_solvers.py (device) both run.

A probe is `probe(op, records) -> out` over float32 records (n, 16), as in tests/box2d_geometry.py.  Each check
returns the indices of the records that break a contract of the step -- complementarity, clamps, residuals,
momentum balance -- recomputed in float64 from the float32 inputs and outputs, not a copy of the step's code.

Bounds count float32 roundings as the geometry checks do: u = 2^-24; a quantity that passes through at most k
roundings, each relative to a magnitude <= S, is within k u S, and the stated factors double that count.  Where a
linear solve is involved the bound is multiplied by the float64 condition number of its matrix (the forward error of a
solve in float32 is the backward error times the condition).  The body angles the device turns into rotations with
rot_of (within 2 ulp of float64 sin / cos, tests/test_box2d_geometry_cpu.py) are turned into rotations here with
float64 sin / cos of the same float32 angle; the 32 u L bounds absorb that difference.
"""
import numpy as np

import box2d_geometry as g

U = g.U
OP_CONTACT_INIT, OP_CONTACT_VELOCITY, OP_CONTACT_POSITION, OP_JOINT_VELOCITY, OP_JOINT_POSITION, OP_INTEGRATE, \
    OP_CONSTS = range(9, 16)
CASE_NONE, CASE_BOTH, CASE_FIRST, CASE_SECOND, CASE_NEITHER, ONE_POINT = 0, 1, 2, 3, 4, -1

# Box2D 2.3 b2Settings.h, as the float32 constants of b2lite.cuh hold them
F32 = lambda x: float(np.float32(x))
DT = F32(1.0 / 50)
POLYGON_RADIUS = F32(0.01)
LINEAR_SLOP = F32(0.005)
ANGULAR_SLOP = F32(2.0 / 180.0 * 3.14159265359)
MAX_LINEAR_CORRECTION = F32(0.2)
MAX_ANGULAR_CORRECTION = F32(8.0 / 180.0 * 3.14159265359)
MAX_TRANSLATION = F32(2.0)
MAX_ROTATION = F32(0.5 * 3.14159265359)
BAUMGARTE = F32(0.2)

# ---------------------------------------------------------------------------------------------------------------------
# the task constants, as gym's lunar_lander.py and bipedal_walker.py write them
# ---------------------------------------------------------------------------------------------------------------------
SCALE = 30.0
LANDER_POLY = [(-14, +17), (-17, 0), (-17, -10), (+17, -10), (+17, 0), (+14, +17)]
LL_LEG_AWAY, LL_LEG_DOWN, LL_LEG_W, LL_LEG_H = 20, 18, 2, 8
HULL_POLY = [(-30, +9), (+6, +9), (+34, +1), (+34, -8), (-30, -8)]
BW_LEG_DOWN, BW_LEG_W, BW_LEG_H = -8 / SCALE, 8 / SCALE, 34 / SCALE
DEFAULT_FRICTION = 0.2      # b2FixtureDef's default: the legs' fixture definitions give none


def box(hx, hy):
    return [(-hx, -hy), (hx, -hy), (hx, hy), (-hx, hy)]


# fixture: (float64 vertices, density, friction)
FIXTURE_DEFS = {
    0: ([(x / SCALE, y / SCALE) for x, y in LANDER_POLY], 5.0, 0.1),
    1: (box(LL_LEG_W / SCALE, LL_LEG_H / SCALE), 1.0, DEFAULT_FRICTION),
    2: ([(x / SCALE, y / SCALE) for x, y in HULL_POLY], 5.0, 0.1),
    3: (box(BW_LEG_W / 2, BW_LEG_H / 2), 1.0, DEFAULT_FRICTION),
    4: (box(0.8 * BW_LEG_W / 2, BW_LEG_H / 2), 1.0, DEFAULT_FRICTION),
}
# joint: (anchorA, anchorB, lower, upper, fixture A, fixture B, maxMotorTorque)
JOINT_DEFS = {
    0: ((0, 0), (-1 * LL_LEG_AWAY / SCALE, LL_LEG_DOWN / SCALE), +0.9 - 0.5, +0.9, 0, 1, 40.0),
    1: ((0, 0), (+1 * LL_LEG_AWAY / SCALE, LL_LEG_DOWN / SCALE), -0.9, -0.9 + 0.5, 0, 1, 40.0),
    2: ((0, BW_LEG_DOWN), (0, BW_LEG_H / 2), -0.8, 1.1, 2, 3, 80.0),
    3: ((0, -BW_LEG_H / 2), (0, BW_LEG_H / 2), -1.6, -0.1, 3, 4, 80.0),
    4: ((0, BW_LEG_DOWN), (0, BW_LEG_H / 2), -0.8, 1.1, 2, 3, 80.0),
    5: ((0, -BW_LEG_H / 2), (0, BW_LEG_H / 2), -1.6, -0.1, 3, 4, 80.0),
}


def polygon_mass(verts, density):
    """Exact float64 mass, centroid and rotational inertia about the centroid of a uniform polygon (Green's theorem);
    the vertices in either winding (b2PolygonShape::Set takes their hull)."""
    v = np.asarray(verts, dtype=np.float64)
    if np.sum(v[:, 0] * np.roll(v[:, 1], -1) - np.roll(v[:, 0], -1) * v[:, 1]) < 0:
        v = v[::-1]
    x, y = v[:, 0], v[:, 1]
    x1, y1 = np.roll(x, -1), np.roll(y, -1)
    cr = x * y1 - x1 * y
    area = cr.sum() / 2
    cx = ((x + x1) * cr).sum() / (6 * area)
    cy = ((y + y1) * cr).sum() / (6 * area)
    i_origin = density * (cr * (x * x + x * x1 + x1 * x1 + y * y + y * y1 + y1 * y1)).sum() / 12
    mass = density * area
    return mass, np.array([cx, cy]), i_origin - mass * (cx * cx + cy * cy)


def check_fixture_consts(fc):
    """What in the fixture constants breaks, against gym's: invMass, localCenter and invI of the five fixtures against
    the exact float64 integrals of the polygons gym builds, with its densities, and friction (b2FixtureDef's default
    0.2 where gym gives none).  The host computes the mass properties in float32 from float32 vertices (relative error
    u each) over at most 6 triangles, each term through <= 8 roundings, all of one sign (the triangles fan out from the
    vertex mean, inside the polygon): 32 u, and moving the inertia to the centroid subtracts m |c|^2, which scales that
    by (I_origin + m |c|^2) / I_centroid."""
    bad = []
    for f, (verts, density, friction) in FIXTURE_DEFS.items():
        mass, cen, inertia = polygon_mass(verts, density)
        c = fc[f]
        L = max(abs(x) for v in verts for x in v)
        growth = (inertia + 2 * mass * float(cen @ cen)) / inertia
        if not abs(1 / c["invMass"] / mass - 1) <= 32 * U:
            bad.append(("mass", f, 1 / c["invMass"], mass))
        if not np.all(np.abs(c["lc"] - cen) <= 32 * U * L):
            bad.append(("localCenter", f, c["lc"], cen))
        if not abs(1 / c["invI"] / inertia - 1) <= 32 * U * growth:
            bad.append(("inertia", f, 1 / c["invI"], inertia))
        if c["friction"] != np.float32(friction) or c["count"] != len(verts):
            bad.append(("friction / vertex count", f, c["friction"], c["count"]))
    return bad


def check_joint_consts(jc):
    """What in the joint constants breaks: anchors, limits and fixture pairs must be float32 of gym's values."""
    bad = []
    for j, (anchorA, anchorB, lower, upper, fA, fB, _) in JOINT_DEFS.items():
        d = jc[j]
        if not (np.array_equal(d["anchorA"], np.float32(anchorA)) and np.array_equal(d["anchorB"], np.float32(anchorB))):
            bad.append(("anchors", j, d["anchorA"], d["anchorB"]))
        if d["lower"] != np.float32(lower) or d["upper"] != np.float32(upper):
            bad.append(("limits", j, d["lower"], d["upper"]))
        if (d["fA"], d["fB"]) != (fA, fB):
            bad.append(("fixtures", j, d["fA"], d["fB"]))
    return bad


def fixture_consts(probe):
    """{fixture: dict(invMass, invI, lc, friction)} as the device constants hold them."""
    r = g.records(5)
    r[:, 1] = np.arange(5)
    o = probe(OP_CONSTS, r).astype(np.float64)
    return {f: {"invMass": o[f, 0], "invI": o[f, 1], "lc": o[f, 2:4], "friction": o[f, 4], "centroid": o[f, 5:7],
                "count": int(o[f, 7])} for f in range(5)}


def joint_consts(probe):
    r = g.records(6)
    r[:, 0] = 1
    r[:, 1] = np.arange(6)
    o = probe(OP_CONSTS, r).astype(np.float64)
    return {j: {"anchorA": o[j, 0:2], "anchorB": o[j, 2:4], "lower": o[j, 4], "upper": o[j, 5], "fA": int(o[j, 6]),
                "fB": int(o[j, 7])} for j in range(6)}


def rot(a):
    a = np.asarray(a, dtype=np.float64)
    return np.sin(a), np.cos(a)


def rmul(s, c, v):
    return np.stack([c * v[..., 0] - s * v[..., 1], s * v[..., 0] + c * v[..., 1]], axis=-1)


def cross(a, b):
    return a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]


def cross_sv(w, r):
    """w x r for a scalar w."""
    return np.stack([-w * r[..., 1], w * r[..., 0]], axis=-1)


def tangent_of(n):
    return np.stack([n[..., 1], -n[..., 0]], axis=-1)


def norm(x):
    return np.linalg.norm(x, axis=-1)


# ---------------------------------------------------------------------------------------------------------------------
# contacts
# ---------------------------------------------------------------------------------------------------------------------
def touching_contacts(probe, polys, seed=21):
    """Contact records {f, c, a, type, localNormal, localPoint, lp1, lp2, pointCount} from the touching poses of the
    geometry tests' edge- and box-polygon generators (every fixture; manifolds with at least one point).  The body
    state is the pose's: a = the angle of (s, c), c = the origin plus the rotated local centre, in float32."""
    from hostsim import sim
    out = []
    for gen, op in ((g.edge_polygon_cases, g.OP_EDGE_POLYGON), (g.box_polygon_cases, g.OP_BOX_POLYGON)):
        rec, _ = gen(polys)
        m = probe(op, rec)
        keep = m[:, 1] > 0
        rec, m = rec[keep], m[keep]
        f = rec[:, 0].astype(int)
        q = rec[:, 7:9].astype(np.float64)
        a = np.arctan2(q[:, 0], q[:, 1]).astype(np.float32)
        s, c = rot(a)
        lc = np.stack([sim.shape_verts(k)[1] for k in range(5)]).astype(np.float64)[f]
        cen = (rec[:, 5:7].astype(np.float64) + rmul(s, c, lc)).astype(np.float32)
        r = g.records(len(rec))
        r[:, 0] = f
        r[:, 1:3] = cen
        r[:, 3] = a
        r[:, 4] = m[:, 0]
        r[:, 5:9] = m[:, 2:6]
        r[:, 9:11] = m[:, 6:8]
        r[:, 11:13] = m[:, 9:11]
        r[:, 13] = m[:, 1]
        out.append(r)
    return np.concatenate(out)


def contact_geometry(rec, fc):
    """float64 world normal (from the ground into the body), the manifold points in world coordinates and their
    separations, at the record's body state.  e_faceA (type 0): the reference face is the ground's, its plane through
    localPoint with normal localNormal; the points are the body's, lp in the body frame.  e_faceB (type 1): the
    reference face is the body's (in its frame), the points the ground's, lp in world coordinates.  The separation is
    the distance from the reference face's plane less both polygons' radii."""
    r = rec.astype(np.float64)
    f = r[:, 0].astype(int)
    cB, a, typ = r[:, 1:3], r[:, 3], r[:, 4]
    ln, lpl = r[:, 5:7], r[:, 7:9]
    lps = [r[:, 9:11], r[:, 11:13]]
    s, c = rot(a)
    lc = np.stack([fc[k]["lc"] for k in f])
    org = cB - rmul(s, c, lc)
    face_a = typ == 0
    n_ref = np.where(face_a[:, None], ln, rmul(s, c, ln))
    plane = np.where(face_a[:, None], lpl, org + rmul(s, c, lpl))
    normal = np.where(face_a[:, None], n_ref, -n_ref)
    pts, seps, mids = [], [], []
    for lp in lps:
        clip = np.where(face_a[:, None], org + rmul(s, c, lp), lp)
        sep = np.sum((clip - plane) * n_ref, axis=1) - 2 * POLYGON_RADIUS
        # the midpoint of the reference face's surface (the clip point projected on the plane, moved out by the
        # radius) and the incident polygon's surface (the clip point moved in by the radius)
        on_ref = clip - (np.sum((clip - plane) * n_ref, axis=1) - POLYGON_RADIUS)[:, None] * n_ref
        on_inc = clip - POLYGON_RADIUS * n_ref
        pts.append(clip)
        seps.append(sep)
        mids.append((on_ref + on_inc) / 2)
    return normal, pts, seps, mids


def masses(fc, f, normal, rBs):
    """float64 normal / tangent masses and the block K of a body's contact points."""
    mB = np.array([fc[k]["invMass"] for k in f])
    iB = np.array([fc[k]["invI"] for k in f])
    t = tangent_of(normal)
    rn = [cross(rb, normal) for rb in rBs]
    rt = [cross(rb, t) for rb in rBs]
    kn = [mB + iB * x * x for x in rn]
    kt = [mB + iB * x * x for x in rt]
    k12 = mB + iB * rn[0] * rn[1]
    return mB, iB, rn, rt, kn, kt, k12


def check_contact_init(rec, out, fc):
    """Indices of PROBE_CONTACT_INIT outputs that break:
      * the normal is the float64 world normal, the points' rB are the float64 midpoints minus the centre of mass,
        within 32 u L (L: the coordinates' magnitude, every quantity passes through <= 16 roundings);
      * normal and tangent masses are 1 / (mB + iB (rB x d)^2) of the float64 rB, within the rB error carried through
        (2 iB |rB x d| |drB| relative to k) plus 8 u;
      * the block K equals the float64 one within the same carried error, and the 2-point record keeps its second
        point exactly when k11^2 < 1000 (k11 k22 - k12^2) in float64, outside the band that error leaves."""
    bad = []
    f = rec[:, 0].astype(int)
    normal, _, _, mids = contact_geometry(rec, fc)
    cB = rec[:, 1:3].astype(np.float64)
    pc_in = rec[:, 13].astype(int)
    o = out.astype(np.float64)
    L = 1.0 + np.max(np.abs(rec[:, 1:13].astype(np.float64)), axis=1)
    tol_r = 32 * U * L
    rBs = [m - cB for m in mids]
    mB, iB, rn, rt, kn, kt, k12 = masses(fc, f, normal, rBs)
    got_n = o[:, 0:2]
    bad_n = norm(got_n - normal) > 32 * U
    for p in range(2):
        live = pc_in > p
        got_r = o[:, 2 + 2 * p:4 + 2 * p]
        dk = 2 * iB * (np.abs(rn[p]) + np.abs(rt[p])) * (tol_r + 32 * U * norm(rBs[p])) + 8 * U * (kn[p] + kt[p])
        bad_r = live & (norm(got_r - rBs[p]) > tol_r)
        with np.errstate(divide="ignore"):
            bad_m = live & ((np.abs(1 / o[:, 6 + p] - kn[p]) > dk) | (np.abs(1 / o[:, 8 + p] - kt[p]) > dk))
        bad += list(np.flatnonzero(bad_r | bad_m))
    two = pc_in == 2
    k11, k22 = kn[0], kn[1]
    # the entries' error dk, the determinant's 2 (k11 + k22 + |k12|) dk + 4 u (k11 k22 + k12^2)
    dk = 2 * iB * (np.abs(rn[0]) + np.abs(rn[1])) * (tol_r + 32 * U * (norm(rBs[0]) + norm(rBs[1]))) \
        + 8 * U * (k11 + k22 + np.abs(k12))
    det = k11 * k22 - k12 * k12
    ddet = 2 * (k11 + k22 + np.abs(k12)) * dk + 4 * U * (k11 * k22 + k12 * k12)
    margin = k11 * k11 - 1000 * det
    dmargin = 2 * k11 * dk + 1000 * ddet + 4 * U * k11 * k11
    want2 = margin < -dmargin
    want1 = margin > dmargin
    got = o[:, 10].astype(int)
    bad += list(np.flatnonzero(two & ((want2 & (got != 2)) | (want1 & (got != 1)))))
    kept = two & (got == 2)
    bad_k = kept & ((np.abs(o[:, 11] - k11) > dk) | (np.abs(o[:, 12] - k12) > dk) | (np.abs(o[:, 13] - k22) > dk))
    bad += list(np.flatnonzero(bad_k | bad_n))
    bad += list(np.flatnonzero((pc_in == 1) & (got != 1)))
    return sorted(set(int(i) for i in bad))


def velocity_records(init_rec, init_out, seed=22):
    """PROBE_CONTACT_VELOCITY records on the normals and rB of contact-init outputs: body velocities of a few m/s and
    rad/s, accumulated impulses 0 .. 0.5 N s (the points' differ, so that a friction clamp on the wrong point shows),
    tangent impulses up to twice the friction cone, the fixtures' and the terrain's friction mixed."""
    rng = np.random.default_rng(seed)
    n = len(init_rec)
    r = g.records(n)
    r[:, 0] = init_rec[:, 0]
    r[:, 1:3] = rng.normal(0, 1.5, (n, 2))
    r[:, 3] = rng.normal(0, 2.0, n)
    r[:, 4:6] = init_out[:, 0:2]
    r[:, 6:10] = init_out[:, 2:6]
    nI = rng.uniform(0, 0.5, (n, 2)) * (rng.random((n, 2)) < 0.8)
    mu = np.sqrt(rng.choice([0.1, 0.2, 2.5], n) * rng.choice([0.1, 0.2], n))
    r[:, 10:12] = nI
    r[:, 12:14] = rng.uniform(-2, 2, (n, 2)) * mu[:, None] * nI
    r[:, 14] = mu
    r[:, 15] = init_out[:, 10]
    return r


def block_records(fc, seed=23, per=600):
    """Hand-made 2-point records on each fixture's bottom face (the normal up, both points below the centre of mass,
    as a body resting on flat ground): velocities and spins chosen so that both points approach, only one does, or
    both leave, and accumulated impulses that are too large, so that every case of the block LCP is taken."""
    from hostsim import sim
    rng = np.random.default_rng(seed)
    recs = []
    for f in range(5):
        verts, lc = sim.shape_verts(f)
        v = verts.astype(np.float64) - lc
        low = v[np.argsort(v[:, 1])[:2]]
        for i in range(per):
            a = rng.uniform(-0.3, 0.3)
            s, c = np.sin(a), np.cos(a)
            r1, r2 = rmul(s, c, low[0]), rmul(s, c, low[1])
            kind = i % 4
            vy = {0: -rng.uniform(0.1, 2), 1: rng.uniform(-1, 1), 2: rng.uniform(-1, 1), 3: rng.uniform(0.1, 2)}[kind]
            w = {0: rng.normal(0, 0.3), 1: rng.uniform(2, 8), 2: -rng.uniform(2, 8), 3: rng.normal(0, 0.3)}[kind]
            r = np.zeros(16, dtype=np.float32)
            r[0] = f
            r[1:3] = (rng.normal(0, 0.5), vy)
            r[3] = w
            r[4:6] = (0.0, 1.0)
            r[6:8], r[8:10] = r1, r2
            r[10:12] = rng.uniform(0, 1.0, 2) * (rng.random() < 0.7)
            r[12:14] = rng.uniform(-0.05, 0.05, 2)
            r[14] = np.sqrt(np.float32(0.2) * np.float32(2.5))
            r[15] = 2
            recs.append(r)
    return np.stack(recs)


def _velocity_terms(rec, out, fc):
    r, o = rec.astype(np.float64), out.astype(np.float64)
    f = r[:, 0].astype(int)
    n = r[:, 4:6]
    t = tangent_of(n)
    rBs = [r[:, 6:8], r[:, 8:10]]
    mB, iB, rn, rt, kn, kt, k12 = masses(fc, f, n, rBs)
    return r, o, f, n, t, rBs, mB, iB, rn, rt, kn, kt, k12


def check_contact_velocity(rec, out, fc):
    """Indices of PROBE_CONTACT_VELOCITY outputs (masses plus one iteration) that break, with V the velocity scale
    (|v| + |w| |rB| in and out, plus the impulses' velocity changes) and eps = 32 u V:
      * impulse balance: v_out - v_in = mB sum(dP), w_out - w_in = iB sum(rB x dP), dP the points' impulse changes
        along the normal and the tangent;
      * friction: |tI| <= mu nI_in exactly (the float32 product the clamp uses), and for an unclamped point the
        tangential velocity right after its own friction impulse (recovered from the outputs) is within eps of 0;
      * 1 point: nI >= 0; nI > 0 gives vn within eps of 0, nI = 0 gives vn >= -eps;
      * 2 points: x >= 0, vn >= -eps * cond(K), x . vn within eps |x| cond(K); the case is the first of Box2D's four
        whose conditions hold in float64 on the velocity after friction, a record within eps cond(K) of a boundary
        may take either; no case leaves the impulses unchanged;
      * the 2-point / 1-point decision follows k11^2 < 1000 det(K) outside its rounding band."""
    r, o, f, n, t, rBs, mB, iB, rn, rt, kn, kt, k12 = _velocity_terms(rec, out, fc)
    bad = set()
    v0, w0, v1, w1 = r[:, 1:3], r[:, 3], o[:, 0:2], o[:, 2]
    nI0, tI0, nI1, tI1 = r[:, 10:12], r[:, 12:14], o[:, 3:5], o[:, 5:7]
    pc_in, kase, pc = r[:, 15].astype(int), o[:, 7].astype(int), o[:, 8].astype(int)
    rmax = np.maximum(norm(rBs[0]), norm(rBs[1]))
    live = [pc >= 1, pc >= 2]
    dn = [np.where(live[p], nI1[:, p] - nI0[:, p], 0.0) for p in range(2)]
    dt_ = [np.where(live[p], tI1[:, p] - tI0[:, p], 0.0) for p in range(2)]
    dP = [dn[p][:, None] * n + dt_[p][:, None] * t for p in range(2)]
    V = norm(v0) + np.abs(w0) * rmax + norm(v1) + np.abs(w1) * rmax + \
        sum((mB + iB * rmax * rmax) * (np.abs(dn[p]) + np.abs(dt_[p]) + np.abs(nI0[:, p]) + np.abs(tI0[:, p]))
            for p in range(2))
    eps = 32 * U * V
    # impulse balance
    dv = v1 - v0 - mB[:, None] * (dP[0] + dP[1])
    dw = w1 - w0 - iB * (cross(rBs[0], dP[0]) + cross(rBs[1], dP[1]))
    bad |= set(np.flatnonzero((norm(dv) > eps) | (np.abs(dw) * rmax > eps)))
    # untouched second point of a 1-point constraint (or a dropped one)
    bad |= set(np.flatnonzero((pc == 1) & ((nI1[:, 1] != nI0[:, 1]) | (tI1[:, 1] != tI0[:, 1]))))
    # friction cone, exactly, on the impulses the iteration started from
    cone = [(rec[:, 14] * rec[:, 10 + p]).astype(np.float64) for p in range(2)]
    for p in range(2):
        bad |= set(np.flatnonzero(live[p] & ~(np.abs(tI1[:, p]) <= cone[p])))
    # the velocity after the friction impulses: the outputs less the normal impulses
    vf = v1 - mB[:, None] * (dn[0][:, None] + dn[1][:, None]) * n
    wf = w1 - iB * (cross(rBs[0], dn[0][:, None] * n) + cross(rBs[1], dn[1][:, None] * n))
    for p in range(2):
        # the velocity right after point p's friction impulse: for the first of two, also less the second's
        vp = vf - np.where(((p == 0) & (pc == 2))[:, None], mB[:, None] * dt_[1][:, None] * t, 0.0)
        wp = wf - np.where((p == 0) & (pc == 2), iB * cross(rBs[1], dt_[1][:, None] * t), 0.0)
        vt = np.sum((vp + cross_sv(wp, rBs[p])) * t, axis=1)
        free = live[p] & (np.abs(tI1[:, p]) < cone[p] * (1 - 8 * U))
        bad |= set(np.flatnonzero(free & (np.abs(vt) > eps)))
    # normal
    vn = [np.sum((v1 + cross_sv(w1, rBs[p])) * n, axis=1) for p in range(2)]
    one = pc == 1
    bad |= set(np.flatnonzero(one & (kase != ONE_POINT)))
    bad |= set(np.flatnonzero(one & ((nI1[:, 0] < 0) | ((nI1[:, 0] > 0) & (np.abs(vn[0]) > eps)) | (vn[0] < -eps))))
    two = pc == 2
    k11, k22 = kn[0], kn[1]
    det = k11 * k22 - k12 * k12
    # the condition number of the symmetric positive definite K: the ratio of its eigenvalues
    root = np.sqrt((k11 - k22) ** 2 + 4 * k12 ** 2)
    cond = np.where(two, (k11 + k22 + root) / np.maximum(k11 + k22 - root, 1e-300), 1.0)
    e2 = eps * cond
    solved = two & (kase >= 1)
    bad |= set(np.flatnonzero(solved & ((nI1[:, 0] < 0) | (nI1[:, 1] < 0) | (vn[0] < -e2) | (vn[1] < -e2) |
                                        (np.abs(nI1[:, 0] * vn[0]) + np.abs(nI1[:, 1] * vn[1]) >
                                         e2 * (np.abs(nI1[:, 0]) + np.abs(nI1[:, 1]) + 1e-30)))))
    bad |= set(np.flatnonzero(two & (kase == CASE_NONE) & ((nI1[:, 0] != nI0[:, 0]) | (nI1[:, 1] != nI0[:, 1]))))
    bad |= set(np.flatnonzero(two & ~np.isin(kase, [0, 1, 2, 3, 4])))
    # which case: Box2D's four in order on b = vn(after friction) - K a
    b1 = np.sum((vf + cross_sv(wf, rBs[0])) * n, axis=1) - (k11 * nI0[:, 0] + k12 * nI0[:, 1])
    b2 = np.sum((vf + cross_sv(wf, rBs[1])) * n, axis=1) - (k12 * nI0[:, 0] + k22 * nI0[:, 1])
    with np.errstate(divide="ignore", invalid="ignore"):
        kmax = np.maximum(k11, k22)
        quant = [
            [-(k22 * b1 - k12 * b2) / kmax, -(k11 * b2 - k12 * b1) / kmax],             # case 1: x = -K^-1 b >= 0
            [-b1, k12 * (-b1 / k11) + b2],                                              # case 2: x1 >= 0, vn2 >= 0
            [-b2, k12 * (-b2 / k22) + b1],                                              # case 3: x2 >= 0, vn1 >= 0
            [b1, b2],                                                                   # case 4: b >= 0
        ]
    for i in np.flatnonzero(two):
        allowed = set()
        for c, qs in enumerate(quant, start=1):
            vals = [q[i] for q in qs]
            if all(v > e2[i] for v in vals):
                allowed.add(c)
                break
            if any(v < -e2[i] for v in vals):
                continue
            allowed.add(c)
        else:
            allowed.add(CASE_NONE)
        if int(kase[i]) not in allowed:
            bad.add(int(i))
    # the condition-number fallback
    tol_k = 8 * U * (k11 + k22 + np.abs(k12))
    margin = k11 * k11 - 1000 * det
    dmargin = 2 * k11 * tol_k + 1000 * (2 * (k11 + k22 + np.abs(k12)) * tol_k)
    bad |= set(np.flatnonzero((pc_in == 2) & (((margin < -dmargin) & (pc != 2)) | ((margin > dmargin) & (pc != 1)))))
    return sorted(int(i) for i in bad)


def check_contact_position(rec, out, fc):
    """Indices of 1-point PROBE_CONTACT_POSITION outputs that break, with s the float64 separation at the input
    state and C = clamp(0.2 (s + linearSlop), -maxLinearCorrection, 0) the Baumgarte correction:
      * minSeparation = s within 32 u L;
      * the body moves along the normal only: c_out - c_in = mB P n, a_out - a_in = iB (rB x n) P;
      * the impulse solves K P = -C, K = mB + iB (rB x n)^2, within 32 u L (1 + K |P| + iB (1 + |rB x n|) |P|): the
        separation's error carried into C, and that of rB carried into K.
    2-point records are checked by check_contact_position_two."""
    bad = set()
    r, o = rec.astype(np.float64), out.astype(np.float64)
    f = r[:, 0].astype(int)
    normal, pts, seps, _ = contact_geometry(rec, fc)
    s = seps[0]
    L = 1.0 + np.max(np.abs(r[:, 1:13]), axis=1)
    tol = 32 * U * L
    bad |= set(np.flatnonzero(np.abs(o[:, 3] - s) > tol))
    C = np.clip(BAUMGARTE * (s + LINEAR_SLOP), -MAX_LINEAR_CORRECTION, 0.0)
    rB = pts[0] - r[:, 1:3]
    mB = np.array([fc[k]["invMass"] for k in f])
    iB = np.array([fc[k]["invI"] for k in f])
    rn = cross(rB, normal)
    K = mB + iB * rn * rn
    dc = o[:, 0:2] - r[:, 1:3]
    P = np.sum(dc * normal, axis=1) / mB
    bad |= set(np.flatnonzero(norm(dc - mB[:, None] * P[:, None] * normal) > tol))
    bad |= set(np.flatnonzero(np.abs((o[:, 2] - r[:, 3]) - iB * rn * P) > tol * (1 + iB * np.abs(rn) * (1 + np.abs(P)))))
    bad |= set(np.flatnonzero(np.abs(K * P + C) > tol * (1 + K * np.abs(P) + iB * (1 + np.abs(rn)) * np.abs(P))))
    return sorted(int(i) for i in bad)


def position_records(contacts):
    """One 1-point PROBE_CONTACT_POSITION record per manifold point of the contact records, and the first points of
    the ground-face ones again with the body sunk 1.5 m into the ground (past the maxLinearCorrection clamp)."""
    first = contacts.copy()
    first[:, 13] = 1
    second = contacts[contacts[:, 13] == 2].copy()
    second[:, 9:11] = second[:, 11:13]
    second[:, 13] = 1
    deep = first[first[:, 4] == 0].copy()
    deep[:, 1:3] -= np.float32(1.5) * deep[:, 5:7]
    return np.concatenate([first, second, deep])


def two_point_position_records(contacts):
    """The 2-point contact records as they are, and again with the body sunk 0.3 m into the ground along the ground
    face's normal (so that the first point's correction moves the pose the second point is measured at)."""
    two = contacts[contacts[:, 13] == 2].copy()
    deep = two[two[:, 4] == 0].copy()
    deep[:, 1:3] -= np.float32(0.3) * deep[:, 5:7]
    return np.concatenate([two, deep])


def position_chain_reference(rec, fc):
    """float64 contact position iteration over both points of 2-point records, point by point: each point's
    separation s at the pose the previous point left, C = clamp(0.2 (s + linearSlop), -maxLinearCorrection, 0), the
    impulse P = -C / K along the normal moving the centre by mB P n and the angle by iB (rB x n) P.  Returns the final
    centre, angle, the smallest separation and the two impulses."""
    r = rec.astype(np.float64)
    f = r[:, 0].astype(int)
    mB = np.array([fc[k]["invMass"] for k in f])
    iB = np.array([fc[k]["invI"] for k in f])
    cur = r.copy()
    seps, imps = [], []
    for p in range(2):
        one = cur.copy()
        one[:, 9:11] = r[:, 9 + 2 * p:11 + 2 * p]
        normal, pts, sep, _ = contact_geometry(one, fc)
        s = sep[0]
        rB = pts[0] - cur[:, 1:3]
        rn = cross(rB, normal)
        K = mB + iB * rn * rn
        P = -np.clip(BAUMGARTE * (s + LINEAR_SLOP), -MAX_LINEAR_CORRECTION, 0.0) / K
        cur[:, 1:3] += (mB * P)[:, None] * normal
        cur[:, 3] += iB * rn * P
        seps.append(s)
        imps.append(P)
    return cur[:, 1:3], cur[:, 3], np.minimum(seps[0], seps[1]), imps


def check_contact_position_two(rec, out, fc):
    """Indices of 2-point PROBE_CONTACT_POSITION outputs off position_chain_reference: the second point is solved at
    the pose the first leaves, and the separation reported is the smaller of the two.  Bound: 64 u L (1 + D), on the
    centre, the angle times the lever arm and the separation, with D = (mB + iB l^2)(|P1| + |P2|) the distance the two
    corrections move a point at lever arm l: each step's pose and separation carry the 32 u L of the 1-point check,
    the first step's error reaches the second point's separation with slope 1, and an impulse's relative error moves
    the pose by that fraction of D."""
    r, o = rec.astype(np.float64), out.astype(np.float64)
    f = r[:, 0].astype(int)
    mB = np.array([fc[k]["invMass"] for k in f])
    iB = np.array([fc[k]["invI"] for k in f])
    c, a, sep, imps = position_chain_reference(rec, fc)
    lc = np.stack([fc[k]["lc"] for k in f])
    lever = np.maximum(norm(r[:, 9:11] - r[:, 1:3]), norm(r[:, 11:13] - r[:, 1:3])) + norm(lc)
    D = (mB + iB * lever * lever) * (np.abs(imps[0]) + np.abs(imps[1]))
    L = 1.0 + np.max(np.abs(r[:, 1:13]), axis=1)
    tol = 64 * U * L * (1 + D)
    bad = (norm(o[:, 0:2] - c) > tol) | (np.abs(o[:, 2] - a) * (1 + lever) > tol) | (np.abs(o[:, 3] - sep) > tol)
    return np.flatnonzero(bad)


# ---------------------------------------------------------------------------------------------------------------------
# joints
# ---------------------------------------------------------------------------------------------------------------------
def joint_velocity_records(fc, seed=24, per=1500):
    """PROBE_JOINT_VELOCITY records for all six joints: joint angles spread over both sides of the limits, exactly at
    each limit (aA = 0, so the float32 angle is the limit), and a few ulp on either side; motor torques 0, random and
    the task maximum (40 / 80); every previous limit state; accumulated impulses of both signs, scaled by the bodies'
    masses so that warm starting changes the velocities by a few m/s and rad/s, as body velocities are."""
    rng = np.random.default_rng(seed)
    recs = []
    for j, (_, _, lo, hi, fA, fB, tmax) in JOINT_DEFS.items():
        lo32, hi32 = np.float32(lo), np.float32(hi)
        lin = 1 / (fc[fA]["invMass"] + fc[fB]["invMass"])
        ang = 1 / (fc[fA]["invI"] + fc[fB]["invI"])
        for i in range(per):
            kind = i % 6
            if kind <= 1:
                aA = np.float32(rng.uniform(-1, 1))
                aB = np.float32(aA + rng.uniform(lo - 0.3, hi + 0.3))
            elif kind <= 3:
                aA = np.float32(0.0)
                lim = lo32 if kind == 2 else hi32
                aB = lim
                k = int(rng.integers(-3, 4)) if i % 12 >= 6 else 0
                for _ in range(abs(k)):
                    aB = np.nextafter(aB, np.float32(np.inf if k > 0 else -np.inf))
            else:
                aA = np.float32(rng.uniform(-1, 1))
                aB = np.float32(aA + (lo if kind == 4 else hi) + rng.uniform(-0.02, 0.02))
            T = [0.0, tmax, rng.uniform(0, tmax)][i % 3]
            speed = rng.choice([-1, 1]) * (0.3 if j < 2 else (4.0 if j % 2 == 0 else 6.0)) * rng.uniform(0, 1)
            r = np.zeros(16, dtype=np.float32)
            r[0] = j
            r[1:3] = rng.normal(0, 1.5, 2)
            r[3] = rng.normal(0, 2)
            r[4] = aA
            r[5:7] = rng.normal(0, 1.5, 2)
            r[7] = rng.normal(0, 3)
            r[8] = aB
            r[9:11] = rng.normal(0, 2 * lin, 2)
            r[11] = rng.normal(0, 3 * ang)
            r[12] = rng.uniform(-1, 1) * T * DT
            r[13] = speed
            r[14] = T
            r[15] = rng.integers(0, 3)
            recs.append(r)
    return np.stack(recs)


def joint_terms(rec, fc, jc):
    """Per record: the bodies' inverse masses and inertias, the anchors relative to the centres of mass in the bodies'
    frames, and the limits."""
    r = rec.astype(np.float64)
    j = r[:, 0].astype(int)
    fA = np.array([jc[k]["fA"] for k in j])
    fB = np.array([jc[k]["fB"] for k in j])
    mA = np.array([fc[k]["invMass"] for k in fA]); iA = np.array([fc[k]["invI"] for k in fA])
    mB = np.array([fc[k]["invMass"] for k in fB]); iB = np.array([fc[k]["invI"] for k in fB])
    lA = np.stack([jc[k]["anchorA"] - fc[jc[k]["fA"]]["lc"] for k in j])
    lB = np.stack([jc[k]["anchorB"] - fc[jc[k]["fB"]]["lc"] for k in j])
    lower = np.array([jc[k]["lower"] for k in j]); upper = np.array([jc[k]["upper"] for k in j])
    return mA, iA, mB, iB, lA, lB, lower, upper


def point_K(mA, iA, mB, iB, rA, rB):
    K = np.zeros((len(mA), 3, 3))
    K[:, 0, 0] = mA + mB + rA[:, 1] ** 2 * iA + rB[:, 1] ** 2 * iB
    K[:, 0, 1] = K[:, 1, 0] = -rA[:, 1] * rA[:, 0] * iA - rB[:, 1] * rB[:, 0] * iB
    K[:, 0, 2] = K[:, 2, 0] = -rA[:, 1] * iA - rB[:, 1] * iB
    K[:, 1, 1] = mA + mB + rA[:, 0] ** 2 * iA + rB[:, 0] ** 2 * iB
    K[:, 1, 2] = K[:, 2, 1] = rA[:, 0] * iA + rB[:, 0] * iB
    K[:, 2, 2] = iA + iB
    return K


def limit_state(d, lower, upper):
    """(wanted state, undecided): the float64 joint angle against the limits; an angle within half an ulp of a limit
    (but not on it) may round onto it."""
    want = np.where(d <= lower, 1, np.where(d >= upper, 2, 0))
    h = 0.5 * g.ulp32(d)
    near = ((np.abs(d - lower) <= h) & (d != lower)) | ((np.abs(d - upper) <= h) & (d != upper))
    return want, near


def check_joint_velocity(rec, out, fc, jc):
    """Indices of PROBE_JOINT_VELOCITY outputs (joint_init with dtRatio 1, then one iteration) that break, with V the
    velocity scale (|v| + |w| |r| of both bodies in and out, |motorSpeed|, the velocity changes of the impulses) and
    eps = 32 u V:
      * the limit state follows the float64 angle aB - aA against the limits, and the warm start keeps the limit
        impulse only where the state stays at the same limit: the limit impulse joint_init applies is 0 with no limit
        or on a change of state, and the given imp[2] (dtRatio 1) otherwise;
      * impulse balance over the warm start and the iteration: with dtRatio 1 the impulses applied in all are the
        output accumulators, so vA_out - vA_in = -mA P, wA_out - wA_in = -iA (rA x P + motorImpulse + imp[2]), and
        the same with + for B, P = imp[0..1] (angular changes compared at the lever arm's scale, times 1 + |rA| + |rB|);
      * motor: |motorImpulse| <= h maxMotorTorque exactly; an unsaturated motor leaves wB - wA - motorSpeed within eps
        of 0 after the motor step;
      * the accumulated limit impulse is 0 with no limit, >= 0 at the lower limit and <= 0 at the upper one;
      * the point constraint's Cdot = vB + wB x rB - vA - wA x rA is within eps cond(K) of 0; with a limit impulse
        left on, the angular Cdot = wB - wA is too; a limit impulse brought to 0 (the reduced re-solve) leaves the
        bodies separating: wB - wA >= -eps cond(K) at the lower limit, <= at the upper."""
    bad = set()
    r, o = rec.astype(np.float64), out.astype(np.float64)
    mA, iA, mB, iB, lA, lB, lower, upper = joint_terms(rec, fc, jc)
    aA, aB = r[:, 4], r[:, 8]
    rA = rmul(*rot(aA), lA)
    rB = rmul(*rot(aB), lB)
    want, near = limit_state(aB - aA, lower, upper)
    st = o[:, 10].astype(int)
    bad |= set(np.flatnonzero(~near & (st != want)))
    bad |= set(np.flatnonzero(near & ~np.isin(st, (0, 1, 2))))
    vA, wA, vB, wB = o[:, 0:2], o[:, 2], o[:, 3:5], o[:, 5]
    ra, rb = norm(rA), norm(rB)
    mi0, mi1 = r[:, 12], o[:, 9]
    K = point_K(mA, iA, mB, iB, rA, rB)
    P0, P1 = np.abs(r[:, 9:12]).sum(axis=1) + np.abs(mi0), np.abs(o[:, 6:9]).sum(axis=1) + np.abs(mi1)
    V = (norm(r[:, 1:3]) + np.abs(r[:, 3]) * ra + norm(r[:, 5:7]) + np.abs(r[:, 7]) * rb + norm(vA) + np.abs(wA) * ra
         + norm(vB) + np.abs(wB) * rb + np.abs(r[:, 13]) + (mA + mB + (iA + iB) * (1 + ra + rb) ** 2) * (P0 + P1))
    eps = 32 * U * V
    # warm start: the limit impulse kept, and the balance of everything applied
    prev, warm2 = r[:, 15].astype(int), o[:, 13]
    keep = (st != 0) & (st == prev)
    bad |= set(np.flatnonzero(np.where(keep, warm2 != r[:, 11], warm2 != 0)))
    P = o[:, 6:8]
    ang = cross(rA, P) + o[:, 9] + o[:, 8], cross(rB, P) + o[:, 9] + o[:, 8]
    lever = 1 + ra + rb
    bad |= set(np.flatnonzero((norm(vA - r[:, 1:3] + mA[:, None] * P) > eps) |
                              (norm(vB - r[:, 5:7] - mB[:, None] * P) > eps) |
                              (np.abs(wA - r[:, 3] + iA * ang[0]) * lever > eps) |
                              (np.abs(wB - r[:, 7] - iB * ang[1]) * lever > eps)))
    # motor
    maxI = (np.float32(DT) * rec[:, 14]).astype(np.float64)
    bad |= set(np.flatnonzero(~(np.abs(mi1) <= maxI)))
    free = np.abs(mi1) < maxI * (1 - 8 * U)
    bad |= set(np.flatnonzero(free & (np.abs(o[:, 12] - o[:, 11] - r[:, 13]) > eps)))
    # limit impulse signs
    imp2 = o[:, 8]
    bad |= set(np.flatnonzero(((st == 0) & (imp2 != 0)) | ((st == 1) & (imp2 < 0)) | ((st == 2) & (imp2 > 0))))
    # residuals
    cdot1 = vB + cross_sv(wB, rB) - vA - cross_sv(wA, rA)
    cdot2 = wB - wA
    cond3 = np.linalg.cond(K)
    cond2 = np.linalg.cond(K[:, :2, :2])
    cond = np.where(st == 0, cond2, cond3)
    e = eps * cond
    bad |= set(np.flatnonzero(norm(cdot1) > e))
    bad |= set(np.flatnonzero((st != 0) & (imp2 != 0) & (np.abs(cdot2) * (1 + ra + rb) > e)))
    bad |= set(np.flatnonzero((st == 1) & (imp2 == 0) & (cdot2 * (1 + ra + rb) < -e)))
    bad |= set(np.flatnonzero((st == 2) & (imp2 == 0) & (cdot2 * (1 + ra + rb) > e)))
    return sorted(int(i) for i in bad)


def joint_position_records(fc, jc, seed=25, per=1500):
    """PROBE_JOINT_POSITION records for all six joints: the anchors apart by up to 2 cm (and exactly together), joint
    angles over both sides of the limits and at them, the limit state the velocity phase would have chosen, or none."""
    rng = np.random.default_rng(seed)
    recs = []
    for j in range(6):
        d = jc[j]
        for i in range(per):
            aA = np.float32(rng.uniform(-1, 1)) if i % 4 else np.float32(0.0)
            kind = i % 3
            lim = d["lower"] if rng.random() < 0.5 else d["upper"]
            ang = rng.uniform(d["lower"] - 0.3, d["upper"] + 0.3) if kind == 0 else lim + rng.uniform(-0.05, 0.05)
            aB = np.float32(aA + ang) if i % 4 else np.float32(lim if kind == 2 else ang)
            cA = rng.uniform(-5, 5, 2)
            rA = rmul(*rot(aA), d["anchorA"] - fc[d["fA"]]["lc"])
            rB = rmul(*rot(aB), d["anchorB"] - fc[d["fB"]]["lc"])
            gap = rng.normal(0, 0.01, 2) * (i % 5 != 0) * (i % 7 != 0 or 0.2)
            cB = cA + rA - rB + gap
            dd = float(aB) - float(aA)
            state = 1 if dd <= d["lower"] else (2 if dd >= d["upper"] else 0)
            if rng.random() < 0.2:
                state = 0
            r = np.zeros(16, dtype=np.float32)
            r[0] = j
            r[1:3] = cA
            r[3] = aA
            r[4:6] = cB
            r[6] = aB
            r[7] = state
            recs.append(r)
    return np.stack(recs)


def check_joint_position(rec, out, fc, jc):
    """Indices of PROBE_JOINT_POSITION outputs that break, in float64 on the float32 inputs:
      * the limit correction: with C the angle's distance past the limit less angularSlop, clamped to
        maxAngularCorrection, the bodies turn by -iA C / (iA + iB) and iB C / (iA + iB) (beyond what the point
        correction turns them);
      * the point correction: at the turned angles, the impulse P with cB_out - cB_in = mB P, cA_out - cA_in = -mA P
        solves K P = -C for the anchors' separation C, within 32 u L cond(K) (L: coordinates and |K| |P|);
      * ok is (|C| <= linearSlop and the angular error <= angularSlop), outside the rounding band of both tests."""
    bad = set()
    r, o = rec.astype(np.float64), out.astype(np.float64)
    mA, iA, mB, iB, lA, lB, lower, upper = joint_terms(rec, fc, jc)
    cA, aA, cB, aB, st = r[:, 1:3], r[:, 3], r[:, 4:6], r[:, 6], r[:, 7].astype(int)
    ang = aB - aA
    C_lim = np.where(st == 1, np.clip(ang - lower + ANGULAR_SLOP, -MAX_ANGULAR_CORRECTION, 0.0),
                     np.where(st == 2, np.clip(ang - upper - ANGULAR_SLOP, 0.0, MAX_ANGULAR_CORRECTION), 0.0))
    ang_err = np.where(st == 1, lower - ang, np.where(st == 2, ang - upper, 0.0))
    limp = -C_lim / (iA + iB)
    aA1, aB1 = aA - iA * limp, aB + iB * limp
    rA = rmul(*rot(aA1), lA)
    rB = rmul(*rot(aB1), lB)
    C = cB + rB - cA - rA
    perr = norm(C)
    K = point_K(mA, iA, mB, iB, rA, rB)[:, :2, :2]
    P = (o[:, 3:5] - cB) / mB[:, None]
    L = 1.0 + np.max(np.abs(r[:, 1:7]), axis=1)
    cond = np.linalg.cond(K)
    KP = np.einsum("nij,nj->ni", K, P)
    tolP = 32 * U * (L + np.max(np.abs(K), axis=(1, 2)) * norm(P)) * cond
    bad |= set(np.flatnonzero(norm(KP + C) > tolP))
    bad |= set(np.flatnonzero(norm((o[:, 0:2] - cA) + mA[:, None] * P) > 32 * U * L))
    # the angular change less the point correction's is the limit correction
    turnA = o[:, 2] - aA + iA * cross(rA, P)
    turnB = o[:, 5] - aB - iB * cross(rB, P)
    tolA = 32 * U * (L + (iA + iB) * (1 + norm(rA) + norm(rB)) * norm(P) + np.abs(C_lim))
    bad |= set(np.flatnonzero((np.abs(turnA + iA * limp) > tolA) | (np.abs(turnB - iB * limp) > tolA)))
    # the relative turn of the limit correction is the clamped C, never more than maxAngularCorrection
    bad |= set(np.flatnonzero(np.abs((turnB - turnA) + C_lim) > 2 * tolA))
    # ok
    tol_p = 32 * U * L
    tol_a = 32 * U * (1 + np.abs(aA) + np.abs(aB))
    want = (perr <= LINEAR_SLOP) & (ang_err <= ANGULAR_SLOP)
    sure = (np.abs(perr - LINEAR_SLOP) > tol_p) & (np.abs(ang_err - ANGULAR_SLOP) > tol_a)
    bad |= set(np.flatnonzero(sure & ((o[:, 6] == 1) != want)))
    return sorted(int(i) for i in bad)


# ---------------------------------------------------------------------------------------------------------------------
# integration
# ---------------------------------------------------------------------------------------------------------------------
def integrate_records(seed=26, per=800):
    """PROBE_INTEGRATE records for every fixture: ordinary states, forces and gravities, and velocities whose step
    h |v| and h |w| sit a few ulp below, at and above maxTranslation and maxRotation, and well past them."""
    rng = np.random.default_rng(seed)
    recs = []
    for f in range(5):
        for i in range(per):
            r = np.zeros(16, dtype=np.float32)
            r[0] = f
            r[1:3] = rng.uniform(-50, 50, 2)
            r[3] = rng.uniform(-10, 10)
            kind = i % 4
            d = rng.normal(size=2)
            d /= np.linalg.norm(d)
            if kind == 0:
                v, w = rng.normal(0, 5, 2), rng.normal(0, 5)
            elif kind == 1:        # at the translation clamp
                v, w = d * MAX_TRANSLATION / DT * (1 + rng.integers(-4, 5) * U), rng.normal(0, 5)
            elif kind == 2:        # at the rotation clamp
                v, w = rng.normal(0, 5, 2), rng.choice([-1, 1]) * MAX_ROTATION / DT * (1 + rng.integers(-4, 5) * U)
            else:                  # far past both
                v, w = d * rng.uniform(100, 1000), rng.choice([-1, 1]) * rng.uniform(80, 800)
            r[4:6], r[6] = v, w
            r[7:9] = rng.normal(0, 50, 2) * (i % 3 != 0)
            r[9] = rng.normal(0, 20) * (i % 3 != 0)
            r[10] = rng.choice([-10.0, -9.8, 0.0, -1.5])
            recs.append(r)
    return np.stack(recs)


def integrate_reference(rec, fc):
    r = rec.astype(np.float64)
    f = r[:, 0].astype(int)
    m = np.array([fc[k]["invMass"] for k in f])
    I = np.array([fc[k]["invI"] for k in f])
    v = r[:, 4:6] + DT * (np.stack([np.zeros(len(r)), r[:, 10]], axis=1) + m[:, None] * r[:, 7:9])
    w = r[:, 6] + DT * I * r[:, 9]
    tr = DT * norm(v)
    v = np.where((tr > MAX_TRANSLATION)[:, None], v * (MAX_TRANSLATION / np.maximum(tr, 1e-300))[:, None], v)
    rt = DT * np.abs(w)
    w = np.where(rt > MAX_ROTATION, w * MAX_ROTATION / np.maximum(rt, 1e-300), w)
    return r[:, 1:3] + DT * v, r[:, 3] + DT * w, v, w


def check_integrate(rec, out, fc):
    """Indices of PROBE_INTEGRATE outputs off the float64 step by more than 32 u of the magnitudes involved (each
    output passes through <= 10 roundings: the velocity update, the clamp ratio's square, root and division, the
    position update); the clamps act at the float64 thresholds, and a velocity within rounding of one is scaled by a
    ratio within that rounding of 1, so the bound holds on both sides without a band."""
    o = out.astype(np.float64)
    r = rec.astype(np.float64)
    f = r[:, 0].astype(int)
    m = np.array([fc[k]["invMass"] for k in f])
    I = np.array([fc[k]["invI"] for k in f])
    c, a, v, w = integrate_reference(rec, fc)
    Sv = norm(r[:, 4:6]) + DT * (np.abs(r[:, 10]) + m * norm(r[:, 7:9]))
    Sw = np.abs(r[:, 6]) + DT * I * np.abs(r[:, 9])
    bad = (norm(o[:, 3:5] - v) > 32 * U * Sv) | (np.abs(o[:, 5] - w) > 32 * U * Sw)
    bad |= norm(o[:, 0:2] - c) > 32 * U * (norm(r[:, 1:3]) + DT * Sv)
    bad |= np.abs(o[:, 2] - a) > 32 * U * (np.abs(r[:, 3]) + DT * Sw)
    return np.flatnonzero(bad)
