// b2probe.cuh -- one case of a Box2D building block on packed float32 records: the dispatch behind
// b200gym_selftest_box2d (b2probe.cu) and its host build (tests/hostsim), so that the CPU suite and the device run the
// same code on the same records.  The tests compare both with float64 geometry (tests/box2d_geometry.py) and with
// float64 restatements of the solver steps' contracts (tests/box2d_solvers.py).
//
// Records are kProbeWords float32 words in and out.  Integer results (manifold type, point count, ray hit, TOI state,
// simplex count) are stored as float values; feature ids as their bit pattern.  Fixture f: 0 lander hull, 1 lander leg,
// 2 walker hull, 3 walker upper leg, 4 walker lower leg -- the ShapeConsts of box2d_consts.h, which the caller loads
// into lunar::kC / walker::kC as b200gym_create does.  An out-of-range fixture, joint or contact point count gives a
// record of NaNs.
#pragma once
#include "lunar.cuh"
#include "walker.cuh"

namespace b2probe {

using namespace b2l;

constexpr int kProbeWords = 16;
enum {
    PROBE_ROT = 0,          // in {x}                                     out {s, c}
    PROBE_EDGE_POLYGON,     // in {f, v1, v2, p, q.s, q.c}                out manifold (below)
    PROBE_BOX_POLYGON,      // in {f, x0, ylo, x1, yhi, p, q.s, q.c}      out manifold
    PROBE_EDGE_RAYCAST,     // in {v1, v2, p1, p2, maxFraction}           out {hit, t}
    PROBE_BOX_RAYCAST,      // in {x0, ylo, x1, yhi, p1, p2, maxFraction} out {hit, t}
    PROBE_GJK,              // in {f, v1, v2, c, a}                       out {distance, simplex count}
    PROBE_TOI,              // in {f, v1, v2, c0, a0, c1, a1}             out {state, t}
    PROBE_SOLVE22,          // in {K[0][0..2], K[1][0..2], K[2][0..2], b} out {x0, x1}
    PROBE_SOLVE33,          // same                                       out {x0, x1, x2}
    // the solver steps of world_step (below: c, v body centre of mass and velocity, a angle, w angular velocity)
    PROBE_CONTACT_INIT,     // in {f, c, a, type, localNormal, localPoint, lp1, lp2, pointCount}
                            // out {normal, rB1, rB2, normalMass1..2, tangentMass1..2, pointCount, k11, k12, k22}
    PROBE_CONTACT_VELOCITY, // in {f, v, w, normal, rB1, rB2, nI1..2, tI1..2, friction, pointCount}
                            // out {v, w, nI1..2, tI1..2, case, pointCount}: the masses, then one iteration
    PROBE_CONTACT_POSITION, // in as PROBE_CONTACT_INIT                   out {c, a, minSeparation}
    PROBE_JOINT_VELOCITY,   // in {j, vA, wA, aA, vB, wB, aB, imp[3], motorImpulse, motorSpeed, maxMotorTorque, limitState}
                            // out {vA, wA, vB, wB, imp[3], motorImpulse, limitState, wA, wB after the motor step,
                            //      imp[2] after joint_init (the limit impulse the warm start applied)}
    PROBE_JOINT_POSITION,   // in {j, cA, aA, cB, aB, limitState}        out {cA, aA, cB, aB, ok}
    PROBE_INTEGRATE,        // in {f, c, a, v, w, force, torque, gravity_y} out {c, a, v, w}
    PROBE_CONSTS,           // in {0, f}: out {invMass, invI, localCenter, friction, centroid, count}
                            // in {1, j}: out {anchorA, anchorB, lower, upper, fixture A, fixture B}
    PROBE_NUM_OPS
};
// manifold record: {type, pointCount, localNormal, localPoint, pts[0].localPoint, pts[0].id, pts[1].localPoint, pts[1].id}
// Joint j: 0, 1 the lander's legs, 2 / 4 the walker's hips, 3 / 5 its knees -- lunar::kC.jd[j] and walker::kC.jd[j - 2],
// between the fixtures of their bodies.  The solver-step ops run with world_step's dt = 1/50 and with dtRatio = 1 (its
// value on every step but an episode's first).  A contact record's body B is fixture f, body A the static ground; its
// pointCount is 1 or 2.  `case` is contact_solve_velocity's: 1..4 the block solver's case, 0 none, -1 one point.

__device__ __forceinline__ const ShapeConst *fixture(float f) {
    if (f == 0.0f) return &lunar::kC.shape[0];
    if (f == 1.0f) return &lunar::kC.shape[1];
    if (f == 2.0f) return &walker::kC.shape[0];
    if (f == 3.0f) return &walker::kC.shape[1];
    if (f == 4.0f) return &walker::kC.shape[2];
    return nullptr;
}

// The fixture index (as above) of body b of the lander or the walker scene
__device__ __forceinline__ int lunar_fixture(int b) { return b == 0 ? 0 : 1; }
__device__ __forceinline__ int walker_fixture(int b) { return b == 0 ? 2 : ((b & 1) ? 3 : 4); }

__device__ __forceinline__ const JointDef *joint(float j, int &fA, int &fB) {
    for (int k = 0; k < lunar::NJ; k++)
        if (j == (float)k) {
            fA = lunar_fixture(lunar::kC.jd[k].bodyA); fB = lunar_fixture(lunar::kC.jd[k].bodyB);
            return &lunar::kC.jd[k];
        }
    for (int k = 0; k < walker::NJ; k++)
        if (j == (float)(lunar::NJ + k)) {
            fA = walker_fixture(walker::kC.jd[k].bodyA); fB = walker_fixture(walker::kC.jd[k].bodyB);
            return &walker::kC.jd[k];
        }
    return nullptr;
}

// a contact constraint's manifold part from {type, localNormal, localPoint, lp1, lp2, pointCount}
__device__ __forceinline__ void contact_record(VC &k, const float *in) {
    k.mType = (int)in[0];
    k.localNormal = V(in[1], in[2]); k.localPoint = V(in[3], in[4]);
    k.lp[0] = V(in[5], in[6]); k.lp[1] = V(in[7], in[8]);
    k.pointCount = k.mPointCount = (int)in[9];
}

__device__ __forceinline__ xform pose(const float *p) {
    xform xf;
    xf.p = V(p[0], p[1]); xf.q.s = p[2]; xf.q.c = p[3];
    return xf;
}

// Edge v1-v2 as one GJK proxy, the vertices of fixture f as the other; the fixture's origin (not its centre of mass)
// sits at the given position, as in the CPU checker's distance and TOI probes
__device__ __forceinline__ void proxies(DProxy &pA, DProxy &pB, const float *in, const ShapeConst &sh) {
    pA.count = 2; pA.v[0] = V(in[1], in[2]); pA.v[1] = V(in[3], in[4]);
    pB.count = sh.count;
    for (int i = 0; i < sh.count; i++) pB.v[i] = sh.verts[i];
}

__device__ __forceinline__ void probe_case(int op, const float *in, float *out) {
    for (int k = 0; k < kProbeWords; k++) out[k] = 0.0f;
    const bool shaped = op == PROBE_EDGE_POLYGON || op == PROBE_BOX_POLYGON || op == PROBE_GJK || op == PROBE_TOI ||
                        op == PROBE_CONTACT_INIT || op == PROBE_CONTACT_VELOCITY || op == PROBE_CONTACT_POSITION ||
                        op == PROBE_INTEGRATE || (op == PROBE_CONSTS && in[0] == 0.0f);
    const bool jointed = op == PROBE_JOINT_VELOCITY || op == PROBE_JOINT_POSITION || (op == PROBE_CONSTS && in[0] == 1.0f);
    const ShapeConst *sh = shaped ? fixture(op == PROBE_CONSTS ? in[1] : in[0]) : nullptr;
    int fA = -1, fB = -1;
    const JointDef *jd = jointed ? joint(op == PROBE_CONSTS ? in[1] : in[0], fA, fB) : nullptr;
    const float pc = op == PROBE_CONTACT_VELOCITY ? in[15] : in[13];
    const bool contact = op == PROBE_CONTACT_INIT || op == PROBE_CONTACT_VELOCITY || op == PROBE_CONTACT_POSITION;
    if ((shaped && !sh) || (jointed && !jd) || (op == PROBE_CONSTS && !shaped && !jointed) ||
        (contact && pc != 1.0f && pc != 2.0f) || op < 0 || op >= PROBE_NUM_OPS) {
        for (int k = 0; k < kProbeWords; k++) out[k] = __uint_as_float(0x7fc00000u);
        return;
    }
    if (op == PROBE_ROT) {
        const rot q = rot_of(in[0]);
        out[0] = q.s; out[1] = q.c;
    } else if (op == PROBE_EDGE_POLYGON || op == PROBE_BOX_POLYGON) {
        Manifold m;
        m.type = 0; m.pointCount = 0;
        m.localNormal = V(0.0f, 0.0f); m.localPoint = V(0.0f, 0.0f);
        for (int p = 0; p < 2; p++) { m.pts[p].localPoint = V(0.0f, 0.0f); m.pts[p].nI = m.pts[p].tI = 0.0f; m.pts[p].id = 0u; }
        if (op == PROBE_EDGE_POLYGON) {
            collide_edge_polygon(m, V(in[1], in[2]), V(in[3], in[4]), *sh, pose(in + 5));
        } else {
            StaticBox sb;
            static_box(sb, in[1], in[2], in[3], in[4]);
            collide_polygons(m, sb, *sh, pose(in + 5));
        }
        out[0] = (float)m.type; out[1] = (float)m.pointCount;
        out[2] = m.localNormal.x; out[3] = m.localNormal.y; out[4] = m.localPoint.x; out[5] = m.localPoint.y;
        for (int p = 0; p < 2; p++) {
            out[6 + 3 * p] = m.pts[p].localPoint.x; out[7 + 3 * p] = m.pts[p].localPoint.y;
            out[8 + 3 * p] = __uint_as_float(m.pts[p].id);
        }
    } else if (op == PROBE_EDGE_RAYCAST || op == PROBE_BOX_RAYCAST) {
        float t = -1.0f;
        bool hit;
        if (op == PROBE_EDGE_RAYCAST) {
            hit = walker::edge_raycast(V(in[0], in[1]), V(in[2], in[3]), V(in[4], in[5]), V(in[6], in[7]), in[8], t);
        } else {
            StaticBox sb;
            static_box(sb, in[0], in[1], in[2], in[3]);
            hit = static_box_raycast(sb, V(in[4], in[5]), V(in[6], in[7]), in[8], t);
        }
        out[0] = hit ? 1.0f : 0.0f; out[1] = t;
    } else if (op == PROBE_GJK) {
        DProxy pA, pB;
        proxies(pA, pB, in, *sh);
        xform xfA, xfB;
        xfA.p = V(0.0f, 0.0f); xfA.q.s = 0.0f; xfA.q.c = 1.0f;
        xfB.q = rot_of(in[7]);
        xfB.p = V(in[5], in[6]);
        SCache cache;
        cache.count = 0;
        out[0] = gjk_distance(cache, pA, xfA, pB, xfB);
        out[1] = (float)cache.count;
    } else if (op == PROBE_TOI) {
        DProxy pA, pB;
        proxies(pA, pB, in, *sh);
        Sweep sA, sB;
        sA.localCenter = V(0.0f, 0.0f); sA.c0 = V(0.0f, 0.0f); sA.c = V(0.0f, 0.0f); sA.a0 = 0.0f; sA.a = 0.0f; sA.alpha0 = 0.0f;
        sB.localCenter = V(0.0f, 0.0f); sB.c0 = V(in[5], in[6]); sB.a0 = in[7]; sB.c = V(in[8], in[9]); sB.a = in[10];
        sB.alpha0 = 0.0f;
        float t = 0.0f;
        out[0] = (float)time_of_impact(t, pA, sA, pB, sB, 1.0f);
        out[1] = t;
    } else if (op == PROBE_CONTACT_INIT || op == PROBE_CONTACT_POSITION) {
        BState s;
        s.c = V(in[1], in[2]); s.a = in[3]; s.v = V(0.0f, 0.0f); s.w = 0.0f;
        VC k;
        contact_record(k, in + 4);
        if (op == PROBE_CONTACT_INIT) {
            k.normal = V(0.0f, 0.0f); k.k11 = k.k12 = k.k22 = 0.0f;
            for (int p = 0; p < 2; p++) { k.p[p].rB = V(0.0f, 0.0f); k.p[p].normalMass = k.p[p].tangentMass = 0.0f; }
            contact_init(k, *sh, s);
            out[0] = k.normal.x; out[1] = k.normal.y;
            out[2] = k.p[0].rB.x; out[3] = k.p[0].rB.y; out[4] = k.p[1].rB.x; out[5] = k.p[1].rB.y;
            out[6] = k.p[0].normalMass; out[7] = k.p[1].normalMass; out[8] = k.p[0].tangentMass; out[9] = k.p[1].tangentMass;
            out[10] = (float)k.pointCount; out[11] = k.k11; out[12] = k.k12; out[13] = k.k22;
        } else {
            float minSep = kFltMax;
            contact_solve_position(k, *sh, s, minSep);
            out[0] = s.c.x; out[1] = s.c.y; out[2] = s.a; out[3] = minSep;
        }
    } else if (op == PROBE_CONTACT_VELOCITY) {
        BState s;
        s.c = V(0.0f, 0.0f); s.a = 0.0f; s.v = V(in[1], in[2]); s.w = in[3];
        VC k;
        k.normal = V(in[4], in[5]);
        k.p[0].rB = V(in[6], in[7]); k.p[1].rB = V(in[8], in[9]);
        k.p[0].nI = in[10]; k.p[1].nI = in[11]; k.p[0].tI = in[12]; k.p[1].tI = in[13];
        k.friction = in[14];
        k.pointCount = k.mPointCount = (int)in[15];
        for (int p = 0; p < k.pointCount; p++) contact_point_masses(k.p[p], k.normal, sh->invMass, sh->invI);
        if (k.pointCount == 2) contact_block_k(k, sh->invMass, sh->invI);
        const int kase = contact_solve_velocity(k, *sh, s);
        out[0] = s.v.x; out[1] = s.v.y; out[2] = s.w;
        out[3] = k.p[0].nI; out[4] = k.p[1].nI; out[5] = k.p[0].tI; out[6] = k.p[1].tI;
        out[7] = (float)kase; out[8] = (float)k.pointCount;
    } else if (op == PROBE_JOINT_VELOCITY || op == PROBE_JOINT_POSITION) {
        const ShapeConst &A = *fixture((float)fA), &B = *fixture((float)fB);
        const float dt = (float)(1.0 / 50);
        Joint j;
        BState sA, sB;
        if (op == PROBE_JOINT_VELOCITY) {
            sA.c = V(0.0f, 0.0f); sA.v = V(in[1], in[2]); sA.w = in[3]; sA.a = in[4];
            sB.c = V(0.0f, 0.0f); sB.v = V(in[5], in[6]); sB.w = in[7]; sB.a = in[8];
            j.imp[0] = in[9]; j.imp[1] = in[10]; j.imp[2] = in[11]; j.motorImpulse = in[12];
            j.motorSpeed = in[13]; j.maxMotorTorque = in[14]; j.limitState = (int)in[15];
            JTemp t;
            joint_init(j, t, *jd, A, B, sA, sB, 1.0f);
            Joint jm = j;
            const float warmLimit = j.imp[2];
            float wA = sA.w, wB = sB.w;
            if (j.limitState != 3) joint_solve_motor(jm, t, A.invI, B.invI, wA, wB, dt);
            joint_solve_velocity(j, t, A, B, sA, sB, dt);
            out[0] = sA.v.x; out[1] = sA.v.y; out[2] = sA.w; out[3] = sB.v.x; out[4] = sB.v.y; out[5] = sB.w;
            out[6] = j.imp[0]; out[7] = j.imp[1]; out[8] = j.imp[2]; out[9] = j.motorImpulse;
            out[10] = (float)j.limitState; out[11] = wA; out[12] = wB; out[13] = warmLimit;
        } else {
            sA.c = V(in[1], in[2]); sA.a = in[3]; sA.v = V(0.0f, 0.0f); sA.w = 0.0f;
            sB.c = V(in[4], in[5]); sB.a = in[6]; sB.v = V(0.0f, 0.0f); sB.w = 0.0f;
            j.imp[0] = j.imp[1] = j.imp[2] = j.motorImpulse = j.motorSpeed = j.maxMotorTorque = 0.0f;
            j.limitState = (int)in[7];
            const bool ok = joint_solve_position(j, *jd, A, B, sA, sB);
            out[0] = sA.c.x; out[1] = sA.c.y; out[2] = sA.a; out[3] = sB.c.x; out[4] = sB.c.y; out[5] = sB.a;
            out[6] = ok ? 1.0f : 0.0f;
        }
    } else if (op == PROBE_INTEGRATE) {
        const float dt = (float)(1.0 / 50);
        BState s;
        s.c = V(in[1], in[2]); s.a = in[3]; s.v = V(in[4], in[5]); s.w = in[6];
        integrate_velocity(s, *sh, V(in[7], in[8]), in[9], V(0.0f, in[10]), dt);
        integrate_position(s, dt);
        out[0] = s.c.x; out[1] = s.c.y; out[2] = s.a; out[3] = s.v.x; out[4] = s.v.y; out[5] = s.w;
    } else if (op == PROBE_CONSTS) {
        if (shaped) {
            out[0] = sh->invMass; out[1] = sh->invI; out[2] = sh->localCenter.x; out[3] = sh->localCenter.y;
            out[4] = sh->friction; out[5] = sh->centroid.x; out[6] = sh->centroid.y; out[7] = (float)sh->count;
        } else {
            out[0] = jd->anchorA.x; out[1] = jd->anchorA.y; out[2] = jd->anchorB.x; out[3] = jd->anchorB.y;
            out[4] = jd->lower; out[5] = jd->upper; out[6] = (float)fA; out[7] = (float)fB;
        }
    } else {
        float K[3][3], b[3], x[3] = {0.0f, 0.0f, 0.0f};
        for (int c = 0; c < 3; c++)
            for (int r = 0; r < 3; r++) K[c][r] = in[3 * c + r];
        for (int r = 0; r < 3; r++) b[r] = in[9 + r];
        if (op == PROBE_SOLVE22) {
            const v2 s = solve22(K, V(b[0], b[1]));
            x[0] = s.x; x[1] = s.y;
        } else {
            solve33(K, b, x);
        }
        out[0] = x[0]; out[1] = x[1]; out[2] = x[2];
    }
}

}  // namespace b2probe
