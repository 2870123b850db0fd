// b2lite.cuh -- the slice of Box2D 2.3's algorithm that gym's Box2D tasks exercise, on the device.
//
// The reference delegates all rigid-body arithmetic to box2d-py 2.3.5 (third party, not in
// /root/reference; gym/envs/box2d/lunar_lander.py:556 and bipedal_walker.py:545 call
// `world.Step(1/50, 180, 60)`).  This header re-derives what that call runs for scenes made of a
// few convex polygons tied by revolute joints (limit + motor) colliding with static edges:
//   Collide: edge-vs-polygon manifolds (reference-face selection with 0.98/0.001 hysteresis,
//            Sutherland-Hodgman clipping, feature ids), begin/end-contact events, warm-start
//            impulse matching by feature id;
//   Solve:   semi-implicit Euler, sequential impulses -- revolute joint (3x3 block with limit
//            state machine, motor clamp), contacts (friction then 2-point block normal solver,
//            condition-number fallback), 180 velocity iterations, translation/rotation clamps,
//            <= 60 Baumgarte position iterations (0.2, slop 0.005) with early exit;
//   Sleep:   0.5 s below 0.01 m/s and 2 deg/s.
// One THREAD per environment: sequential impulses are a Gauss-Seidel sweep, inherently serial
// per env, while 2^16 envs give 2^16-way parallelism; every lane runs the same 180-iteration
// loop so a warp stays converged except for contact-dependent work.
//   TOI:     b2World::SolveTOI for dynamic-vs-static pairs (b2lite_toi.cuh).
// Deviations from Box2D (also listed in DESIGN.md): exhaustive pair tests
// behind the fat-AABB reject instead of the dynamic-tree broad phase, fixed in-island constraint
// order (scene's island order x descending edge index), polynomial sin/cos for body angles.
// float32 throughout, one rounding per operation (-fmad=false), so an independent CPU
// implementation can be matched bit for bit.
#pragma once
#include <cstdint>
#include <type_traits>

// An optimisation barrier that makes a float opaque to the compiler (it must then live in a register instead of
// being recomputed); a no-op for the host build of this header that tests/hostsim uses.
#ifdef __CUDA_ARCH__
#define B2L_KEEP_IN_REGISTER(x) asm volatile("" : "+f"(x))
#else
#define B2L_KEEP_IN_REGISTER(x) ((void)0)
#endif

namespace b2l {

#define LD __device__ __forceinline__
struct v2 { float x, y; };
struct rot { float s, c; };
struct xform { v2 p; rot q; };

#define LD __device__ __forceinline__
LD v2 V(float x, float y) { v2 r; r.x = x; r.y = y; return r; }
LD v2 add(v2 a, v2 b) { return V(a.x + b.x, a.y + b.y); }
LD v2 sub(v2 a, v2 b) { return V(a.x - b.x, a.y - b.y); }
LD v2 neg(v2 a) { return V(-a.x, -a.y); }
LD v2 scl(float s, v2 a) { return V(s * a.x, s * a.y); }
LD float dot(v2 a, v2 b) { return a.x * b.x + a.y * b.y; }
LD float crs(v2 a, v2 b) { return a.x * b.y - a.y * b.x; }
LD v2 crs_vs(v2 a, float s) { return V(s * a.y, -s * a.x); }
LD v2 crs_sv(float s, v2 a) { return V(-s * a.y, s * a.x); }
LD v2 rmul(rot q, v2 v) { return V(q.c * v.x - q.s * v.y, q.s * v.x + q.c * v.y); }
LD v2 xmul(xform T, v2 v) { return V((T.q.c * v.x - T.q.s * v.y) + T.p.x, (T.q.s * v.x + T.q.c * v.y) + T.p.y); }
LD v2 xmulT(xform T, v2 v) {
    const float px = v.x - T.p.x, py = v.y - T.p.y;
    return V(T.q.c * px + T.q.s * py, -T.q.s * px + T.q.c * py);
}
LD float fmin_(float a, float b) { return a < b ? a : b; }
LD float fmax_(float a, float b) { return a > b ? a : b; }
LD float clampf(float a, float lo, float hi) { return fmax_(lo, fmin_(a, hi)); }

// sin/cos of a body angle: two-step Cody-Waite reduction by pi/2 + minimax polynomials.  Each of s, c is within
// 1 ulp of the result + ulp(r1)/2 + ulp(r)/2 (the two rounded fmaf) + |k| * |pi/2 - (C1 - C2)| (1.8e-15 per
// quadrant) of float64 sin/cos(x); tests/test_box2d_geometry_cpu.py asserts that bound.  rot_of(-0.0).s is +0.0.
LD rot rot_of(float x) {
    const float kf = rintf(x * 0.636619772367581343f);
    const int k = (int)kf;
    float r = fmaf(kf, -1.5707963705062866f, x);
    r = fmaf(kf, 4.371139000186241e-08f, r);
    const float r2 = r * r;
    float ps = -1.9515295891e-4f;
    ps = ps * r2 + 8.3321608736e-3f;
    ps = ps * r2 + -1.6666654611e-1f;
    const float sr = r + r * r2 * ps;
    float pc = 2.443315711809948e-5f;
    pc = pc * r2 + -1.388731625493765e-3f;
    pc = pc * r2 + 4.166664568298827e-2f;
    const float cr = (1.0f - 0.5f * r2) + r2 * r2 * pc;
    rot q;
    switch (k & 3) {
    case 0: q.s = sr; q.c = cr; break;
    case 1: q.s = cr; q.c = -sr; break;
    case 2: q.s = -sr; q.c = -cr; break;
    default: q.s = -cr; q.c = sr; break;
    }
    return q;
}

// Box2D 2.3 b2Settings.h
constexpr float kLinearSlop = 0.005f;
constexpr float kAngularSlop = 2.0f / 180.0f * 3.14159265359f;
constexpr float kPolygonRadius = 2.0f * kLinearSlop;
constexpr float kMaxLinearCorrection = 0.2f;
constexpr float kMaxAngularCorrection = 8.0f / 180.0f * 3.14159265359f;
constexpr float kMaxTranslation = 2.0f;
constexpr float kMaxRotation = 0.5f * 3.14159265359f;
constexpr float kBaumgarte = 0.2f;
constexpr float kTimeToSleep = 0.5f;
constexpr float kLinearSleepTol = 0.01f;
constexpr float kAngularSleepTol = 2.0f / 180.0f * 3.14159265359f;
constexpr float kAabbExtension = 0.1f;
constexpr float kFltMax = 3.402823466e+38f;

constexpr int MAXV = 6;
constexpr uint32_t kFlagStepped = 16u;  // World::flags bit: the b2World has stepped before (inv_dt0 != 0)
constexpr uint32_t kFlagOverflow = 32u; // World::flags bit (sticky, survives reset): a touching pair was dropped because
                                        // the scene's manifold table (kMaxVC) was full -- see world_step
constexpr uint32_t kFlagsKept = kFlagStepped | kFlagOverflow;   // what reset() keeps of World::flags

// Shape / mass constants of a polygon fixture + its body, computed once on the host with the same
// float32 operations Box2D uses (b2PolygonShape::Set / ComputeMass, b2Body::ResetMassData).
struct ShapeConst {
    int count;
    v2 verts[MAXV], normals[MAXV], centroid, localCenter;
    float friction, invMass, invI;
};
struct JointDef {  // b2RevoluteJointDef (referenceAngle 0, enableLimit, enableMotor)
    int bodyA, bodyB;
    v2 anchorA, anchorB;
    float lower, upper;
};
struct Body {
    v2 c, v;
    float a, w, sleepTime;
    xform xf;
    // b2Sweep of the current step (continuous collision, b2lite_toi.cuh); not part of the persistent record
    v2 c0;
    float a0, alpha0;
};
struct MPoint { v2 localPoint; float nI, tI; uint32_t id; };
struct Manifold { int type, pointCount; v2 localNormal, localPoint; MPoint pts[2]; };
struct Joint { float imp[3], motorImpulse, motorSpeed, maxMotorTorque; int limitState; };
struct BState { v2 c, v; float a, w; };

// per-env solver state that persists between steps, sized by the scene
template <int NB_, int NJ_, int KS_>
struct WorldBase {
    Body b[NB_];
    Joint j[NJ_];
    uint32_t flags;
    // warm-start store: the contacts that were touching after the last step
    uint32_t slot_key[KS_];      // (body * NE + edge) | (pointCount + 1) << 16 ; 0 = empty
    uint32_t slot_id[KS_][2];
    float slot_nI[KS_][2], slot_tI[KS_][2];
};

LD void sync_xf(Body &b, const ShapeConst &sh) {  // b2Body::SynchronizeTransform
    b.xf.q = rot_of(b.a);
    b.xf.p = sub(b.c, rmul(b.xf.q, sh.localCenter));
}

// ---- b2CollideEdgeAndPolygon (edge without adjacent vertices, moon body at the identity) ---------
struct ClipV { v2 v; uint32_t id; };
LD uint32_t make_id(uint32_t ia, uint32_t ib, uint32_t ta, uint32_t tb) { return ia | (ib << 8) | (ta << 16) | (tb << 24); }

LD int clip_segment(ClipV (&out)[2], const ClipV (&in)[2], v2 normal, float offset, int vertexIndexA) {
    int n = 0;
    const float d0 = dot(normal, in[0].v) - offset, d1 = dot(normal, in[1].v) - offset;
    if (d0 <= 0.0f) out[n++] = in[0];
    if (d1 <= 0.0f) out[n++] = in[1];
    if (d0 * d1 < 0.0f) {
        const float interp = d0 / (d0 - d1);
        out[n].v = add(in[0].v, scl(interp, sub(in[1].v, in[0].v)));
        out[n].id = make_id((uint32_t)vertexIndexA, (in[0].id >> 8) & 0xff, 0u, 1u);
        n++;
    }
    return n;
}

__device__ __noinline__ void collide_edge_polygon(Manifold &m, v2 v1, v2 v2_, const ShapeConst &sh, const xform &xf) {
    const int count = sh.count;
    const v2 centroidB = xmul(xf, sh.centroid);
    v2 edge1 = sub(v2_, v1);
    const float len = sqrtf(edge1.x * edge1.x + edge1.y * edge1.y);
    const float inv = 1.0f / len;
    edge1 = V(edge1.x * inv, edge1.y * inv);
    const v2 normal1 = V(edge1.y, -edge1.x);
    const float offset1 = dot(normal1, sub(centroidB, v1));
    const bool front = offset1 >= 0.0f;
    v2 normal, lower, upper;
    if (front) { normal = normal1; lower = neg(normal1); upper = neg(normal1); }
    else { normal = neg(normal1); lower = normal1; upper = normal1; }
    v2 pv[MAXV], pn[MAXV];
    for (int i = 0; i < count; i++) { pv[i] = xmul(xf, sh.verts[i]); pn[i] = rmul(xf.q, sh.normals[i]); }
    const float radius = 2.0f * kPolygonRadius;
    m.pointCount = 0;
    float edgeSep = kFltMax;
    for (int i = 0; i < count; i++) { const float s = dot(normal, sub(pv[i], v1)); if (s < edgeSep) edgeSep = s; }
    if (edgeSep > radius) return;
    int polyType = 0, polyIndex = -1;
    float polySep = -kFltMax;
    const v2 perp = V(-normal.y, normal.x);
    for (int i = 0; i < count; i++) {
        const v2 n = neg(pn[i]);
        const float s1 = dot(n, sub(pv[i], v1)), s2 = dot(n, sub(pv[i], v2_));
        const float s = fmin_(s1, s2);
        if (s > radius) { polyType = 1; polyIndex = i; polySep = s; break; }
        if (dot(n, perp) >= 0.0f) { if (dot(sub(n, upper), normal) < -kAngularSlop) continue; }
        else { if (dot(sub(n, lower), normal) < -kAngularSlop) continue; }
        if (s > polySep) { polyType = 1; polyIndex = i; polySep = s; }
    }
    if (polyType != 0 && polySep > radius) return;
    bool primaryEdge;
    if (polyType == 0) primaryEdge = true;
    else if (polySep > 0.98f * edgeSep + 0.001f) primaryEdge = false;
    else primaryEdge = true;

    ClipV ie[2];
    int rf_i1, rf_i2;
    v2 rf_v1, rf_v2, rf_normal;
    if (primaryEdge) {
        m.type = 0;
        int best = 0;
        float bestVal = dot(normal, pn[0]);
        for (int i = 1; i < count; i++) { const float val = dot(normal, pn[i]); if (val < bestVal) { bestVal = val; best = i; } }
        const int i1 = best, i2 = i1 + 1 < count ? i1 + 1 : 0;
        ie[0].v = pv[i1]; ie[0].id = make_id(0u, (uint32_t)i1, 1u, 0u);
        ie[1].v = pv[i2]; ie[1].id = make_id(0u, (uint32_t)i2, 1u, 0u);
        if (front) { rf_i1 = 0; rf_i2 = 1; rf_v1 = v1; rf_v2 = v2_; rf_normal = normal1; }
        else { rf_i1 = 1; rf_i2 = 0; rf_v1 = v2_; rf_v2 = v1; rf_normal = neg(normal1); }
    } else {
        m.type = 1;
        ie[0].v = v1; ie[0].id = make_id(0u, (uint32_t)polyIndex, 0u, 1u);
        ie[1].v = v2_; ie[1].id = make_id(0u, (uint32_t)polyIndex, 0u, 1u);
        rf_i1 = polyIndex; rf_i2 = rf_i1 + 1 < count ? rf_i1 + 1 : 0;
        rf_v1 = pv[rf_i1]; rf_v2 = pv[rf_i2]; rf_normal = pn[rf_i1];
    }
    const v2 side1 = V(rf_normal.y, -rf_normal.x), side2 = neg(side1);
    const float off1 = dot(side1, rf_v1), off2 = dot(side2, rf_v2);
    ClipV c1[2], c2[2];
    if (clip_segment(c1, ie, side1, off1, rf_i1) < 2) return;
    if (clip_segment(c2, c1, side2, off2, rf_i2) < 2) return;
    if (primaryEdge) { m.localNormal = rf_normal; m.localPoint = rf_v1; }
    else { m.localNormal = sh.normals[rf_i1]; m.localPoint = sh.verts[rf_i1]; }
    int pc = 0;
    for (int i = 0; i < 2; i++) {
        const float sep = dot(rf_normal, sub(c2[i].v, rf_v1));
        if (sep <= radius) {
            MPoint &cp = m.pts[pc];
            if (primaryEdge) { cp.localPoint = xmulT(xf, c2[i].v); cp.id = c2[i].id; }
            else {
                const uint32_t id = c2[i].id;
                cp.localPoint = c2[i].v;
                cp.id = make_id((id >> 8) & 0xff, id & 0xff, (id >> 24) & 0xff, (id >> 16) & 0xff);
            }
            pc++;
        }
    }
    m.pointCount = pc;
}

// ---- b2CollidePolygons (Box2D 2.3.1+: brute-force b2FindMaxSeparation), polygon A = a static 4-gon at the
// identity transform (BipedalWalkerHardcore's stumps, stair steps, pit walls), polygon B = a body's fixture ----
struct StaticBox { v2 verts[4], normals[4]; };

// b2PolygonShape::Set on the corners of an axis-aligned box: hull from the right-most lowest corner, CCW
LD void static_box(StaticBox &s, float x0, float ylo, float x1, float yhi) {
    s.verts[0] = V(x1, ylo); s.verts[1] = V(x1, yhi); s.verts[2] = V(x0, yhi); s.verts[3] = V(x0, ylo);
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const v2 edge = sub(s.verts[(i + 1) & 3], s.verts[i]);
        const v2 nr = crs_vs(edge, 1.0f);
        const float len = sqrtf(nr.x * nr.x + nr.y * nr.y);
        const float inv = 1.0f / len;
        s.normals[i] = V(inv * nr.x, inv * nr.y);
    }
}

LD v2 rmulT(rot q, v2 v) { return V(q.c * v.x + q.s * v.y, -q.s * v.x + q.c * v.y); }
LD xform xf_mulT(const xform &A, const xform &B) {  // b2MulT(A, B)
    xform C;
    C.q.s = A.q.c * B.q.s - A.q.s * B.q.c;
    C.q.c = A.q.c * B.q.c + A.q.s * B.q.s;
    C.p = rmulT(A.q, sub(B.p, A.p));
    return C;
}

LD float find_max_separation(int &edgeIndex, int count1, const v2 *n1s, const v2 *v1s, const xform &xf1, int count2,
                             const v2 *v2s, const xform &xf2) {
    const xform xf = xf_mulT(xf2, xf1);
    int bestIndex = 0;
    float maxSeparation = -kFltMax;
    for (int i = 0; i < count1; i++) {
        const v2 n = rmul(xf.q, n1s[i]);
        const v2 v1 = xmul(xf, v1s[i]);
        float si = kFltMax;
        for (int j = 0; j < count2; j++) { const float sij = dot(n, sub(v2s[j], v1)); if (sij < si) si = sij; }
        if (si > maxSeparation) { maxSeparation = si; bestIndex = i; }
    }
    edgeIndex = bestIndex;
    return maxSeparation;
}

__device__ __noinline__ void collide_polygons(Manifold &m, const StaticBox &A, const ShapeConst &sh, const xform &xfB) {
    xform xfA;
    xfA.p = V(0.0f, 0.0f); xfA.q.s = 0.0f; xfA.q.c = 1.0f;
    m.pointCount = 0;
    const float totalRadius = kPolygonRadius + kPolygonRadius;
    int edgeA = 0, edgeB = 0;
    const float separationA = find_max_separation(edgeA, 4, A.normals, A.verts, xfA, sh.count, sh.verts, xfB);
    if (separationA > totalRadius) return;
    const float separationB = find_max_separation(edgeB, sh.count, sh.normals, sh.verts, xfB, 4, A.verts, xfA);
    if (separationB > totalRadius) return;
    const v2 *verts1, *normals1, *verts2, *normals2;
    int count1, count2, edge1;
    bool flip;
    xform xf1, xf2;
    const float k_tol = 0.1f * kLinearSlop;
    if (separationB > separationA + k_tol) {
        verts1 = sh.verts; normals1 = sh.normals; count1 = sh.count; verts2 = A.verts; normals2 = A.normals; count2 = 4;
        xf1 = xfB; xf2 = xfA; edge1 = edgeB; m.type = 1; flip = true;
    } else {
        verts1 = A.verts; normals1 = A.normals; count1 = 4; verts2 = sh.verts; normals2 = sh.normals; count2 = sh.count;
        xf1 = xfA; xf2 = xfB; edge1 = edgeA; m.type = 0; flip = false;
    }
    ClipV ie[2];
    {   // b2FindIncidentEdge
        const v2 normal1 = rmulT(xf2.q, rmul(xf1.q, normals1[edge1]));
        int index = 0;
        float minDot = kFltMax;
        for (int i = 0; i < count2; i++) { const float d = dot(normal1, normals2[i]); if (d < minDot) { minDot = d; index = i; } }
        const int i1 = index, i2 = i1 + 1 < count2 ? i1 + 1 : 0;
        ie[0].v = xmul(xf2, verts2[i1]); ie[0].id = make_id((uint32_t)edge1, (uint32_t)i1, 1u, 0u);
        ie[1].v = xmul(xf2, verts2[i2]); ie[1].id = make_id((uint32_t)edge1, (uint32_t)i2, 1u, 0u);
    }
    const int iv1 = edge1, iv2 = edge1 + 1 < count1 ? edge1 + 1 : 0;
    v2 v11 = verts1[iv1], v12 = verts1[iv2];
    v2 localTangent = sub(v12, v11);
    {
        const float len = sqrtf(localTangent.x * localTangent.x + localTangent.y * localTangent.y);
        if (len >= 1.1920929e-07f) { const float inv = 1.0f / len; localTangent.x *= inv; localTangent.y *= inv; }
    }
    const v2 localNormal = crs_vs(localTangent, 1.0f);
    const v2 planePoint = scl(0.5f, add(v11, v12));
    const v2 tangent = rmul(xf1.q, localTangent);
    const v2 normal = crs_vs(tangent, 1.0f);
    v11 = xmul(xf1, v11); v12 = xmul(xf1, v12);
    const float frontOffset = dot(normal, v11);
    const float sideOffset1 = -dot(tangent, v11) + totalRadius;
    const float sideOffset2 = dot(tangent, v12) + totalRadius;
    ClipV c1[2], c2[2];
    if (clip_segment(c1, ie, neg(tangent), sideOffset1, iv1) < 2) return;
    if (clip_segment(c2, c1, tangent, sideOffset2, iv2) < 2) return;
    m.localNormal = localNormal;
    m.localPoint = planePoint;
    int pc = 0;
    for (int i = 0; i < 2; i++) {
        const float separation = dot(normal, c2[i].v) - frontOffset;
        if (separation <= totalRadius) {
            MPoint &cp = m.pts[pc];
            cp.localPoint = xmulT(xf2, c2[i].v);
            const uint32_t id = c2[i].id;
            cp.id = flip ? make_id((id >> 8) & 0xff, id & 0xff, (id >> 24) & 0xff, (id >> 16) & 0xff) : id;
            pc++;
        }
    }
    m.pointCount = pc;
}

// b2PolygonShape::RayCast against a static box at the identity transform
LD bool static_box_raycast(const StaticBox &s, v2 p1_, v2 p2_, float maxFraction, float &t_out) {
    rot qi;
    qi.s = 0.0f; qi.c = 1.0f;
    const v2 p1 = rmulT(qi, sub(p1_, V(0.0f, 0.0f))), p2 = rmulT(qi, sub(p2_, V(0.0f, 0.0f)));
    const v2 d = sub(p2, p1);
    float lower = 0.0f, upper = maxFraction;
    int index = -1;
    for (int i = 0; i < 4; i++) {
        const float numerator = dot(s.normals[i], sub(s.verts[i], p1));
        const float denominator = dot(s.normals[i], d);
        if (denominator == 0.0f) { if (numerator < 0.0f) return false; }
        else {
            if (denominator < 0.0f && numerator < lower * denominator) { lower = numerator / denominator; index = i; }
            else if (denominator > 0.0f && numerator < upper * denominator) upper = numerator / denominator;
        }
        if (upper < lower) return false;
    }
    if (index >= 0) { t_out = lower; return true; }
    return false;
}

// compile-time loop: f(std::integral_constant<int, I>{}) for I in [I0, N)
template <int I, int N, typename F>
__device__ __forceinline__ void static_for(F &&f) {
    if constexpr (I < N) {
        f(std::integral_constant<int, I>{});
        static_for<I + 1, N>(static_cast<F &&>(f));
    }
}

// ---- constraints ---------------------------------------------------------------------------------
struct VCP { v2 rB; float nI, tI, normalMass, tangentMass; };
struct VC {
    int body, edge, pointCount, mPointCount, mType;
    v2 normal, localNormal, localPoint, lp[2];
    VCP p[2];
    float k11, k12, k22, n11, n12, n22;  // K and its inverse (symmetric)
    float friction;
};

struct JTemp { v2 rA, rB; float K[3][3], motorMass; };

LD void solve33(const float (&K)[3][3], const float (&b)[3], float (&x)[3]) {
    const float *ex = K[0], *ey = K[1], *ez = K[2];
    const float cx = ey[1] * ez[2] - ey[2] * ez[1], cy = ey[2] * ez[0] - ey[0] * ez[2], cz = ey[0] * ez[1] - ey[1] * ez[0];
    float det = ex[0] * cx + ex[1] * cy + ex[2] * cz;
    if (det != 0.0f) det = 1.0f / det;
    x[0] = det * (b[0] * cx + b[1] * cy + b[2] * cz);
    const float bx = b[1] * ez[2] - b[2] * ez[1], by = b[2] * ez[0] - b[0] * ez[2], bz = b[0] * ez[1] - b[1] * ez[0];
    x[1] = det * (ex[0] * bx + ex[1] * by + ex[2] * bz);
    const float dx = ey[1] * b[2] - ey[2] * b[1], dy = ey[2] * b[0] - ey[0] * b[2], dz = ey[0] * b[1] - ey[1] * b[0];
    x[2] = det * (ex[0] * dx + ex[1] * dy + ex[2] * dz);
}
LD v2 solve22(const float (&K)[3][3], v2 b) {
    const float a11 = K[0][0], a12 = K[1][0], a21 = K[0][1], a22 = K[1][1];
    float det = a11 * a22 - a12 * a21;
    if (det != 0.0f) det = 1.0f / det;
    return V(det * (a22 * b.x - a12 * b.y), det * (a11 * b.y - a21 * b.x));
}

// b2RevoluteJoint::InitVelocityConstraints (bodyA = lander, bodyB = leg li)
// b2RevoluteJoint::InitVelocityConstraints
LD void joint_init(Joint &j, JTemp &t, const JointDef &d, const ShapeConst &A, const ShapeConst &B, BState &sA, BState &sB,
                   float dtRatio) {
    const float mA = A.invMass, mB = B.invMass, iA = A.invI, iB = B.invI;
    const rot qA = rot_of(sA.a), qB = rot_of(sB.a);
    t.rA = rmul(qA, sub(d.anchorA, A.localCenter));
    t.rB = rmul(qB, sub(d.anchorB, B.localCenter));
    const v2 rA = t.rA, rB = t.rB;
    t.K[0][0] = mA + mB + rA.y * rA.y * iA + rB.y * rB.y * iB;
    t.K[1][0] = -rA.y * rA.x * iA - rB.y * rB.x * iB;
    t.K[2][0] = -rA.y * iA - rB.y * iB;
    t.K[0][1] = t.K[1][0];
    t.K[1][1] = mA + mB + rA.x * rA.x * iA + rB.x * rB.x * iB;
    t.K[2][1] = rA.x * iA + rB.x * iB;
    t.K[0][2] = t.K[2][0];
    t.K[1][2] = t.K[2][1];
    t.K[2][2] = iA + iB;
    t.motorMass = iA + iB;
    if (t.motorMass > 0.0f) t.motorMass = 1.0f / t.motorMass;
    // K is loop-invariant over the 180 velocity iterations; without this the compiler prefers to recompute its
    // entries from rA / rB inside the loop (10 % of all executed instructions in the ncu source view)
#pragma unroll
    for (int c = 0; c < 3; c++)
#pragma unroll
        for (int r = c; r < 3; r++) { B2L_KEEP_IN_REGISTER(t.K[c][r]); t.K[r][c] = t.K[c][r]; }
    const float jointAngle = sB.a - sA.a - 0.0f;
    const float lower = d.lower, upper = d.upper;
    if (fabsf(upper - lower) < 2.0f * kAngularSlop) j.limitState = 3;
    else if (jointAngle <= lower) { if (j.limitState != 1) j.imp[2] = 0.0f; j.limitState = 1; }
    else if (jointAngle >= upper) { if (j.limitState != 2) j.imp[2] = 0.0f; j.limitState = 2; }
    else { j.limitState = 0; j.imp[2] = 0.0f; }
    j.imp[0] *= dtRatio; j.imp[1] *= dtRatio; j.imp[2] *= dtRatio; j.motorImpulse *= dtRatio;
    const v2 P = V(j.imp[0], j.imp[1]);
    sA.v = sub(sA.v, scl(mA, P));
    sA.w -= iA * (crs(rA, P) + j.motorImpulse + j.imp[2]);
    sB.v = add(sB.v, scl(mB, P));
    sB.w += iB * (crs(rB, P) + j.motorImpulse + j.imp[2]);
}

LD void joint_solve_velocity(Joint &j, const JTemp &t, const ShapeConst &A, const ShapeConst &B, BState &sA,
                                                  BState &sB, float dt) {
    const float mA = A.invMass, mB = B.invMass, iA = A.invI, iB = B.invI;
    v2 vA = sA.v, vB = sB.v;
    float wA = sA.w, wB = sB.w;
    if (j.limitState != 3) {
        const float Cdot = wB - wA - j.motorSpeed;
        float impulse = -t.motorMass * Cdot;
        const float oldImpulse = j.motorImpulse, maxImpulse = dt * j.maxMotorTorque;
        j.motorImpulse = clampf(oldImpulse + impulse, -maxImpulse, maxImpulse);
        impulse = j.motorImpulse - oldImpulse;
        wA -= iA * impulse;
        wB += iB * impulse;
    }
    if (j.limitState != 0) {
        const v2 Cdot1 = sub(sub(add(vB, crs_sv(wB, t.rB)), vA), crs_sv(wA, t.rA));
        const float Cdot2 = wB - wA;
        const float Cd[3] = {Cdot1.x, Cdot1.y, Cdot2};
        float imp[3];
        solve33(t.K, Cd, imp);
        imp[0] = -imp[0]; imp[1] = -imp[1]; imp[2] = -imp[2];
        if (j.limitState == 3) { j.imp[0] += imp[0]; j.imp[1] += imp[1]; j.imp[2] += imp[2]; }
        else {
            const float newImpulse = j.imp[2] + imp[2];
            const bool violated = (j.limitState == 1) ? (newImpulse < 0.0f) : (newImpulse > 0.0f);
            if (violated) {
                const v2 rhs = add(neg(Cdot1), scl(j.imp[2], V(t.K[2][0], t.K[2][1])));
                const v2 red = solve22(t.K, rhs);
                imp[0] = red.x; imp[1] = red.y; imp[2] = -j.imp[2];
                j.imp[0] += red.x; j.imp[1] += red.y; j.imp[2] = 0.0f;
            } else { j.imp[0] += imp[0]; j.imp[1] += imp[1]; j.imp[2] += imp[2]; }
        }
        const v2 P = V(imp[0], imp[1]);
        vA = sub(vA, scl(mA, P)); wA -= iA * (crs(t.rA, P) + imp[2]);
        vB = add(vB, scl(mB, P)); wB += iB * (crs(t.rB, P) + imp[2]);
    } else {
        const v2 Cdot = sub(sub(add(vB, crs_sv(wB, t.rB)), vA), crs_sv(wA, t.rA));
        const v2 imp = solve22(t.K, neg(Cdot));
        j.imp[0] += imp.x; j.imp[1] += imp.y;
        vA = sub(vA, scl(mA, imp)); wA -= iA * crs(t.rA, imp);
        vB = add(vB, scl(mB, imp)); wB += iB * crs(t.rB, imp);
    }
    sA.v = vA; sA.w = wA; sB.v = vB; sB.w = wB;
}

LD bool joint_solve_position(const Joint &j, const JointDef &d, const ShapeConst &A, const ShapeConst &B,
                                                  BState &sA, BState &sB) {
    const float mA = A.invMass, mB = B.invMass, iA = A.invI, iB = B.invI;
    v2 cA = sA.c, cB = sB.c;
    float aA = sA.a, aB = sB.a, angularError = 0.0f, positionError;
    if (j.limitState != 0) {
        float motorMass = iA + iB;
        if (motorMass > 0.0f) motorMass = 1.0f / motorMass;
        const float angle = aB - aA - 0.0f;
        float limitImpulse = 0.0f;
        if (j.limitState == 3) {
            const float C = clampf(angle - d.lower, -kMaxAngularCorrection, kMaxAngularCorrection);
            limitImpulse = -motorMass * C; angularError = fabsf(C);
        } else if (j.limitState == 1) {
            float C = angle - d.lower; angularError = -C;
            C = clampf(C + kAngularSlop, -kMaxAngularCorrection, 0.0f); limitImpulse = -motorMass * C;
        } else {
            float C = angle - d.upper; angularError = C;
            C = clampf(C - kAngularSlop, 0.0f, kMaxAngularCorrection); limitImpulse = -motorMass * C;
        }
        aA -= iA * limitImpulse;
        aB += iB * limitImpulse;
    }
    {
        const rot qA = rot_of(aA), qB = rot_of(aB);
        const v2 rA = rmul(qA, sub(d.anchorA, A.localCenter)), rB = rmul(qB, sub(d.anchorB, B.localCenter));
        const v2 C = sub(sub(add(cB, rB), cA), rA);
        positionError = sqrtf(C.x * C.x + C.y * C.y);
        const float k11 = mA + mB + iA * rA.y * rA.y + iB * rB.y * rB.y;
        const float k12 = -iA * rA.x * rA.y - iB * rB.x * rB.y;
        const float k22 = mA + mB + iA * rA.x * rA.x + iB * rB.x * rB.x;
        float det = k11 * k22 - k12 * k12;
        if (det != 0.0f) det = 1.0f / det;
        const v2 imp = V(-(det * (k22 * C.x - k12 * C.y)), -(det * (k11 * C.y - k12 * C.x)));
        cA = sub(cA, scl(mA, imp)); aA -= iA * crs(rA, imp);
        cB = add(cB, scl(mB, imp)); aB += iB * crs(rB, imp);
    }
    sA.c = cA; sA.a = aA; sB.c = cB; sB.a = aB;
    return positionError <= kLinearSlop && angularError <= kAngularSlop;
}

#include "b2lite_toi.cuh"

// ---- b2World::Step(1/50, 180, 60) for one env ------------------------------------------------------
// Scene supplies: NB, NJ, kSlots, kMaxVC, World (with b[], j[], flags, slot_*), shape(b), jdef(k),
// body_order(k), joint_order(k), joint_body_a(k), joint_body_b(k) (all constexpr), edge(W, e, v1, v2, friction), edge_range(W, lox, hix, lo, hi), NP (+ poly(W, p,
// x0, ylo, x1, yhi, friction), poly_range(W, lox, hix, lo, hi) when NP > 0), on_event(W, body, begin).  `force0` / `torque0` are the force and torque accumulated on body 0 before the
// step (b2Body::ApplyForceToCenter / ApplyTorque), `gravity_y` the world's gravity (0, gravity_y).  `live`: mask of
// the warp's lanes that call world_step together (they synchronise inside solve_toi), or 0.
template <typename Scene>
__device__ __noinline__ void world_step(typename Scene::World &W, v2 force0, float torque0, float gravity_y,
                                        bool &island_awake, unsigned live = 0u, bool run_toi = true) {
    constexpr int NB = Scene::NB, NJ = Scene::NJ, kSlots = Scene::kSlots, kMaxVC = Scene::kMaxVC;
    constexpr int NE = Scene::NE, NP = Scene::NP, NF = NE + NP;
    const float dt = (float)(1.0 / 50);
    const float inv_dt0 = (W.flags & kFlagStepped) ? 1.0f / dt : 0.0f;
    const float dtRatio = inv_dt0 * dt;
    const v2 gravity = V(0.0f, gravity_y);

    // --- Collide + begin/end events; touching pairs become velocity constraints in island order
    VC vc[kMaxVC];
    int nvc = 0;
    int cend[NB];   // contacts of island position oi: vc[cend[oi - 1] .. cend[oi])
#pragma unroll
    for (int oi = 0; oi < NB; oi++) {
        const int b = Scene::body_order(oi);
        const ShapeConst &sh = Scene::shape(b);
        // fat AABB of the polygon (broad-phase stand-in)
        float lox = kFltMax, loy = kFltMax, hix = -kFltMax, hiy = -kFltMax;
        for (int i = 0; i < sh.count; i++) {
            const v2 p = xmul(W.b[b].xf, sh.verts[i]);
            lox = fmin_(lox, p.x); loy = fmin_(loy, p.y); hix = fmax_(hix, p.x); hiy = fmax_(hiy, p.y);
        }
        const float ext = kPolygonRadius + kAabbExtension;
        // candidate ground fixtures: those the scene says can overlap the AABB, widened to every fixture this
        // body was touching last step (so that leaving it raises EndContact).  Fixture index f: edges 0..NE-1,
        // static polygons NE..NE+NP-1; visited in descending f (polygons first, then edges).
        int e_lo, e_hi, p_lo = 0, p_hi = -1;
        Scene::edge_range(W, lox - ext, hix + ext, e_lo, e_hi);
        if constexpr (NP > 0) Scene::poly_range(W, lox - ext, hix + ext, p_lo, p_hi);
        for (int s = 0; s < kSlots; s++)
            if ((W.slot_key[s] >> 16) && (int)((W.slot_key[s] & 0xffffu) / NF) == b) {
                const int pf = (int)((W.slot_key[s] & 0xffffu) % NF);
                if (pf < NE) { e_lo = pf < e_lo ? pf : e_lo; e_hi = pf > e_hi ? pf : e_hi; }
                else if (p_hi < p_lo) { p_lo = p_hi = pf - NE; }
                else { p_lo = pf - NE < p_lo ? pf - NE : p_lo; p_hi = pf - NE > p_hi ? pf - NE : p_hi; }
            }
        for (int f = (NP > 0 && p_hi >= p_lo) ? NE + p_hi : e_hi; f >= e_lo;) {
            const int pair = b * NF + f;
            bool was = false;
            for (int s = 0; s < kSlots; s++) was = was || ((W.slot_key[s] >> 16) && (int)(W.slot_key[s] & 0xffffu) == pair);
            float efric;
            Manifold m;
            m.pointCount = 0;
            if (NP > 0 && f >= NE) {
                if constexpr (NP > 0) {
                    float x0, ylo, x1, yhi;
                    Scene::poly(W, f - NE, x0, ylo, x1, yhi, efric);
                    if (!(lox - ext > x1 + ext || x0 - ext > hix + ext || loy - ext > yhi + ext || ylo - ext > hiy + ext)) {
                        StaticBox sb;
                        static_box(sb, x0, ylo, x1, yhi);
                        collide_polygons(m, sb, sh, W.b[b].xf);
                    }
                }
            } else {
                v2 v1, v2_;
                Scene::edge(W, f, v1, v2_, efric);
                const float elox = fmin_(v1.x, v2_.x) - ext, ehix = fmax_(v1.x, v2_.x) + ext;
                const float eloy = fmin_(v1.y, v2_.y) - ext, ehiy = fmax_(v1.y, v2_.y) + ext;
                if (!(lox - ext > ehix || elox > hix + ext || loy - ext > ehiy || eloy > hiy + ext))
                    collide_edge_polygon(m, v1, v2_, sh, W.b[b].xf);
            }
            const int e = f;
            f--;
            if (f > e_hi && f < NE + p_lo) f = e_hi;   // from the lowest candidate polygon down to the highest candidate edge
            bool touching = m.pointCount > 0;
            if (touching && nvc >= kMaxVC) {
                // manifold table full: the pair is treated as NOT touching (no constraint, no warm-start slot, no
                // BeginContact; EndContact if it was touching) -- the CPU checker in the test tree applies the same
                // rule with the same capacity, so the two stay bit-identical even here; the env is marked so that
                // tests / b200gym_box2d_overflows can assert it never happens in practice
                touching = false;
                W.flags |= kFlagOverflow;
            }
            if (touching != was) Scene::on_event(W, b, touching);  // Begin/EndContact listener
            if (!touching) continue;
            {
                VC &k = vc[nvc++];
                k.body = b; k.edge = e; k.mType = m.type; k.mPointCount = m.pointCount; k.pointCount = m.pointCount;
                k.localNormal = m.localNormal; k.localPoint = m.localPoint;
                k.friction = sqrtf(efric * sh.friction);
                for (int p = 0; p < m.pointCount; p++) {
                    k.lp[p] = m.pts[p].localPoint;
                    float nI = 0.0f, tI = 0.0f;
                    if (was)  // match old contact ids to new contact ids (b2Contact::Update)
                        for (int s = 0; s < kSlots; s++)
                            if ((W.slot_key[s] & 0xffffu) == (uint32_t)pair && (W.slot_key[s] >> 16)) {
                                const int oc = (int)(W.slot_key[s] >> 16) - 1;
                                for (int q = 0; q < oc; q++)
                                    if (W.slot_id[s][q] == m.pts[p].id) { nI = W.slot_nI[s][q]; tI = W.slot_tI[s][q]; break; }
                            }
                    k.p[p].nI = dtRatio * nI;
                    k.p[p].tI = dtRatio * tI;
                    k.lp[p] = m.pts[p].localPoint;
                    // keep the feature id in the slot arrays of the NEW store (written below)
                    k.p[p].normalMass = __uint_as_float(m.pts[p].id);
                }
            }
        }
        cend[oi] = nvc;
    }

    // From here on every body / joint index is a compile-time constant (static_for over the scene's island
    // order), so st[], jn[], jt[] live in registers for the whole 180 + 60 iteration solve; only the contact
    // constraints (their number is data dependent) stay in local memory.  Contacts were appended body by body
    // in island order: those of island position oi are vc[cbeg(oi) .. cend[oi]).
    // --- integrate velocities
    BState st[NB];
    static_for<0, NB>([&](auto I) {
        constexpr int i = decltype(I)::value;
        const ShapeConst &sh = Scene::shape(i);
        v2 v = W.b[i].v;
        float w = W.b[i].w;
        const v2 force = i == 0 ? force0 : V(0.0f, 0.0f);
        v = add(v, scl(dt, add(gravity, scl(sh.invMass, force))));
        w = w + dt * sh.invI * (i == 0 ? torque0 : 0.0f);
        v = scl(1.0f / (1.0f + dt * 0.0f), v);
        w = w * (1.0f / (1.0f + dt * 0.0f));
        st[i].c = W.b[i].c; st[i].a = W.b[i].a; st[i].v = v; st[i].w = w;
    });
    Joint jn[NJ];
    static_for<0, NJ>([&](auto K) { constexpr int k = decltype(K)::value; jn[k] = W.j[k]; });
    // --- InitializeVelocityConstraints (+ remember the feature ids for the new store)
    uint32_t ids[kMaxVC][2];
    static_for<0, NB>([&](auto OI) {
        constexpr int oi = decltype(OI)::value, body = Scene::body_order(oi);
        const ShapeConst &sh = Scene::shape(body);
        const BState &sB = st[body];
        const float mB = sh.invMass, iB = sh.invI;
        for (int ci = oi == 0 ? 0 : cend[oi == 0 ? 0 : oi - 1]; ci < cend[oi]; ci++) {
            VC &k = vc[ci];
            ids[ci][0] = __float_as_uint(k.p[0].normalMass);
            ids[ci][1] = k.pointCount > 1 ? __float_as_uint(k.p[1].normalMass) : 0u;
            xform xfB;
            xfB.q = rot_of(sB.a);
            xfB.p = sub(sB.c, rmul(xfB.q, sh.localCenter));
            v2 pts[2];
            xform xfA;  // the ground body: identity transform (kept as explicit arithmetic, like Box2D does)
            xfA.p = V(0.0f, 0.0f); xfA.q.s = 0.0f; xfA.q.c = 1.0f;
            if (k.mType == 0) {  // b2WorldManifold::Initialize, e_faceA
                k.normal = rmul(xfA.q, k.localNormal);
                const v2 plane = xmul(xfA, k.localPoint);
                for (int p = 0; p < k.pointCount; p++) {
                    const v2 clip = xmul(xfB, k.lp[p]);
                    const v2 cA = add(clip, scl(kPolygonRadius - dot(sub(clip, plane), k.normal), k.normal));
                    const v2 cB = sub(clip, scl(kPolygonRadius, k.normal));
                    pts[p] = scl(0.5f, add(cA, cB));
                }
            } else {             // e_faceB
                v2 nrm = rmul(xfB.q, k.localNormal);
                const v2 plane = xmul(xfB, k.localPoint);
                for (int p = 0; p < k.pointCount; p++) {
                    const v2 clip = xmul(xfA, k.lp[p]);
                    const v2 cB = add(clip, scl(kPolygonRadius - dot(sub(clip, plane), nrm), nrm));
                    const v2 cA = sub(clip, scl(kPolygonRadius, nrm));
                    pts[p] = scl(0.5f, add(cA, cB));
                }
                k.normal = neg(nrm);
            }
            for (int p = 0; p < k.pointCount; p++) {
                VCP &cp = k.p[p];
                cp.rB = sub(pts[p], sB.c);
                const float rnB = crs(cp.rB, k.normal);
                const float kN = mB + iB * rnB * rnB;
                cp.normalMass = kN > 0.0f ? 1.0f / kN : 0.0f;
                const v2 tangent = crs_vs(k.normal, 1.0f);
                const float rtB = crs(cp.rB, tangent);
                const float kT = mB + iB * rtB * rtB;
                cp.tangentMass = kT > 0.0f ? 1.0f / kT : 0.0f;
            }
            if (k.pointCount == 2) {
                const float rn1B = crs(k.p[0].rB, k.normal), rn2B = crs(k.p[1].rB, k.normal);
                const float k11 = mB + iB * rn1B * rn1B, k22 = mB + iB * rn2B * rn2B, k12 = mB + iB * rn1B * rn2B;
                if (k11 * k11 < 1000.0f * (k11 * k22 - k12 * k12)) {
                    k.k11 = k11; k.k12 = k12; k.k22 = k22;
                    float det = k11 * k22 - k12 * k12;
                    if (det != 0.0f) det = 1.0f / det;
                    k.n11 = det * k22; k.n12 = -det * k12; k.n22 = det * k11;
                } else k.pointCount = 1;
            }
        }
    });
    // --- WarmStart
    static_for<0, NB>([&](auto OI) {
        constexpr int oi = decltype(OI)::value, body = Scene::body_order(oi);
        const ShapeConst &sh = Scene::shape(body);
        BState &sB = st[body];
        for (int ci = oi == 0 ? 0 : cend[oi == 0 ? 0 : oi - 1]; ci < cend[oi]; ci++) {
            VC &k = vc[ci];
            const v2 tangent = crs_vs(k.normal, 1.0f);
            for (int p = 0; p < k.pointCount; p++) {
                const v2 P = add(scl(k.p[p].nI, k.normal), scl(k.p[p].tI, tangent));
                sB.w += sh.invI * crs(k.p[p].rB, P);
                sB.v = add(sB.v, scl(sh.invMass, P));
            }
        }
    });
    // --- joints in island order
    JTemp jt[NJ];
    static_for<0, NJ>([&](auto Q) {
        constexpr int k = Scene::joint_order(decltype(Q)::value), bA = Scene::joint_body_a(k), bB = Scene::joint_body_b(k);
        joint_init(jn[k], jt[k], Scene::jdef(k), Scene::shape(bA), Scene::shape(bB), st[bA], st[bB], dtRatio);
    });

    // --- 180 velocity iterations
#pragma unroll 1
    for (int it = 0; it < 180; it++) {
        static_for<0, NJ>([&](auto Q) {
            constexpr int k = Scene::joint_order(decltype(Q)::value), bA = Scene::joint_body_a(k), bB = Scene::joint_body_b(k);
            joint_solve_velocity(jn[k], jt[k], Scene::shape(bA), Scene::shape(bB), st[bA], st[bB], dt);
        });
        if (nvc != 0) static_for<0, NB>([&](auto OI) {
            constexpr int oi = decltype(OI)::value, body = Scene::body_order(oi);
            const ShapeConst &sh = Scene::shape(body);
            const float mB = sh.invMass, iB = sh.invI;
            for (int ci = oi == 0 ? 0 : cend[oi == 0 ? 0 : oi - 1]; ci < cend[oi]; ci++) {
                VC &k = vc[ci];
                v2 vB = st[body].v;
                float wB = st[body].w;
                const v2 normal = k.normal, tangent = crs_vs(normal, 1.0f);
                for (int p = 0; p < k.pointCount; p++) {
                    VCP &cp = k.p[p];
                    const v2 dv = add(vB, crs_sv(wB, cp.rB));
                    const float vt = dot(dv, tangent) - 0.0f;
                    float lambda = cp.tangentMass * (-vt);
                    const float maxF = k.friction * cp.nI;
                    const float newImp = clampf(cp.tI + lambda, -maxF, maxF);
                    lambda = newImp - cp.tI;
                    cp.tI = newImp;
                    const v2 P = scl(lambda, tangent);
                    vB = add(vB, scl(mB, P)); wB += iB * crs(cp.rB, P);
                }
                if (k.pointCount == 1) {
                    VCP &cp = k.p[0];
                    const v2 dv = add(vB, crs_sv(wB, cp.rB));
                    const float vn = dot(dv, normal);
                    float lambda = -cp.normalMass * (vn - 0.0f);
                    const float newImp = fmax_(cp.nI + lambda, 0.0f);
                    lambda = newImp - cp.nI;
                    cp.nI = newImp;
                    const v2 P = scl(lambda, normal);
                    vB = add(vB, scl(mB, P)); wB += iB * crs(cp.rB, P);
                } else {
                    VCP &c1 = k.p[0], &c2 = k.p[1];
                    const v2 a = V(c1.nI, c2.nI);
                    const v2 dv1 = add(vB, crs_sv(wB, c1.rB)), dv2 = add(vB, crs_sv(wB, c2.rB));
                    float vn1 = dot(dv1, normal), vn2 = dot(dv2, normal);
                    v2 b = V(vn1 - 0.0f, vn2 - 0.0f);
                    b = sub(b, V(k.k11 * a.x + k.k12 * a.y, k.k12 * a.x + k.k22 * a.y));
                    v2 x;
                    bool solved = false;
                    x = V(-(k.n11 * b.x + k.n12 * b.y), -(k.n12 * b.x + k.n22 * b.y));
                    if (x.x >= 0.0f && x.y >= 0.0f) solved = true;
                    if (!solved) {
                        x.x = -c1.normalMass * b.x; x.y = 0.0f;
                        vn2 = k.k12 * x.x + b.y;
                        if (x.x >= 0.0f && vn2 >= 0.0f) solved = true;
                    }
                    if (!solved) {
                        x.x = 0.0f; x.y = -c2.normalMass * b.y;
                        vn1 = k.k12 * x.y + b.x;
                        if (x.y >= 0.0f && vn1 >= 0.0f) solved = true;
                    }
                    if (!solved) {
                        x.x = 0.0f; x.y = 0.0f;
                        if (b.x >= 0.0f && b.y >= 0.0f) solved = true;
                    }
                    if (solved) {
                        const v2 d = sub(x, a);
                        const v2 P1 = scl(d.x, normal), P2 = scl(d.y, normal);
                        vB = add(vB, scl(mB, add(P1, P2)));
                        wB += iB * (crs(c1.rB, P1) + crs(c2.rB, P2));
                        c1.nI = x.x; c2.nI = x.y;
                    }
                }
                st[body].v = vB; st[body].w = wB;
            }
        });
    }
    // --- StoreImpulses: rebuild the warm-start store from this step's touching contacts
    for (int s = 0; s < kSlots; s++) W.slot_key[s] = 0u;
    for (int ci = 0; ci < nvc; ci++) {
        const VC &k = vc[ci];
        W.slot_key[ci] = (uint32_t)(k.body * NF + k.edge) | ((uint32_t)(k.mPointCount + 1) << 16);
        for (int p = 0; p < 2; p++) {
            W.slot_id[ci][p] = ids[ci][p];
            // points dropped by the condition-number fallback keep the impulse they were given
            W.slot_nI[ci][p] = p < k.mPointCount ? k.p[p].nI : 0.0f;
            W.slot_tI[ci][p] = p < k.mPointCount ? k.p[p].tI : 0.0f;
        }
    }
    // --- integrate positions
    static_for<0, NB>([&](auto I) {
        constexpr int i = decltype(I)::value;
        v2 v = st[i].v;
        float w = st[i].w;
        const v2 tr = scl(dt, v);
        if (dot(tr, tr) > kMaxTranslation * kMaxTranslation) { const float ratio = kMaxTranslation / sqrtf(dot(tr, tr)); v = scl(ratio, v); }
        const float rotn = dt * w;
        if (rotn * rotn > kMaxRotation * kMaxRotation) { const float ratio = kMaxRotation / fabsf(rotn); w *= ratio; }
        st[i].c = add(st[i].c, scl(dt, v));
        st[i].a = st[i].a + dt * w;
        st[i].v = v; st[i].w = w;
    });
    // --- <= 60 position iterations
    bool positionSolved = false;
#pragma unroll 1
    for (int it = 0; it < 60; it++) {
        float minSep = 0.0f;
        if (nvc != 0)
            static_for<0, NB>([&](auto OI) {
                constexpr int oi = decltype(OI)::value, body = Scene::body_order(oi);
                const ShapeConst &sh = Scene::shape(body);
                const float mB = sh.invMass, iB = sh.invI;
                for (int ci = oi == 0 ? 0 : cend[oi == 0 ? 0 : oi - 1]; ci < cend[oi]; ci++) {
                    const VC &k = vc[ci];
                    v2 cB = st[body].c;
                    float aB = st[body].a;
                    for (int p = 0; p < k.mPointCount; p++) {
                        xform xfB;
                        xfB.q = rot_of(aB);
                        xfB.p = sub(cB, rmul(xfB.q, sh.localCenter));
                        v2 normal, point;
                        float separation;
                        if (k.mType == 0) {
                            normal = k.localNormal;
                            const v2 clip = xmul(xfB, k.lp[p]);
                            separation = dot(sub(clip, k.localPoint), normal) - kPolygonRadius - kPolygonRadius;
                            point = clip;
                        } else {
                            normal = rmul(xfB.q, k.localNormal);
                            const v2 plane = xmul(xfB, k.localPoint);
                            const v2 clip = k.lp[p];
                            separation = dot(sub(clip, plane), normal) - kPolygonRadius - kPolygonRadius;
                            point = clip;
                            normal = neg(normal);
                        }
                        const v2 rB = sub(point, cB);
                        minSep = fmin_(minSep, separation);
                        const float C = clampf(kBaumgarte * (separation + kLinearSlop), -kMaxLinearCorrection, 0.0f);
                        const float rnB = crs(rB, normal);
                        const float K = mB + iB * rnB * rnB;
                        const float impulse = K > 0.0f ? -C / K : 0.0f;
                        const v2 P = scl(impulse, normal);
                        cB = add(cB, scl(mB, P));
                        aB += iB * crs(rB, P);
                    }
                    st[body].c = cB; st[body].a = aB;
                }
            });
        const bool contactsOkay = minSep >= -3.0f * kLinearSlop;
        bool jointsOkay = true;
        static_for<0, NJ>([&](auto Q) {
            constexpr int k = Scene::joint_order(decltype(Q)::value), bA = Scene::joint_body_a(k), bB = Scene::joint_body_b(k);
            const bool ok = joint_solve_position(jn[k], Scene::jdef(k), Scene::shape(bA), Scene::shape(bB), st[bA], st[bB]);
            jointsOkay = jointsOkay && ok;
        });
        if (contactsOkay && jointsOkay) { positionSolved = true; break; }
    }
    // --- copy back, sleep management
    float minSleep = kFltMax;
    const float linTol = kLinearSleepTol * kLinearSleepTol, angTol = kAngularSleepTol * kAngularSleepTol;
    static_for<0, NJ>([&](auto K) { constexpr int k = decltype(K)::value; W.j[k] = jn[k]; });
    static_for<0, NB>([&](auto I) {
        constexpr int i = decltype(I)::value;
        Body &b = W.b[i];
        b.c0 = b.c; b.a0 = b.a;   // b2Island::Solve: "store positions for continuous collision"
        b.c = st[i].c; b.a = st[i].a; b.v = st[i].v; b.w = st[i].w;
        sync_xf(b, Scene::shape(i));
        if (b.w * b.w > angTol || dot(b.v, b.v) > linTol) { b.sleepTime = 0.0f; minSleep = 0.0f; }
        else { b.sleepTime += dt; minSleep = fmin_(minSleep, b.sleepTime); }
    });
    island_awake = true;
    if (minSleep >= kTimeToSleep && positionSolved) {
        island_awake = false;
        for (int i = 0; i < NB; i++) { W.b[i].sleepTime = 0.0f; W.b[i].v = V(0.0f, 0.0f); W.b[i].w = 0.0f; }
    }
    // --- SolveTOI: continuous collision against the static fixtures (a sleeping island is skipped)
    // (`live`: the warp's lanes that are in this call together, see solve_toi; 0 on divergent callers)
    // run_toi = false: the caller runs SolveTOI itself (deferred to the TOI kernel, see toi_needed)
    if (run_toi && (live != 0u || island_awake)) solve_toi<Scene>(W, dt, island_awake, live);
    W.flags |= kFlagStepped;
}

#undef LD
}  // namespace b2l
