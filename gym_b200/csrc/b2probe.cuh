// b2probe.cuh -- one case of a Box2D building block on packed float32 records: the dispatch behind
// b200gym_selftest_box2d (b2probe.cu) and its host build (tests/hostsim), so that the CPU suite and the device run the
// same code on the same records.  The tests compare both with float64 geometry (tests/box2d_geometry.py).
//
// Records are kProbeWords float32 words in and out.  Integer results (manifold type, point count, ray hit, TOI state,
// simplex count) are stored as float values; feature ids as their bit pattern.  Fixture f: 0 lander hull, 1 lander leg,
// 2 walker hull, 3 walker upper leg, 4 walker lower leg -- the ShapeConsts of box2d_consts.h, which the caller loads
// into lunar::kC / walker::kC as b200gym_create does.  An out-of-range fixture gives a record of NaNs.
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
    PROBE_NUM_OPS
};
// manifold record: {type, pointCount, localNormal, localPoint, pts[0].localPoint, pts[0].id, pts[1].localPoint, pts[1].id}

__device__ __forceinline__ const ShapeConst *fixture(float f) {
    if (f == 0.0f) return &lunar::kC.shape[0];
    if (f == 1.0f) return &lunar::kC.shape[1];
    if (f == 2.0f) return &walker::kC.shape[0];
    if (f == 3.0f) return &walker::kC.shape[1];
    if (f == 4.0f) return &walker::kC.shape[2];
    return nullptr;
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
    const bool shaped = op == PROBE_EDGE_POLYGON || op == PROBE_BOX_POLYGON || op == PROBE_GJK || op == PROBE_TOI;
    const ShapeConst *sh = shaped ? fixture(in[0]) : nullptr;
    if ((shaped && !sh) || op < 0 || op >= PROBE_NUM_OPS) {
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
