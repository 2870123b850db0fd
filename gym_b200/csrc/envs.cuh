// envs.cuh -- per-environment dynamics as device functions.
//
// One struct per env kind; each exposes
//   S / D / A / NACT      float64 state words, obs floats, Box action dim (0 = Discrete), #actions
//   default_bounds()      the reset() sampling bounds when no options are given
//   reset(s, g, lo, hi, obs)
//   step(s, fresh, act, param0, obs, reward, terminated)
//
// Precision contract (SURVEY.md H1/H3): the reference integrates in float64
// (Python floats / np.float64) and only casts the *returned* observation to
// float32, except where numpy >= 2 (NEP 50) keeps float32 operands in float32
// (Pendulum's torque terms, MountainCarContinuous after its first step).  These
// functions follow that dtype flow operation by operation; the translation
// unit is compiled with -fmad=false so every multiply and add rounds
// separately, as in CPython.  sin / cos are glibc's own results, bit for bit
// (glibc_trig.cuh): that is what makes the chaotic systems (Acrobot) match the
// reference over whole free-running episodes.  The one remaining difference to
// the CPU reference is x*x standing in for libm powf(x, 2.0) in Pendulum's
// float32 torque cost (0.08 % of inputs, 1 float32 ulp, reward only).
#pragma once
#include <cmath>
#include <cstdint>

#include "../../include/b200gym.h"
#include "glibc_trig.cuh"
#include "rng.cuh"

namespace bgym {

#define B200_PI 3.141592653589793

template <int KIND>
struct Env;

// np.clip(x, lo, hi) == minimum(maximum(x, lo), hi) on float64 scalars
__device__ __forceinline__ double clip64(double x, double lo, double hi) {
    const double m = (x < lo) ? lo : x;
    return (m > hi) ? hi : m;
}

// Correctly rounded IEEE-754 x / c for a constant c, without the reciprocal computation of the
// generic division routine (MUFU.RCP64H + Newton steps + fix-up, ~30 instructions): with
// rc = RN(1/c) folded at compile time, two residual-correction steps
//     q <- q + (x - q*c) * rc          (the residual x - q*c is exact in an FMA)
// land on RN(x/c) (Markstein's theorem; the second step makes the "q within 1 ulp" premise
// hold with margin).  The explicit fma() calls are not affected by -fmad=false.  Huge, tiny,
// zero and non-finite x take the generic division so that signed zeros, infinities and the
// subnormal range behave exactly like `/`.  b200gym_selftest() checks bit-equality with `/`
// on the device for billions of inputs.
__device__ __forceinline__ double div_by_const(double x, double c, double rc) {
    const double ax = fabs(x);
    if (!(ax < 1e290) || ax < 1e-290) return x / c;
    double q = x * rc;
    double r = fma(-q, c, x);
    q = fma(r, rc, q);
    r = fma(-q, c, x);
    return fma(r, rc, q);
}

// sin and cos of a small angle without range reduction.  CartPole's pole angle stays inside
// +-0.42 rad for every state that is still stepped under autoreset, so the generic sincos()
// (Cody-Waite reduction, quadrant logic, ~75 instructions of which many only materialise
// 64-bit immediates) is replaced by the two minimax kernels of the classic fdlibm
// __kernel_sin / __kernel_cos (|x| <= pi/4, < 1 ulp), evaluated with explicit FMAs and with the
// coefficients read from the constant bank.  Larger angles (plain-Env mode after termination)
// take the library path.
__constant__ double kSinCoef[6] = {-1.66666666666666324348e-01, 8.33333333332248946124e-03,
                                   -1.98412698298579493134e-04, 2.75573137070700676789e-06,
                                   -2.50507602534068634195e-08, 1.58969099521155010221e-10};
__constant__ double kCosCoef[6] = {4.16666666666666019037e-02, -1.38888888888741095749e-03,
                                   2.48015872894767294178e-05, -2.75573143513906633035e-07,
                                   2.08757232129817482790e-09, -1.13596475577881948265e-11};

// the library path of sincos_small, out of line: it only runs in plain-Env mode after termination, and inlined it
// costs the 32-register hot loop of the step kernels spill slots.  It returns both values in registers: with pointer
// out-parameters sn and cs would live in the caller's stack frame, and every step -- library path or not -- would
// store them to local memory and load cos back on the dependence chain
struct SinCos {
    double sn, cs;
};
__device__ __noinline__ SinCos sincos_library(double x) { return SinCos{gt::sin(x), gt::cos(x)}; }

__device__ __forceinline__ void sincos_small(double x, double &sn, double &cs) {
    if (fabs(x) < 0.7) {
        const double z = x * x;
        double r = kSinCoef[5];
        r = fma(r, z, kSinCoef[4]);
        r = fma(r, z, kSinCoef[3]);
        r = fma(r, z, kSinCoef[2]);
        r = fma(r, z, kSinCoef[1]);
        const double v = z * x;
        sn = fma(v, fma(z, r, kSinCoef[0]), x);
        double c = kCosCoef[5];
        c = fma(c, z, kCosCoef[4]);
        c = fma(c, z, kCosCoef[3]);
        c = fma(c, z, kCosCoef[2]);
        c = fma(c, z, kCosCoef[1]);
        c = fma(c, z, kCosCoef[0]);
        const double zr = z * c;
        // 1 - (z/2 - z*r), with the fdlibm split that keeps the subtraction exact near |x| ~ 0.3 .. 0.7
        const double qx = fabs(x) < 0.3 ? 0.0 : 0.25 * fabs(x);
        const double hz = fma(0.5, z, -qx);
        cs = (1.0 - qx) - (hz - z * zr);
    } else {
        const SinCos r = sincos_library(x);
        sn = r.sn;
        cs = r.cs;
    }
}

__constant__ double kInvTotalMass = 1.0 / (0.1 + 1.0);

// CartPole's physical constants, also kept in the constant bank (float64 immediates cost two UMOVs each)
__constant__ double kCartPole[10] = {9.8, 0.1, 0.1 + 1.0, 0.5, 0.1 * 0.5, 10.0, 0.02, 12 * 2 * B200_PI / 360, 2.4, 4.0 / 3.0};

// ---------------------------------------------------------------------------
// CartPole-v0/v1 -- gym/envs/classic_control/cartpole.py
// ---------------------------------------------------------------------------
template <>
struct Env<B200GYM_CARTPOLE> {
    static constexpr int S = 4, D = 4, A = 0, NACT = 2;

    __host__ __device__ static void default_bounds(double &lo, double &hi) {
        lo = -0.05;  // cartpole.py:199-201
        hi = 0.05;
    }

    // cartpole.py:190-207
    __device__ static void reset(double (&s)[S], Pcg64 &g, double lo, double hi, float (&obs)[D]) {
#pragma unroll
        for (int k = 0; k < 4; k++) s[k] = pcg64_uniform(g, lo, hi);  // :202 uniform(size=(4,))
#pragma unroll
        for (int k = 0; k < 4; k++) obs[k] = (float)s[k];             // :207
    }

    // the observation of the current state (cartpole.py:188), without stepping
    __device__ static void observe(const double (&s)[S], float (&obs)[D]) {
#pragma unroll
        for (int k = 0; k < 4; k++) obs[k] = (float)s[k];
    }

    // x and theta after one Euler step (cartpole.py:150, :152) and the termination test on them (:162-167).  Neither
    // depends on the action, so whether a state terminates on its next step is known before the step runs
    // (will_terminate); step() computes `terminated` through the same two functions, so the two always agree
    __device__ static void next_x_theta(const double (&s)[S], double &x, double &theta) {
        const double tau = kCartPole[6];
        x = s[0] + tau * s[1];
        theta = s[2] + tau * s[3];
    }
    __device__ static bool out_of_bounds(double x, double theta) {
        const double theta_threshold = kCartPole[7], x_threshold = kCartPole[8];
        return (x < -x_threshold) || (x > x_threshold) || (theta < -theta_threshold) || (theta > theta_threshold);
    }
    __device__ static bool will_terminate(const double (&s)[S]) {
        double x, theta;
        next_x_theta(s, x, theta);
        return out_of_bounds(x, theta);
    }

    // cartpole.py:130-188, "euler" integrator (:149-153)
    __device__ static void step(double (&s)[S], bool /*fresh*/, int action, float /*a0*/,
                                double /*param0*/, float (&obs)[D], double &reward, bool &terminated) {
        const double gravity = kCartPole[0], masspole = kCartPole[1];        // :90-92 (masscart = 1.0)
        const double total_mass = kCartPole[2];                              // :93  masspole + masscart
        const double length = kCartPole[3];                                  // :94
        const double polemass_length = kCartPole[4];                         // :95  masspole * length
        const double force_mag = kCartPole[5], tau = kCartPole[6];           // :96-97

        double x_dot = s[1], theta = s[2], theta_dot = s[3];
        const double force = (action == 1) ? force_mag : -force_mag;         // :135
        double sintheta, costheta;
        sincos_small(theta, sintheta, costheta);                             // :136-137
        const double inv_total_mass = kInvTotalMass;     // RN(1 / total_mass), folded by the compiler
        const double temp = div_by_const(
            force + polemass_length * (theta_dot * theta_dot) * sintheta, total_mass, inv_total_mass);  // :141-143
        const double thetaacc =
            (gravity * sintheta - costheta * temp) /
            (length * (kCartPole[9] - div_by_const(masspole * (costheta * costheta), total_mass,
                                                inv_total_mass)));                         // :144-146
        const double xacc = temp - div_by_const(polemass_length * thetaacc * costheta, total_mass,
                                                inv_total_mass);                           // :147
        double x;
        next_x_theta(s, x, theta);                                           // :150, :152
        x_dot = x_dot + tau * xacc;                                          // :151
        theta_dot = theta_dot + tau * thetaacc;                              // :153
        s[0] = x; s[1] = x_dot; s[2] = theta; s[3] = theta_dot;              // :160
        terminated = out_of_bounds(x, theta);                                // :162-167
        reward = 1.0;                                                        // :169-174
        obs[0] = (float)x; obs[1] = (float)x_dot; obs[2] = (float)theta; obs[3] = (float)theta_dot;  // :188
    }
};

// ---------------------------------------------------------------------------
// MountainCar-v0 -- gym/envs/classic_control/mountain_car.py
// ---------------------------------------------------------------------------
template <>
struct Env<B200GYM_MOUNTAINCAR> {
    static constexpr int S = 2, D = 2, A = 0, NACT = 3;

    __host__ __device__ static void default_bounds(double &lo, double &hi) {
        lo = -0.6;  // mountain_car.py:159
        hi = -0.4;
    }

    // mountain_car.py:150-164
    __device__ static void reset(double (&s)[S], Pcg64 &g, double lo, double hi, float (&obs)[D]) {
        s[0] = pcg64_uniform(g, lo, hi);  // :160
        s[1] = 0.0;
        obs[0] = (float)s[0];
        obs[1] = 0.0f;
    }

    __device__ static void observe(const double (&s)[S], float (&obs)[D]) { obs[0] = (float)s[0]; obs[1] = (float)s[1]; }

    // mountain_car.py:127-148
    __device__ static void step(double (&s)[S], bool /*fresh*/, int action, float /*a0*/,
                                double goal_velocity, float (&obs)[D], double &reward, bool &terminated) {
        const double min_position = -1.2, max_position = 0.6, max_speed = 0.07;
        const double goal_position = 0.5, force = 0.001, gravity = 0.0025;   // :104-111
        double position = s[0], velocity = s[1];
        velocity += (double)(action - 1) * force + gt::cos(3 * position) * (-gravity);  // :132
        velocity = clip64(velocity, -max_speed, max_speed);                  // :133
        position += velocity;                                                // :134
        position = clip64(position, min_position, max_position);             // :135
        if (position == min_position && velocity < 0) velocity = 0;          // :136-137
        terminated = (position >= goal_position) && (velocity >= goal_velocity);  // :139-141
        reward = -1.0;                                                       // :142
        s[0] = position; s[1] = velocity;                                    // :144
        obs[0] = (float)position; obs[1] = (float)velocity;                  // :148
    }
};

// ---------------------------------------------------------------------------
// MountainCarContinuous-v0 -- continuous_mountain_car.py:142-186
//
// Under numpy >= 2 `self.state` is a float64 array only between reset (:182)
// and the first step; afterwards it is the float32 array built at :171, so the
// arithmetic runs in float32 against "weak" Python constants (SURVEY.md A.3).
// `fresh` (TimeLimit counter == 0) selects the dtype position/velocity have.
// The HBM state is float64 in both cases (a float32 value is exact in it).
// ---------------------------------------------------------------------------
template <>
struct Env<B200GYM_MOUNTAINCAR_CONT> {
    static constexpr int S = 2, D = 2, A = 1, NACT = 0;

    __host__ __device__ static void default_bounds(double &lo, double &hi) {
        lo = -0.6;  // continuous_mountain_car.py:181
        hi = -0.4;
    }

    __device__ static void reset(double (&s)[S], Pcg64 &g, double lo, double hi, float (&obs)[D]) {
        s[0] = pcg64_uniform(g, lo, hi);  // :182
        s[1] = 0.0;
        obs[0] = (float)s[0];
        obs[1] = 0.0f;
    }

    __device__ static void observe(const double (&s)[S], float (&obs)[D]) { obs[0] = (float)s[0]; obs[1] = (float)s[1]; }

    __device__ static void step(double (&s)[S], bool fresh, int /*action*/, float a0,
                                double goal_velocity, float (&obs)[D], double &reward, bool &terminated) {
        const double min_action = -1.0, max_action = 1.0, min_position = -1.2, max_position = 0.6;
        const double max_speed = 0.07, goal_position = 0.45, power = 0.0015;  // :110-119
        // a Python float meeting a numpy scalar is first rounded to that scalar's dtype
        auto T = [fresh](double c) { return fresh ? c : (double)(float)c; };
        double position = s[0], velocity = s[1];  // :144-145
        bool vel_py = false, pos_py = false;      // the value became a plain Python number

        // :146 min(max(action[0], -1.0), 1.0) returns the Python constant only when it clips
        bool force_py = false;
        double force_c = 0.0;
        if (a0 < (float)min_action) { force_py = true; force_c = min_action; }
        else if (a0 > (float)max_action) { force_py = true; force_c = max_action; }

        // :148 velocity += force * power - 0.0025 * math.cos(3 * position)
        const double three_p = fresh ? 3 * position : (double)(3.0f * (float)position);
        const double c = 0.0025 * gt::cos(three_p);
        if (force_py) {
            const double inc = force_c * power - c;
            velocity = fresh ? velocity + inc : (double)((float)velocity + (float)inc);
        } else {
            const float inc = a0 * (float)power - (float)c;
            velocity = fresh ? velocity + (double)inc : (double)((float)velocity + inc);
        }
        if (velocity > T(max_speed)) { velocity = max_speed; vel_py = true; }               // :149-150
        if (vel_py ? (velocity < -max_speed) : (velocity < T(-max_speed))) {                // :151-152
            velocity = -max_speed; vel_py = true;
        }
        position = fresh ? position + velocity : (double)((float)position + (float)velocity);  // :153
        if (position > T(max_position)) { position = max_position; pos_py = true; }         // :154-155
        if (pos_py ? (position < min_position) : (position < T(min_position))) {            // :156-157
            position = min_position; pos_py = true;
        }
        const bool at_min = pos_py ? (position == min_position) : (position == T(min_position));
        if (at_min && velocity < 0) { velocity = 0; vel_py = true; }                        // :158-159

        const bool pos_ok = pos_py ? (position >= goal_position) : (position >= T(goal_position));
        const bool vel_ok = vel_py ? (velocity >= goal_velocity) : (velocity >= T(goal_velocity));
        terminated = pos_ok && vel_ok;                                                      // :162-164
        double r = terminated ? 100.0 : 0.0;                                                // :166-168
        const double a0d = (double)a0;
        r -= gt::sq(a0d) * 0.1;                                                             // :169 math.pow(action[0], 2) * 0.1
        reward = r;
        const float pf = (float)position, vf = (float)velocity;                             // :171 dtype=np.float32
        s[0] = (double)pf; s[1] = (double)vf;
        obs[0] = pf; obs[1] = vf;                                                           // :175
    }
};

// ---------------------------------------------------------------------------
// Pendulum-v1 -- gym/envs/classic_control/pendulum.py
// ---------------------------------------------------------------------------
template <>
struct Env<B200GYM_PENDULUM> {
    static constexpr int S = 2, D = 3, A = 1, NACT = 0;

    __host__ __device__ static void default_bounds(double &x_init, double &y_init) {
        x_init = B200_PI;  // pendulum.py:14-15 DEFAULT_X, DEFAULT_Y
        y_init = 1.0;
    }

    // pendulum.py:161-163
    __device__ static void get_obs(const double (&s)[S], float (&obs)[D]) {
        const double sn = gt::sin(s[0]), cs = gt::cos(s[0]);
        obs[0] = (float)cs; obs[1] = (float)sn; obs[2] = (float)s[1];
    }

    __device__ static void observe(const double (&s)[S], float (&obs)[D]) { get_obs(s, obs); }

    // pendulum.py:141-159: uniform(low=-high, high=high) with high = [x_init, y_init]
    __device__ static void reset(double (&s)[S], Pcg64 &g, double x_init, double y_init, float (&obs)[D]) {
        s[0] = pcg64_uniform(g, -x_init, x_init);
        s[1] = pcg64_uniform(g, -y_init, y_init);
        get_obs(s, obs);
    }

    // Python-style float modulo, as numpy evaluates `%` on float64 scalars
    __device__ static double py_mod(double a, double b) {
        double m = fmod(a, b);
        if (m != 0.0) {
            if ((b < 0) != (m < 0)) m += b;
        } else {
            m = copysign(0.0, b);
        }
        return m;
    }

    // pendulum.py:119-139
    __device__ static void step(double (&s)[S], bool /*fresh*/, int /*action*/, float a0, double g,
                                float (&obs)[D], double &reward, bool &terminated) {
        const double max_speed = 8, dt = 0.05, m = 1.0, l = 1.0;  // :96-101
        const float max_torque = 2.0f;
        const double th = s[0], thdot = s[1];
        // :127 u = np.clip(u, -2, 2)[0] -> np.float32
        float u = (a0 < -max_torque) ? -max_torque : a0;
        u = (u > max_torque) ? max_torque : u;
        // :129 costs = angle_normalize(th)**2 + .1*thdot**2 + .001*(u**2); the u term is float32
        const double an = py_mod(th + B200_PI, 2 * B200_PI) - B200_PI;  // :270-271
        const float u_term = (float)0.001 * (u * u);
        const double costs = gt::sq(an) + 0.1 * gt::sq(thdot) + (double)u_term;   // np.float64 ** 2 = libm pow
        // :131 3.0/(m*l**2)*u is float32 and is promoted by the add
        const float tq = (float)(3.0 / (m * (l * l))) * u;
        double newthdot = thdot + (3 * g / (2 * l) * gt::sin(th) + (double)tq) * dt;
        newthdot = clip64(newthdot, -max_speed, max_speed);  // :132
        const double newth = th + newthdot * dt;             // :133
        s[0] = newth; s[1] = newthdot;                       // :135
        get_obs(s, obs);
        reward = -costs;                                     // :139
        terminated = false;
    }
};

// ---------------------------------------------------------------------------
// Acrobot-v1 -- gym/envs/classic_control/acrobot.py
// ---------------------------------------------------------------------------
template <>
struct Env<B200GYM_ACROBOT> {
    static constexpr int S = 4, D = 6, A = 0, NACT = 3;

    __host__ __device__ static void default_bounds(double &lo, double &hi) {
        lo = -0.1;  // acrobot.py:185-187
        hi = 0.1;
    }

    // acrobot.py:225-230
    __device__ static void get_obs(const double (&s)[S], float (&obs)[D], double &cos0) {
        const double s0 = gt::sin(s[0]), c0 = gt::cos(s[0]), s1 = gt::sin(s[1]), c1 = gt::cos(s[1]);
        obs[0] = (float)c0; obs[1] = (float)s0; obs[2] = (float)c1; obs[3] = (float)s1;
        obs[4] = (float)s[2]; obs[5] = (float)s[3];
        cos0 = c0;
    }

    __device__ static void observe(const double (&s)[S], float (&obs)[D]) { double c0; get_obs(s, obs, c0); }

    // acrobot.py:181-194: uniform(size=(4,)).astype(np.float32); the reference then
    // evaluates numpy's float32 cos/sin on it -- we return the correctly rounded
    // float32 of the float64 result (<= 1 float32 ulp from numpy's kernel; reset
    // observations never feed the dynamics).
    __device__ static void reset(double (&s)[S], Pcg64 &g, double lo, double hi, float (&obs)[D]) {
#pragma unroll
        for (int k = 0; k < 4; k++) s[k] = (double)(float)pcg64_uniform(g, lo, hi);  // :188-190
        double c0;
        get_obs(s, obs, c0);
    }

    // acrobot.py:237-277, "book" branch (:271-276); y = (theta1, theta2, dtheta1, dtheta2), a = torque
    __device__ static void dsdt(const double (&y)[4], double a, double (&k)[4]) {
        const double m1 = 1.0, m2 = 1.0, l1 = 1.0, lc1 = 0.5, lc2 = 0.5, I1 = 1.0, I2 = 1.0;  // :145-151
        const double g = 9.8;                                                                // :245
        const double theta1 = y[0], theta2 = y[1], dtheta1 = y[2], dtheta2 = y[3];
        const double sin2 = gt::sin(theta2), cos2 = gt::cos(theta2);
        const double d1 = m1 * (lc1 * lc1) + m2 * ((l1 * l1) + (lc2 * lc2) + 2 * l1 * lc2 * cos2) + I1 + I2;  // :252-257
        const double d2 = m2 * ((lc2 * lc2) + l1 * lc2 * cos2) + I2;                          // :258
        const double phi2 = m2 * lc2 * g * gt::cos(theta1 + theta2 - B200_PI / 2.0);             // :259
        const double phi1 = -m2 * l1 * lc2 * gt::sq(dtheta2) * sin2
                            - 2 * m2 * l1 * lc2 * dtheta2 * dtheta1 * sin2
                            + (m1 * lc1 + m2 * l1) * g * gt::cos(theta1 - B200_PI / 2)
                            + phi2;                                                          // :260-265
        const double ddtheta2 =
            (a + d2 / d1 * phi1 - m2 * l1 * lc2 * gt::sq(dtheta1) * sin2 - phi2) /
            (m2 * (lc2 * lc2) + I2 - gt::sq(d2) / d1);      // x**2 = libm pow(x, 2.0)                                         // :273-275
        const double ddtheta1 = -(d2 * ddtheta2 + phi1) / d1;                                // :276
        k[0] = dtheta1; k[1] = dtheta2; k[2] = ddtheta1; k[3] = ddtheta2;                    // :277
    }

    // acrobot.py:378-396
    __device__ static double wrap(double x, double m, double M) {
        const double diff = M - m;
        while (x > M) x = x - diff;
        while (x < m) x = x + diff;
        return x;
    }

    // acrobot.py:196-223 with rk4 (:418-465) over t = [0, 0.2]
    __device__ static void step(double (&s)[S], bool /*fresh*/, int action, float /*a0*/,
                                double /*param0*/, float (&obs)[D], double &reward, bool &terminated) {
        const double MAX_VEL_1 = 4 * B200_PI, MAX_VEL_2 = 9 * B200_PI;  // :153-154
        const double dt = 0.2, dt2 = dt / 2.0;                          // :453-455
        const double torque = (double)(action - 1);                     // :156 AVAIL_TORQUE[a]
        double y0[4] = {s[0], s[1], s[2], s[3]};
        double k1[4], k2[4], k3[4], k4[4], y[4];
        dsdt(y0, torque, k1);                                           // :458
#pragma unroll
        for (int i = 0; i < 4; i++) y[i] = y0[i] + dt2 * k1[i];
        dsdt(y, torque, k2);                                            // :459
#pragma unroll
        for (int i = 0; i < 4; i++) y[i] = y0[i] + dt2 * k2[i];
        dsdt(y, torque, k3);                                            // :460
#pragma unroll
        for (int i = 0; i < 4; i++) y[i] = y0[i] + dt * k3[i];
        dsdt(y, torque, k4);                                            // :461
        double ns[4];
#pragma unroll
        for (int i = 0; i < 4; i++)
            ns[i] = y0[i] + dt / 6.0 * (k1[i] + 2 * k2[i] + 2 * k3[i] + k4[i]);  // :462
        ns[0] = wrap(ns[0], -B200_PI, B200_PI);                         // :213-214
        ns[1] = wrap(ns[1], -B200_PI, B200_PI);
        ns[2] = fmin(fmax(ns[2], -MAX_VEL_1), MAX_VEL_1);               // :215-216 bound()
        ns[3] = fmin(fmax(ns[3], -MAX_VEL_2), MAX_VEL_2);
#pragma unroll
        for (int i = 0; i < 4; i++) s[i] = ns[i];                       // :217
        double cos0;
        get_obs(s, obs, cos0);
        terminated = (-cos0 - gt::cos(s[1] + s[0]) > 1.0);                  // :235
        reward = terminated ? 0.0 : -1.0;                               // :219
    }
};

}  // namespace bgym
