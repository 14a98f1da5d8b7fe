// mpc_core.h -- host/device core of the sm_90a solver: workspace layout and the reference restatement of the
// elementary OCP functions.  Everything here is `__host__ __device__` so that tests/emu can run the SAME code on a
// CPU warp emulator (test infrastructure); the product only ever runs it inside the CUDA kernels of mpcb200.cu.
//
// Reference files restated here (R/ = mpc_local_planner/ in rst-tu-dortmund/mpc_local_planner):
//   normalize_theta / interpolate_angle   R/include/mpc_local_planner/utils/math_utils.h:81-103
//   robot dynamics                        R/include/mpc_local_planner/systems/{unicycle_robot.h:59-68,simple_car.h:68-77,131-141,
//                                          kinematic_bicycle_model.h:65-77}
//   footprint distances                   teb_local_planner RobotFootprintModel::calculateDistance semantics (SURVEY App. B.3),
//                                          used at R/src/optimal_control/stage_inequality_se2.cpp:109,173
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define HD __host__ __device__
#define NOINL __noinline__   /* big leaf functions are real functions on the device: the solve kernel is bound by instruction fetch */
#else
#define HD
#define NOINL
#endif

#include "../../include/mpcb200.h"

#define KW MPCB200_KKT_WORDS
#define MAXSEG (MPCB200_MAX_POLY + 2)

// ---- per-instance workspace layout (doubles).  Every array field is [component][k], k fastest, so that the
//      lanes of the warp that owns the instance touch consecutive addresses (stage-contiguous, coalesced). ----
struct WsLayout
{
    int N, K, RS, M, V;      // grid points, obstacle rows per stage, row slots, max obstacles, max via-points
    int64_t stride;          // doubles per instance (multiple of 16 -> 128-byte aligned blocks)
    int oX, oU, oNU, oS, oLAM, oSTEP, oOBS, oSCAL, oDS, oVPST, oSTATE_END;
    int oR0, oOG;            // row residuals at the current point (RS x N), obstacle row value + gradient (4K x N)
    int oKKT, oMM;           // condensed KKT stage records [k][RSTR]; stage matrices + gains of the KKT sweep [k][MSTR]
    int oIN;                 // x0(3) xf(3) u_prev(2) n_obst n_vp has_xinit reinit
    int oOBST, oOTYPE, oVP, oXINIT, oOGIDX;
};
#define IN_X0 0
#define IN_XF 3
#define IN_UPREV 6
#define IN_NOBST 8
#define IN_NVP 9
#define IN_HASXINIT 10
#define IN_REINIT 11
#define IN_NRES 12         /* obstacles in the resident list (= IN_NOBST unless the list stays in global memory) */
#define IN_WORDS 16

// solver constants (same values as the oracle)
#define KAPPA_EPS 10.0
#define KAPPA_MU 0.2
#define THETA_MU 1.5
#define TAU_MIN 0.99
#define SLACK_PUSH 1e-2
#define ARMIJO 1e-4
#define MAX_BACKTRACK 3
#define MAX_INERTIA_TRIES 2      // factorisations per IPM iteration (escalation resumes in the next iteration: a retry of one lane stalls its whole launch)
#define MAX_DELTA 1e8
#define DELTA_FLOOR 1e-5
// Clipped slack steps (see the oracle, ORC_CLIP_*): the rows that block the step most -- at most 1/CLIP_DIV of the rows, in
// whole sqrt(2)-wide bins of their step ratio -- are excluded from the fraction-to-the-boundary rule; their slacks are clipped.
#define CLIP_DIV 8
#define CLIP_FLOOR 0.01
#define CLIP_BINS 40
#define TINY_STEP 1e-8
#define TINY_STEP_COUNT 2
#define KAPPA_SIGMA 1e10
#define SMAX 100.0
#define PROJ_MARGIN 0.05
#define PROJ_SWEEPS 6
#define INIT_SHRINK 0.9

typedef mpcb200_config Cfg;

// ---- config predicates ----
HD inline bool xf_all_fixed(const Cfg& c) { return c.xf_fixed[0] && c.xf_fixed[1] && c.xf_fixed[2]; }
HD inline bool has_quadratic(const Cfg& c) { return c.objective == MPCB200_OBJ_QUADRATIC_FORM; }
HD inline bool is_midpoint(const Cfg& c) { return c.collocation == MPCB200_COLLOC_MIDPOINT; }
// quadratic_form/hybrid_cost_minimum_time (src/controller.cpp:595-620): honoured only for zero state weights and non-zero
// control weights (corbo::MinTimeQuadraticControls: dt per interval + the quadratic control term); otherwise the reference
// logs an error and falls back to the plain quadratic form
HD inline bool has_hybrid_mintime(const Cfg& c)
{
    if (!c.hybrid_cost_minimum_time || c.objective != MPCB200_OBJ_QUADRATIC_FORM) return false;
    bool qz = true, rz = true;
    for (int i = 0; i < 9; ++i) qz = qz && c.Q[i] == 0.0;
    for (int i = 0; i < 4; ++i) rz = rz && c.R[i] == 0.0;
    return qz && !rz;
}
HD inline bool has_mintime(const Cfg& c)
{
    return c.objective == MPCB200_OBJ_MINIMUM_TIME || c.objective == MPCB200_OBJ_MINIMUM_TIME_VIA_POINTS || has_hybrid_mintime(c);
}
HD inline bool has_viapoints(const Cfg& c)
{
    return c.objective == MPCB200_OBJ_MINIMUM_TIME_VIA_POINTS ||
           (c.objective == MPCB200_OBJ_QUADRATIC_FORM && c.vp_attraction_with_quadratic);
}
HD inline bool has_terminal_cost(const Cfg& c) { return c.terminal_cost && !xf_all_fixed(c); }
// Integral form of the quadratic running cost (quadratic_cost_se2.cpp:54-84 through corbo's LeftSumCostEdge /
// TrapezoidalIntegralCostEdge, finite_differences_grid_se2.cpp:57-72): the state term of stage k enters with weight
// dt * integral_state_weight -- left sum 1 for k <= N-2 and 0 at k = N-1; trapezoidal rule 1/2 at both ends, 1 between --
// the control term of interval k with weight dt in both rules (both ends of the trapezoid use u_k).
HD inline bool has_trapezoid(const Cfg& c)
{ return has_quadratic(c) && c.quadratic_integral_form != 0 && c.cost_integration == MPCB200_COST_TRAPEZOIDAL; }
HD inline double integral_state_weight(const Cfg& c, int N, int k)
{
    if (c.cost_integration == MPCB200_COST_TRAPEZOIDAL) return (k == 0 || k == N - 1) ? 0.5 : 1.0;
    return k <= N - 2 ? 1.0 : 0.0;
}
#define BALL_SLOT 2
HD inline bool ball_active(const Cfg& c) { return c.terminal_ball != 0 && !xf_all_fixed(c); }
// the control row of linear row slot 0..7 (u_lb0, u_ub0, u_lb1, u_ub1, du_lb0, du_ub0, du_lb1, du_ub1) has a finite bound
HD inline bool control_row_finite(const Cfg& c, int slot)
{
    if (slot < 4) { const int i = slot >> 1; return (slot & 1) ? (c.u_ub[i] < MPCB200_INF) : (c.u_lb[i] > -MPCB200_INF); }
    const int i = (slot - 4) >> 1;
    return ((slot - 4) & 1) ? (c.du_ub[i] < MPCB200_INF) : (c.du_lb[i] > -MPCB200_INF);
}

// ---- per-robot limits (mpcb200_set_robot_limits): a record of MPCB200_LIMIT_WORDS doubles in place of nine config values ----
// A record may change values, never the row set: each of the eight control rows is finite in the record exactly where it is in
// `c` (the kernel variant and the fixed-dt key are chosen from `c`), the rule of mpcb200_create (u_ub > u_lb) holds, no word is
// NaN and the clearance is finite and >= 0.  The blocking setter checks every record with this on the host, the solve kernel
// checks the record of each robot with it in the instance's prologue.
HD inline bool robot_limits_valid(const Cfg& c, const double* r)
{
    for (int w = 0; w < MPCB200_LIMIT_WORDS; ++w)
        if (r[w] != r[w]) return false;
    for (int i = 0; i < 2; ++i)
    {
        if (!(r[MPCB200_LIM_U_UB + i] > r[MPCB200_LIM_U_LB + i])) return false;
        if ((r[MPCB200_LIM_U_LB + i] > -MPCB200_INF) != control_row_finite(c, 2 * i)) return false;
        if ((r[MPCB200_LIM_U_UB + i] < MPCB200_INF) != control_row_finite(c, 2 * i + 1)) return false;
        if ((r[MPCB200_LIM_DU_LB + i] > -MPCB200_INF) != control_row_finite(c, 4 + 2 * i)) return false;
        if ((r[MPCB200_LIM_DU_UB + i] < MPCB200_INF) != control_row_finite(c, 5 + 2 * i)) return false;
    }
    const double d = r[MPCB200_LIM_MIN_OBSTACLE_DIST];
    return d >= 0.0 && d <= 1.7976931348623157e308;
}
// the configuration of a robot: its record's nine values in place of the configuration's, every other field untouched
HD inline void apply_robot_limits(Cfg& c, const double* r)
{
    for (int i = 0; i < 2; ++i)
    {
        c.u_lb[i] = r[MPCB200_LIM_U_LB + i];
        c.u_ub[i] = r[MPCB200_LIM_U_UB + i];
        c.du_lb[i] = r[MPCB200_LIM_DU_LB + i];
        c.du_ub[i] = r[MPCB200_LIM_DU_UB + i];
    }
    c.min_obstacle_dist = r[MPCB200_LIM_MIN_OBSTACLE_DIST];
}

// ---- per-robot geometry (mpcb200_set_robot_geometry): a record of MPCB200_GEOMETRY_WORDS doubles ----
// robot_type and footprint_type stay the handle's (unless model records are set: robot_model_valid); a record supplies the values
// those two types read and nothing else, so the
// check and the patch look at exactly those words (the others may hold anything, NaN included).  The blocking setter checks every
// record with this on the host, the solve kernel checks the record of each robot with it in the instance's prologue.
HD inline bool geo_finite(double v) { return v >= -1.7976931348623157e308 && v <= 1.7976931348623157e308; }
HD inline bool robot_geometry_valid(const Cfg& c, const double* r)
{
    switch (c.robot_type)
    {
        case MPCB200_ROBOT_SIMPLE_CAR:
        case MPCB200_ROBOT_SIMPLE_CAR_FRONT:
            if (!(geo_finite(r[MPCB200_GEO_WHEELBASE]) && r[MPCB200_GEO_WHEELBASE] > 0.0)) return false;
            break;
        case MPCB200_ROBOT_KIN_BICYCLE:
            if (!(geo_finite(r[MPCB200_GEO_LENGTH_REAR]) && r[MPCB200_GEO_LENGTH_REAR] > 0.0)) return false;
            if (!(geo_finite(r[MPCB200_GEO_LENGTH_FRONT]) && r[MPCB200_GEO_LENGTH_FRONT] >= 0.0)) return false;
            break;
        default: break;
    }
    const double* f = r + MPCB200_GEO_FOOTPRINT;
    switch (c.footprint_type)
    {
        case MPCB200_FOOTPRINT_CIRCULAR: return geo_finite(f[0]) && f[0] >= 0.0;
        case MPCB200_FOOTPRINT_TWO_CIRCLES:   // front offset, front radius, rear offset, rear radius
            return geo_finite(f[0]) && geo_finite(f[2]) && geo_finite(f[1]) && f[1] >= 0.0 && geo_finite(f[3]) && f[3] >= 0.0;
        case MPCB200_FOOTPRINT_LINE: return geo_finite(f[0]) && geo_finite(f[1]) && geo_finite(f[2]) && geo_finite(f[3]);
        case MPCB200_FOOTPRINT_POLYGON:
        {
            const double np = r[MPCB200_GEO_N_POLY];
            if (!(np >= 1.0 && np <= (double)MPCB200_MAX_POLY) || np != floor(np)) return false;
            for (int i = 0; i < 2 * (int)np; ++i)
                if (!geo_finite(r[MPCB200_GEO_POLY_XY + i])) return false;
            return true;
        }
        default: return true;
    }
}
// the configuration of a robot: the record's values of the fields its robot and footprint types read, every other field untouched
// (polygon vertices past n_poly included: nothing reads them)
HD inline void apply_robot_geometry(Cfg& c, const double* r)
{
    switch (c.robot_type)
    {
        case MPCB200_ROBOT_SIMPLE_CAR:
        case MPCB200_ROBOT_SIMPLE_CAR_FRONT: c.wheelbase = r[MPCB200_GEO_WHEELBASE]; break;
        case MPCB200_ROBOT_KIN_BICYCLE:
            c.length_rear = r[MPCB200_GEO_LENGTH_REAR];
            c.length_front = r[MPCB200_GEO_LENGTH_FRONT];
            break;
        default: break;
    }
    switch (c.footprint_type)
    {
        case MPCB200_FOOTPRINT_CIRCULAR: c.footprint_params[0] = r[MPCB200_GEO_FOOTPRINT]; break;
        case MPCB200_FOOTPRINT_TWO_CIRCLES:
        case MPCB200_FOOTPRINT_LINE:
            for (int i = 0; i < 4; ++i) c.footprint_params[i] = r[MPCB200_GEO_FOOTPRINT + i];
            break;
        case MPCB200_FOOTPRINT_POLYGON:
            c.n_poly = (int)r[MPCB200_GEO_N_POLY];
            for (int i = 0; i < 2 * c.n_poly; ++i) c.poly_xy[i] = r[MPCB200_GEO_POLY_XY + i];
            break;
        default: break;
    }
}
// a handle whose robot and footprint types read no geometry word (a unicycle with a point footprint): nothing to vary
HD inline bool reads_geometry(const Cfg& c)
{
    return c.robot_type != MPCB200_ROBOT_UNICYCLE || c.footprint_type != MPCB200_FOOTPRINT_POINT;
}

// ---- per-robot model (mpcb200_set_robot_model): a record of MPCB200_MODEL_WORDS doubles, robot_type and footprint_type ----
// A record changes the two types and nothing else: the row set, the objective, the grid and the kernel variant stay the handle's, and
// the solve runs the MODEL_GENERIC key, which reads both types from the configuration.  A record is valid when both words are
// integers in range (-0 is 0) and the geometry the robot uses is valid for its types (robot_geometry_valid on the configuration
// patched with the record's types): its geometry record `geo` when geometry records are set, else the configuration's own values
// as a record holds them (geometry_record_of).  The blocking setters check every record with this on the host, the solve kernel
// checks the record of each robot with it in the instance's prologue.

// the record holding a configuration's own geometry values in every word (what apply_robot_geometry writes back unchanged)
HD inline void geometry_record_of(const Cfg& c, double* r)
{
    r[MPCB200_GEO_WHEELBASE] = c.wheelbase;
    r[MPCB200_GEO_LENGTH_REAR] = c.length_rear;
    r[MPCB200_GEO_LENGTH_FRONT] = c.length_front;
    for (int i = 0; i < 4; ++i) r[MPCB200_GEO_FOOTPRINT + i] = c.footprint_params[i];
    r[MPCB200_GEO_N_POLY] = (double)c.n_poly;
    for (int i = 0; i < 2 * MPCB200_MAX_POLY; ++i) r[MPCB200_GEO_POLY_XY + i] = c.poly_xy[i];
}
HD inline bool model_word_valid(double v, int max) { return v >= 0.0 && v <= (double)max && v == floor(v); }
// the configuration of a robot: the record's two types, every other field untouched
HD inline void apply_robot_model(Cfg& c, const double* m)
{
    c.robot_type = (int)m[MPCB200_MOD_ROBOT_TYPE];
    c.footprint_type = (int)m[MPCB200_MOD_FOOTPRINT_TYPE];
}
HD inline bool robot_model_valid(const Cfg& c0, const double* m, const double* geo)
{
    if (!model_word_valid(m[MPCB200_MOD_ROBOT_TYPE], MPCB200_ROBOT_KIN_BICYCLE) ||
        !model_word_valid(m[MPCB200_MOD_FOOTPRINT_TYPE], MPCB200_FOOTPRINT_POLYGON))
        return false;
    Cfg t = c0;   // (robot_geometry_valid reads the two types of t and nothing else)
    apply_robot_model(t, m);
    if (geo) return robot_geometry_valid(t, geo);
    double r[MPCB200_GEOMETRY_WORDS];
    geometry_record_of(c0, r);
    return robot_geometry_valid(t, r);
}

// ---- per-robot weights (mpcb200_set_robot_weights): a record of MPCB200_WEIGHT_WORDS doubles ----
// The objective, the terminal-cost switch and the via-point mode stay the handle's; a record supplies the weights the handle's
// objective reads (Q and R for the quadratic form, Qf with a terminal cost, the two via-point weights with via-points) and nothing
// else, so the check and the patch look at exactly those words (the others may hold anything, NaN included).  The hybrid
// minimum-time term is on for a quadratic form of zero Q and non-zero R (has_hybrid_mintime): a record keeps it as the handle has
// it, so has_mintime, the kernel variant and key, and the variable_dt rule of mpcb200_create hold for every robot.  No definiteness
// test: mpcb200_create makes none either.  The blocking setter checks every record with this on the host, the solve kernel checks
// the record of each robot with it in the instance's prologue.
HD inline bool reads_weights(const Cfg& c) { return has_quadratic(c) || has_terminal_cost(c) || has_viapoints(c); }
HD inline bool robot_weights_valid(const Cfg& c, const double* r)
{
    if (has_quadratic(c))
    {
        bool qz = true, rz = true;
        for (int i = 0; i < 9; ++i) { if (!geo_finite(r[MPCB200_WGT_Q + i])) return false; qz = qz && r[MPCB200_WGT_Q + i] == 0.0; }
        for (int i = 0; i < 4; ++i) { if (!geo_finite(r[MPCB200_WGT_R + i])) return false; rz = rz && r[MPCB200_WGT_R + i] == 0.0; }
        if ((c.hybrid_cost_minimum_time && qz && !rz) != has_hybrid_mintime(c)) return false;
    }
    if (has_terminal_cost(c))
        for (int i = 0; i < 9; ++i)
            if (!geo_finite(r[MPCB200_WGT_QF + i])) return false;
    if (has_viapoints(c) && !(geo_finite(r[MPCB200_WGT_VP_POSITION]) && geo_finite(r[MPCB200_WGT_VP_ORIENTATION]))) return false;
    return true;
}
// the configuration of a robot: the record's values of the weights its objective reads, every other field untouched
HD inline void apply_robot_weights(Cfg& c, const double* r)
{
    if (has_quadratic(c))
    {
        for (int i = 0; i < 9; ++i) c.Q[i] = r[MPCB200_WGT_Q + i];
        for (int i = 0; i < 4; ++i) c.R[i] = r[MPCB200_WGT_R + i];
    }
    if (has_terminal_cost(c))
        for (int i = 0; i < 9; ++i) c.Qf[i] = r[MPCB200_WGT_QF + i];
    if (has_viapoints(c))
    {
        c.vp_position_weight = r[MPCB200_WGT_VP_POSITION];
        c.vp_orientation_weight = r[MPCB200_WGT_VP_ORIENTATION];
    }
}

// ---- model / problem key of a kernel variant ----
// MODEL_GENERIC reads the robot and footprint model from the configuration at run time.  MODEL_UNI_POINT is compiled for the
// unicycle with a point footprint (the BASELINE configurations 2, 4 and 5): the tests of the two fields fold at compile time and the
// code of the other models is not part of the solve kernel, whose iteration is bound by instruction fetch (DESIGN.md section 4).
// MODEL_UNI_POINT_QF is MODEL_UNI_POINT for the fixed-dt quadratic-form problem of those configurations (qf_key_matches): no dt
// terms, no integral form or minimum-time term, no terminal ball, all eight control rows present.  Via-points and the terminal cost
// stay run-time tests.  The two other keys answer the problem questions from the configuration.  The C ABI reports this key as the
// pair (MPCB200_MODEL_UNI_POINT, MPCB200_PROBLEM_FIXED_DT_QF): model_key_of / problem_key_of.
#define MODEL_GENERIC MPCB200_MODEL_GENERIC
#define MODEL_UNI_POINT MPCB200_MODEL_UNI_POINT
#define MODEL_UNI_POINT_QF 2
HD inline int model_key_of(int key) { return key == MODEL_UNI_POINT_QF ? MPCB200_MODEL_UNI_POINT : key; }
HD inline int problem_key_of(int key) { return key == MODEL_UNI_POINT_QF ? MPCB200_PROBLEM_FIXED_DT_QF : MPCB200_PROBLEM_GENERIC; }
template <int MODEL> struct ModelTraits
{
    HD static int robot(const Cfg& c) { return c.robot_type; }
    HD static int footprint(const Cfg& c) { return c.footprint_type; }
    static constexpr bool DT_TERMS = true;   // the code carries the terms of a free dt (whether dt is free: variable_dt)
    HD static bool variable_dt(const Cfg& c) { return c.variable_dt != 0; }
    HD static bool quadratic(const Cfg& c) { return has_quadratic(c); }
    HD static bool integral(const Cfg& c) { return c.quadratic_integral_form != 0; }
    HD static bool trapezoid(const Cfg& c) { return has_trapezoid(c); }
    HD static bool mintime(const Cfg& c) { return has_mintime(c); }
    HD static bool ball(const Cfg& c) { return ball_active(c); }
    HD static bool row_finite(const Cfg& c, int slot) { return control_row_finite(c, slot); }
};
template <> struct ModelTraits<MODEL_UNI_POINT> : ModelTraits<MODEL_GENERIC>
{
    HD static constexpr int robot(const Cfg&) { return MPCB200_ROBOT_UNICYCLE; }
    HD static constexpr int footprint(const Cfg&) { return MPCB200_FOOTPRINT_POINT; }
};
template <> struct ModelTraits<MODEL_UNI_POINT_QF> : ModelTraits<MODEL_UNI_POINT>
{
    static constexpr bool DT_TERMS = false;
    HD static constexpr bool variable_dt(const Cfg&) { return false; }
    HD static constexpr bool quadratic(const Cfg&) { return true; }
    HD static constexpr bool integral(const Cfg&) { return false; }
    HD static constexpr bool trapezoid(const Cfg&) { return false; }
    HD static constexpr bool mintime(const Cfg&) { return false; }
    HD static constexpr bool ball(const Cfg&) { return false; }
    HD static constexpr bool row_finite(const Cfg&, int) { return true; }
};
// the configuration is the problem MODEL_UNI_POINT_QF is compiled for (the unbordered KKT included: no free dt, no fixed final
// state component).  Line / moving obstacles and midpoint differences are a property of the launch (LINES) and tested there.
HD inline bool qf_key_matches(const Cfg& c)
{
    bool rows = true;
    for (int sl = 0; sl < 8; ++sl) rows = rows && control_row_finite(c, sl);
    return c.robot_type == MPCB200_ROBOT_UNICYCLE && c.footprint_type == MPCB200_FOOTPRINT_POINT && !c.variable_dt &&
           !c.xf_fixed[0] && !c.xf_fixed[1] && !c.xf_fixed[2] && has_quadratic(c) && !c.quadratic_integral_form && !has_mintime(c) &&
           !ball_active(c) && rows;
}

// ---- elementary functions ----
HD NOINL inline double normalize_theta_wrap(double theta)
{
    const double PI = 3.14159265358979323846;
    double multiplier = floor(theta / (2.0 * PI));
    theta = theta - multiplier * 2.0 * PI;
    if (theta >= PI) theta -= 2.0 * PI;
    if (theta < -PI) theta += 2.0 * PI;
    return theta;
}
HD inline double normalize_theta(double theta)
{
    const double PI = 3.14159265358979323846;
    if (theta >= -PI && theta < PI) return theta;
    return normalize_theta_wrap(theta);
}
HD inline double interpolate_angle(double a1, double a2, double factor)
{
    return normalize_theta(a1 + factor * normalize_theta(a2 - a1));
}

// f(x,u) and derivatives wrt q = (theta, u0, u1): J[j*3+i] = df_j/dq_i, Hc = sum_j nu_j Hess f_j packed (tt,t0,t1,00,01,11)
template <int MODEL = MODEL_GENERIC>
HD NOINL inline void dynamics_derivs(const Cfg& c, double th, double v, double w, const double* nu, double* f, double* J,
                                       double* Hc, const double* sc = nullptr)
{
    const int robot = ModelTraits<MODEL>::robot(c);
#pragma unroll
    for (int i = 0; i < 9; ++i) J[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) Hc[i] = 0.0;
    if (robot != MPCB200_ROBOT_KIN_BICYCLE)
    {
        double s, co;
        if (sc) { s = sc[0]; co = sc[1]; }
        else sincos(th, &s, &co);
        f[0] = v * co; f[1] = v * s;
        J[0] = -v * s; J[1] = co;
        J[3] = v * co; J[4] = s;
        Hc[0] = nu[0] * (-v * co) + nu[1] * (-v * s);
        Hc[1] = nu[0] * (-s) + nu[1] * co;
        if (robot == MPCB200_ROBOT_UNICYCLE)
        {
            f[2] = w; J[8] = 1.0;
        }
        else if (robot == MPCB200_ROBOT_SIMPLE_CAR)
        {
            const double L = c.wheelbase, t = tan(w), sec2 = 1.0 + t * t;
            f[2] = v * t / L; J[7] = t / L; J[8] = v * sec2 / L;
            Hc[4] += nu[2] * sec2 / L;
            Hc[5] += nu[2] * 2.0 * v * t * sec2 / L;
        }
        else
        {
            const double L = c.wheelbase;
            double sp, cp;
            sincos(w, &sp, &cp);
            f[2] = v * sp / L; J[7] = sp / L; J[8] = v * cp / L;
            Hc[4] += nu[2] * cp / L;
            Hc[5] += nu[2] * (-v * sp / L);
        }
    }
    else
    {
        const double lr = c.length_rear, kap = lr / (c.length_front + lr);
        const double t = tan(w), sec2 = 1.0 + t * t, den = 1.0 + kap * kap * t * t;
        const double beta = atan(kap * t);
        const double b1 = kap * sec2 / den;
        const double b2 = 2.0 * kap * t * (1.0 - kap * kap) * sec2 / (den * den);
        double s, co, sb, cb;
        sincos(th + beta, &s, &co);
        sincos(beta, &sb, &cb);
        f[0] = v * co; f[1] = v * s; f[2] = v * sb / lr;
        J[0] = -v * s; J[1] = co; J[2] = -v * s * b1;
        J[3] = v * co; J[4] = s;  J[5] = v * co * b1;
        J[6] = 0.0;    J[7] = sb / lr; J[8] = v * cb * b1 / lr;
        Hc[0] += nu[0] * (-v * co) + nu[1] * (-v * s);
        Hc[1] += nu[0] * (-s) + nu[1] * co;
        Hc[2] += nu[0] * (-v * co * b1) + nu[1] * (-v * s * b1);
        Hc[4] += nu[0] * (-s * b1) + nu[1] * (co * b1) + nu[2] * (cb * b1 / lr);
        Hc[5] += nu[0] * (-v * co * b1 * b1 - v * s * b2) + nu[1] * (-v * s * b1 * b1 + v * co * b2) +
                 nu[2] * (v * (-sb * b1 * b1 + cb * b2) / lr);
    }
}

HD NOINL inline void dynamics_value(const Cfg& c, double th, double v, double w, double* f)
{
    if (c.robot_type != MPCB200_ROBOT_KIN_BICYCLE)
    {
        double s, co;
        sincos(th, &s, &co);
        f[0] = v * co; f[1] = v * s;
        if (c.robot_type == MPCB200_ROBOT_UNICYCLE) f[2] = w;
        else if (c.robot_type == MPCB200_ROBOT_SIMPLE_CAR) f[2] = v * tan(w) / c.wheelbase;
        else f[2] = v * sin(w) / c.wheelbase;
    }
    else
    {
        double beta = atan(c.length_rear / (c.length_front + c.length_rear) * tan(w));
        f[0] = v * cos(th + beta); f[1] = v * sin(th + beta); f[2] = v * sin(beta) / c.length_rear;
    }
}

// ---- footprint geometry ----
// distance footprint(pose) <-> point/circle obstacle; optional gradient (x,y,theta) and Hessian (xx,xy,xt,yy,yt,tt)
// LINES = false compiles the line-obstacle path out (the host knows whether a batch contains line obstacles; the hot
// kernels are instantiated both ways so that point / circle batches do not pay its registers)
template <bool WITH_GRAD, bool WITH_HESS, bool LINES = true, int MODEL = MODEL_GENERIC>
HD inline double footprint_distance_sc(const Cfg& c, double px, double py, double s, double co, int obst_type, const double* op,
                                       double* grad3, double* hess6);

template <bool WITH_GRAD, bool WITH_HESS>
HD inline double footprint_distance(const Cfg& c, double px, double py, double pth, int obst_type, const double* op,
                                            double* grad3, double* hess6)
{
    double s, co;
    sincos(pth, &s, &co);
    return footprint_distance_sc<WITH_GRAD, WITH_HESS, true>(c, px, py, s, co, obst_type, op, grad3, hess6);
}

// footprint <-> obstacle POINT (wx, wy) (+ obstacle radius r_obst): the point is taken to the robot frame and the closest
// footprint feature is differentiated through q = R(theta)'(w - p)
template <bool WITH_GRAD, bool WITH_HESS, int MODEL = MODEL_GENERIC>
HD NOINL inline double footprint_distance_point(const Cfg& c, double px, double py, double s, double co, double wx, double wy, double r_obst,
                                          double* grad3, double* hess6)
{
    const int footprint = ModelTraits<MODEL>::footprint(c);
    const double ox = wx - px, oy = wy - py;
    const double qx = co * ox + s * oy, qy = -s * ox + co * oy;
    double best = 1e300, bcx = 0, bcy = 0, brho = 0;
    int bvert = 1;
    // iterate the footprint features without materialising the segment list (register pressure)
    int ns;
    switch (footprint)
    {
        case MPCB200_FOOTPRINT_POINT:
        case MPCB200_FOOTPRINT_CIRCULAR:
        case MPCB200_FOOTPRINT_LINE: ns = 1; break;
        case MPCB200_FOOTPRINT_TWO_CIRCLES: ns = 2; break;
        default: ns = c.n_poly <= 2 ? 1 : c.n_poly;
    }
    for (int i = 0; i < ns; ++i)
    {
        double ax, ay, bx, by, rad = 0.0;
        switch (footprint)
        {
            case MPCB200_FOOTPRINT_POINT: ax = ay = bx = by = 0.0; break;
            case MPCB200_FOOTPRINT_CIRCULAR: ax = ay = bx = by = 0.0; rad = c.footprint_params[0]; break;
            case MPCB200_FOOTPRINT_TWO_CIRCLES:
                if (i == 0) { ax = bx = c.footprint_params[0]; ay = by = 0.0; rad = c.footprint_params[1]; }
                else { ax = bx = -c.footprint_params[2]; ay = by = 0.0; rad = c.footprint_params[3]; }
                break;
            case MPCB200_FOOTPRINT_LINE:
                ax = c.footprint_params[0]; ay = c.footprint_params[1]; bx = c.footprint_params[2]; by = c.footprint_params[3];
                break;
            default:
            {
                int n = c.n_poly;
                int j = (n <= 2) ? (n - 1) : ((i + 1) % n);
                ax = c.poly_xy[2 * i]; ay = c.poly_xy[2 * i + 1]; bx = c.poly_xy[2 * j]; by = c.poly_xy[2 * j + 1];
            }
        }
        double dx = bx - ax, dy = by - ay;
        double sq = dx * dx + dy * dy;
        double t = 0.0;
        if (sq > 0.0) t = ((qx - ax) * dx + (qy - ay) * dy) / sq;
        int isv = 0;
        if (!(sq > 0.0) || t <= 0.0) { t = 0.0; isv = 1; }
        else if (t >= 1.0) { t = 1.0; isv = 1; }
        double cx = ax + t * dx, cy = ay + t * dy;
        double ex = qx - cx, ey = qy - cy;
        double rho = sqrt(ex * ex + ey * ey);
        double d = rho - rad;
        if (d < best) { best = d; bcx = cx; bcy = cy; brho = rho; bvert = isv; }
    }
    double dist = best - r_obst;
    if (WITH_GRAD)
    {
        double rho = brho > 1e-12 ? brho : 1e-12;
        double nx = (qx - bcx) / rho, ny = (qy - bcy) / rho;
        double J0[3] = {-co, -s, qy}, J1[3] = {s, -co, -qx};
#pragma unroll
        for (int i = 0; i < 3; ++i) grad3[i] = nx * J0[i] + ny * J1[i];
        if (WITH_HESS)
        {
            double h00 = 0, h01 = 0, h11 = 0;
            if (bvert) { h00 = (1 - nx * nx) / rho; h01 = -nx * ny / rho; h11 = (1 - ny * ny) / rho; }
            // H = J0 (h00 J0 + h01 J1)' + J1 (h01 J0 + h11 J1)' with explicit fused multiply-adds: left to the compiler, the
            // contraction differed between this loop and its point-footprint form (MODEL_UNI_POINT, the segment folded away), and
            // with it the Hessian's last bits.  The form is the one the compiler chose for the loop.
            double a[3], b[3], H[3][3];
#pragma unroll
            for (int j = 0; j < 3; ++j) a[j] = fma(h00, J0[j], h01 * J1[j]);
            b[0] = fma(h11, J1[0], h01 * J0[0]);
            b[1] = fma(h01, J0[1], h11 * J1[1]);
            b[2] = fma(h01, J0[2], h11 * J1[2]);
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) H[i][j] = fma(J0[i], a[j], J1[i] * b[j]);
            double mx = fma(ny, co, nx * s);
            double my = -nx * co + ny * s;
            H[0][2] += mx; H[2][0] += mx;
            H[1][2] += my; H[2][1] += my;
            H[2][2] += -fma(qy, ny, qx * nx);
            hess6[0] = H[0][0]; hess6[1] = H[0][1]; hess6[2] = H[0][2];
            hess6[3] = H[1][1]; hess6[4] = H[1][2]; hess6[5] = H[2][2];
        }
    }
    return dist;
}


// number of footprint vertices / circle centres and the i-th one in the robot frame (with its radius)
HD inline int footprint_num_vertices(const Cfg& c)
{
    switch (c.footprint_type)
    {
        case MPCB200_FOOTPRINT_POINT:
        case MPCB200_FOOTPRINT_CIRCULAR: return 1;
        case MPCB200_FOOTPRINT_TWO_CIRCLES:
        case MPCB200_FOOTPRINT_LINE: return 2;
        default: return c.n_poly;
    }
}
HD inline void footprint_vertex(const Cfg& c, int i, double* vx, double* vy, double* rad)
{
    *rad = 0.0;
    switch (c.footprint_type)
    {
        case MPCB200_FOOTPRINT_POINT: *vx = 0.0; *vy = 0.0; break;
        case MPCB200_FOOTPRINT_CIRCULAR: *vx = 0.0; *vy = 0.0; *rad = c.footprint_params[0]; break;
        case MPCB200_FOOTPRINT_TWO_CIRCLES:
            if (i == 0) { *vx = c.footprint_params[0]; *vy = 0.0; *rad = c.footprint_params[1]; }
            else { *vx = -c.footprint_params[2]; *vy = 0.0; *rad = c.footprint_params[3]; }
            break;
        case MPCB200_FOOTPRINT_LINE: *vx = c.footprint_params[2 * i]; *vy = c.footprint_params[2 * i + 1]; break;
        default: *vx = c.poly_xy[2 * i]; *vy = c.poly_xy[2 * i + 1];
    }
}
// proper crossing of segments (p1,p2) and (p3,p4) (teb's check_line_segments_intersection_2d: touching counts)
HD inline bool segments_intersect(double p1x, double p1y, double p2x, double p2y, double p3x, double p3y, double p4x, double p4y)
{
    const double d1x = p2x - p1x, d1y = p2y - p1y, d2x = p4x - p3x, d2y = p4y - p3y;
    const double den = d1x * d2y - d1y * d2x;
    if (fabs(den) < 1e-14) return false;  // parallel (collinear overlap is left to the endpoint distances: they are 0 then)
    const double rx = p3x - p1x, ry = p3y - p1y;
    const double t = (rx * d2y - ry * d2x) / den, u = (rx * d1y - ry * d1x) / den;
    return t >= 0.0 && t <= 1.0 && u >= 0.0 && u <= 1.0;
}
// footprint <-> LINE obstacle (a, b) (SURVEY App. B.3): 0 if an edge of a line / polygon footprint crosses the segment, else the
// smaller of (i) the footprint's distance to the two end points and (ii) the distance of the footprint's vertices /
// circle centres to the interior of the segment.
template <bool WITH_GRAD, bool WITH_HESS>
HD NOINL inline double footprint_distance_line(const Cfg& c, double px, double py, double s, double co, const double* op, double* grad3, double* hess6)
{
    const double ax = op[0], ay = op[1], bx = op[2], by = op[3];
    double ux = bx - ax, uy = by - ay;
    const double len = sqrt(ux * ux + uy * uy);
    if (!(len > 1e-12)) return footprint_distance_point<WITH_GRAD, WITH_HESS>(c, px, py, s, co, ax, ay, 0.0, grad3, hess6);
    ux /= len; uy /= len;
    const double nx = -uy, ny = ux;
    const int nv = footprint_num_vertices(c);
    if (c.footprint_type == MPCB200_FOOTPRINT_LINE || (c.footprint_type == MPCB200_FOOTPRINT_POLYGON && c.n_poly >= 2))
    {
        const int ne = (c.footprint_type == MPCB200_FOOTPRINT_LINE || c.n_poly == 2) ? 1 : nv;
        for (int i = 0; i < ne; ++i)
        {
            double v0x, v0y, v1x, v1y, r0;
            footprint_vertex(c, i, &v0x, &v0y, &r0);
            footprint_vertex(c, (i + 1) % nv, &v1x, &v1y, &r0);
            const double w0x = px + co * v0x - s * v0y, w0y = py + s * v0x + co * v0y;
            const double w1x = px + co * v1x - s * v1y, w1y = py + s * v1x + co * v1y;
            if (segments_intersect(w0x, w0y, w1x, w1y, ax, ay, bx, by))
            {
                if (WITH_GRAD) { grad3[0] = grad3[1] = grad3[2] = 0.0; }
                if (WITH_HESS) { for (int j = 0; j < 6; ++j) hess6[j] = 0.0; }
                return 0.0;
            }
        }
    }
    // (ii) vertices against the interior of the obstacle segment
    double best = 1e300, bsig = 1.0, bvx = 0.0, bvy = 0.0;
    for (int i = 0; i < nv; ++i)
    {
        double vx, vy, rad;
        footprint_vertex(c, i, &vx, &vy, &rad);
        const double wx = px + co * vx - s * vy, wy = py + s * vx + co * vy;
        const double t = ((wx - ax) * ux + (wy - ay) * uy) / len;
        if (!(t > 0.0 && t < 1.0)) continue;
        const double sd = (wx - ax) * nx + (wy - ay) * ny;
        const double d = fabs(sd) - rad;
        if (d < best) { best = d; bsig = sd >= 0.0 ? 1.0 : -1.0; bvx = vx; bvy = vy; }
    }
    // (i) the two end points as point obstacles
    double ga[3], ha[6], gb[3], hb[6];
    const double da = footprint_distance_point<WITH_GRAD, WITH_HESS>(c, px, py, s, co, ax, ay, 0.0, ga, ha);
    const double db = footprint_distance_point<WITH_GRAD, WITH_HESS>(c, px, py, s, co, bx, by, 0.0, gb, hb);
    if (da <= best && da <= db)
    {
        if (WITH_GRAD) { grad3[0] = ga[0]; grad3[1] = ga[1]; grad3[2] = ga[2]; }
        if (WITH_HESS) { for (int j = 0; j < 6; ++j) hess6[j] = ha[j]; }
        return da;
    }
    if (db <= best)
    {
        if (WITH_GRAD) { grad3[0] = gb[0]; grad3[1] = gb[1]; grad3[2] = gb[2]; }
        if (WITH_HESS) { for (int j = 0; j < 6; ++j) hess6[j] = hb[j]; }
        return db;
    }
    if (WITH_GRAD)
    {
        // d = sigma n.(p + R v - a) - rad:  dR/dtheta v = (-s vx - co vy, co vx - s vy),  d2R/dtheta2 v = -(R v)
        const double rx = co * bvx - s * bvy, ry = s * bvx + co * bvy;
        grad3[0] = bsig * nx; grad3[1] = bsig * ny; grad3[2] = bsig * (nx * (-ry) + ny * rx);
        if (WITH_HESS)
        {
            hess6[0] = hess6[1] = hess6[2] = hess6[3] = hess6[4] = 0.0;
            hess6[5] = -bsig * (nx * rx + ny * ry);
        }
    }
    return best;
}

// distance footprint(pose) <-> obstacle (point, circle: params x, y, -, -, radius; line: x0, y0, x1, y1) with the sine / cosine of
// the heading supplied by the caller (one sincos per stage, shared by all rows)
template <bool WITH_GRAD, bool WITH_HESS, bool LINES, int MODEL>
HD inline double footprint_distance_sc(const Cfg& c, double px, double py, double s, double co, int obst_type, const double* op,
                                       double* grad3, double* hess6)
{
    if (LINES && obst_type == MPCB200_OBST_LINE) return footprint_distance_line<WITH_GRAD, WITH_HESS>(c, px, py, s, co, op, grad3, hess6);
    return footprint_distance_point<WITH_GRAD, WITH_HESS, MODEL>(c, px, py, s, co, op[0], op[1], obst_type == MPCB200_OBST_CIRCLE ? op[4] : 0.0, grad3, hess6);
}

// A dynamic obstacle (collision_avoidance/enable_dynamic_obstacles, velocity op[5..6] != 0) enters stage k at the position
// predicted for t = k dt with constant velocity (teb estimateSpatioTemporalDistance, R/src/optimal_control/stage_inequality_se2.cpp:177-189)
HD inline bool obstacle_is_dynamic(const Cfg& c, const double* op) { return c.enable_dynamic_obstacles != 0 && (op[5] != 0.0 || op[6] != 0.0); }
HD inline const double* obstacle_at(const Cfg& c, const double* op, int k, double dt, double* buf)
{
    if (!obstacle_is_dynamic(c, op)) return op;
    const double t = (double)k * dt;
    buf[0] = op[0] + t * op[5]; buf[1] = op[1] + t * op[6];
    buf[2] = op[2] + t * op[5]; buf[3] = op[3] + t * op[6];
    buf[4] = op[4];
    return buf;
}

// centroid of an obstacle (teb getCentroid(): point / circle centre, segment midpoint) -- the side test of the association
HD inline void obstacle_centroid(int obst_type, const double* op, double* cx, double* cy)
{
    if (obst_type == MPCB200_OBST_LINE) { *cx = 0.5 * (op[0] + op[2]); *cy = 0.5 * (op[1] + op[3]); }
    else { *cx = op[0]; *cy = op[1]; }
}

HD NOINL inline int clip_bin(double ratio)  // bin j holds the ratios in (2^(-(j+1)/2), 2^(-j/2)]
{
    const int j = (int)floor(-2.0 * log2(ratio));
    return j < 0 ? 0 : (j >= CLIP_BINS ? CLIP_BINS - 1 : j);
}
// threshold bin from the histogram of blocking ratios: the bins jt.. hold at most rows / CLIP_DIV rows
HD inline int clip_threshold_bin(const int* hist, int rows)
{
    int jt = CLIP_BINS, cum = 0;
    for (int j = CLIP_BINS - 1; j >= 0; --j)
    {
        if (cum + hist[j] > rows / CLIP_DIV) break;
        cum += hist[j]; jt = j;
    }
    return jt;
}

// ---- terminal ball (TerminalBallSE2, R/src/optimal_control/final_state_conditions_se2.cpp:54-64): row slot 2 of stage N-1 ----
// g = d'Sd - gamma, d = x - x_f (theta wrapped); optional gradient (S + S')d and Hessian S + S' (packed xx,xy,xt,yy,yt,tt)
HD inline double ball_row(const Cfg& c, const double* x, const double* xf, double* grad3, double* hess6)
{
    const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
    double g = -c.terminal_ball_gamma;
#pragma unroll
    for (int i = 0; i < 3; ++i)
    {
        double gi = 0.0;
#pragma unroll
        for (int j = 0; j < 3; ++j)
        {
            g += d[i] * c.terminal_ball_S[i * 3 + j] * d[j];
            gi += (c.terminal_ball_S[i * 3 + j] + c.terminal_ball_S[j * 3 + i]) * d[j];
        }
        if (grad3) grad3[i] = gi;
    }
    if (hess6)
    {
        int q = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = i; j < 3; ++j, ++q) hess6[q] = c.terminal_ball_S[i * 3 + j] + c.terminal_ball_S[j * 3 + i];
    }
    return g;
}

// ---- linear inequality rows (slots 0..7; see DESIGN.md "row slots") ----
// slot < 4, k <= N-2: control bounds; k == N-1: dt bounds.  slot 4..7: control-rate rows of stage k.
template <int MODEL = MODEL_GENERIC>
HD inline bool lin_row_active(const Cfg& c, int N, int k, int slot, double uprev_dt)
{
    if (slot < 4)
    {
        if (k <= N - 2) return ModelTraits<MODEL>::row_finite(c, slot);
        if (!ModelTraits<MODEL>::variable_dt(c)) return false;
        if (slot == 0) return c.dt_lb > -MPCB200_INF;
        if (slot == 1) return c.dt_ub < MPCB200_INF;
        return false;
    }
    if (k == 0 && uprev_dt == 0.0) return false;
    return ModelTraits<MODEL>::row_finite(c, slot);
}

// value of a linear row; gradient entries wrt u_k[i] (gu), u_{k-1}[i] (gum) and dt (gdt), i = component of the row.
// uk / um: the two control values of component i (um = u_prev for k = 0; uk = u_ref = 0 for k = N-1)
template <int MODEL = MODEL_GENERIC>
HD inline double lin_row(const Cfg& c, int N, int k, int slot, double uk, double um, double dt, double uprev_dt,
                                          double& gu, double& gum, double& gdt)
{
    gu = gum = gdt = 0.0;
    if (slot < 4)
    {
        if (k <= N - 2)
        {
            int i = slot >> 1;
            if (slot & 1) { gu = 1.0; return uk - c.u_ub[i]; }
            gu = -1.0;
            return c.u_lb[i] - uk;
        }
        if (slot == 0) { gdt = -1.0; return c.dt_lb - dt; }
        gdt = 1.0;
        return dt - c.dt_ub;
    }
    int i = (slot - 4) >> 1, ub = (slot - 4) & 1;
    double T = (k >= 1) ? dt : uprev_dt;
    double sgn = ub ? 1.0 : -1.0;
    double bnd = ub ? c.du_ub[i] : c.du_lb[i];
    if (k <= N - 2) gu = sgn;
    if (k >= 1) gum = -sgn;
    if (k >= 1 && ModelTraits<MODEL>::variable_dt(c)) gdt = -sgn * bnd;
    return sgn * ((uk - um) - bnd * T);
}

HD inline int hidx(int i, int j) { return i * 5 - (i * (i - 1)) / 2 + (j - i); }

HD NOINL inline double scaled_error(double dual_inf, double prim_inf, double sl_max, double sl_min, double sum_nu,
                                               double sum_lam, int m_eq, int m_ineq, double mu)
{
    double sd = (sum_nu + sum_lam) / (double)(m_eq + m_ineq > 0 ? m_eq + m_ineq : 1);
    sd = (sd > SMAX ? sd : SMAX) / SMAX;
    double sc = m_ineq > 0 ? sum_lam / (double)m_ineq : 0.0;
    sc = (sc > SMAX ? sc : SMAX) / SMAX;
    double compl_ = 0.0;
    if (m_ineq > 0)
    {
        double a = sl_max - mu, b = mu - sl_min;
        compl_ = a > b ? a : b;
        if (compl_ < 0) compl_ = 0;
    }
    double e = dual_inf / sd;
    if (prim_inf > e) e = prim_inf;
    if (compl_ / sc > e) e = compl_ / sc;
    return e;
}
