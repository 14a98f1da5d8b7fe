// mpcb200_controller.hpp -- C++ host side above the C ABI: a ROS-free mirror of mpc_local_planner::Controller for the
// hot path (reference: mpc_local_planner/include/mpc_local_planner/controller.h:53-143,
// mpc_local_planner/src/controller.cpp:58-179, 807-857).  Same method names, argument meaning and error behaviour
// (bool returns, no exception crosses step()); ROS / corbo / teb types are replaced by PODs with the same meaning:
//
//   teb_local_planner::PoseSE2          -> mpcb200::PoseSE2 {x, y, theta}
//   geometry_msgs::Twist                -> mpcb200::Twist {linear_x, linear_y, angular_z}
//   std::vector<PoseStamped> (plan)     -> std::vector<mpcb200::PoseSE2>
//   corbo::TimeSeries::Ptr              -> mpcb200::TimeSeries {time[], values[] (row-major [k][dim]), dim}
//   teb ObstContainer / via-point list  -> mpcb200::Obstacle / PoseSE2 vectors owned by the CALLER and read at every
//                                          step (the reference holds them by const reference, inc/controller.h:61-63)
//
// One Controller drives one robot (B = 1), exactly like the reference; many robots that share a configuration are
// driven with ONE mpcb200_step_batch call on the C ABI (this is where the GPU pays off).  Header-only; link against
// libmpcb200.so.
#ifndef MPCB200_CONTROLLER_HPP_
#define MPCB200_CONTROLLER_HPP_

#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "mpcb200.h"

namespace mpcb200 {

struct PoseSE2 { double x = 0, y = 0, theta = 0; };
struct Twist { double linear_x = 0, linear_y = 0, angular_z = 0; };
struct Obstacle { int type = MPCB200_OBST_POINT; double x0 = 0, y0 = 0, x1 = 0, y1 = 0, radius = 0, vx = 0, vy = 0; };  // (vx, vy): centroid velocity of a dynamic obstacle

struct TimeSeries
{
    int dim = 0;
    std::vector<double> time;    // N samples
    std::vector<double> values;  // [k][dim]
    void clear() { time.clear(); values.clear(); }
    bool isEmpty() const { return time.empty(); }
};

// normalize_theta / interpolate_angle: inc/utils/math_utils.h:81-103
inline double normalize_theta(double theta)
{
    if (theta >= -M_PI && theta < M_PI) return theta;
    double multiplier = std::floor(theta / (2.0 * M_PI));
    theta = theta - multiplier * 2.0 * M_PI;
    if (theta >= M_PI) theta -= 2.0 * M_PI;
    if (theta < -M_PI) theta += 2.0 * M_PI;
    return theta;
}
inline double interpolate_angle(double a1, double a2, double f) { return normalize_theta(a1 + f * normalize_theta(a2 - a1)); }

// controller-level parameters that are not part of the OCP (src/controller.cpp:70-88; SURVEY App. D)
struct ControllerParams
{
    double force_reinit_new_goal_dist = 1.0;
    double force_reinit_new_goal_angular = 0.5 * M_PI;
    int force_reinit_num_steps = 0;
    bool allow_init_with_backward_motion = true;
    bool global_plan_overwrite_orientation = true;  // _initial_plan_estimate_orientation
    bool print_cpu_time = false;
    // grid/variable_grid/grid_adaptation/* (src/controller.cpp:247-262; used only with a variable grid, config.variable_dt):
    // TimeBasedSingleStep with adapt_first_iter = true -- before every step but the first after a (re-)initialisation the
    // horizon grows by one grid point when the last optimal dt exceeds dt_ref (1 + dt_hyst_ratio) and shrinks by one when
    // it is below dt_ref (1 - dt_hyst_ratio) (finite_differences_variable_grid_se2.cpp:99-121).  The reference's defaults.
    bool grid_adaptation = true;
    int max_grid_size = 50;
    int min_grid_size = 2;   // the solver needs 3 grid points: values below 3 act as 3
    double dt_hyst_ratio = 0.1;
    // multistart (mpcb200_step_batch_multistart with B = 1): K > 1 solves the robot's problem from its usual initial guess and
    // from K - 1 other bumped lines in one launch and keeps the best local optimum; a challenger replaces a converged plan only
    // when its objective is below obj - (1 - multistart_hysteresis) |obj| (teb's selection_cost_hysteresis).  1: off.
    int multistart_candidates = 1;
    double multistart_hysteresis = 1.0;
};

// initial state trajectory from an initial plan (Controller::generateInitialStateTrajectory, src/controller.cpp:807-857,
// sampled like TimeSeriesSE2 linear interpolation, src/utils/time_series_se2.cpp:86-102): x_init[k] = x(k * dt_ref)
inline bool generateInitialStateTrajectory(const mpcb200_config& cfg, const PoseSE2& x0, const PoseSE2& xf,
                                           const std::vector<PoseSE2>& initial_plan, bool backward, bool estimate_orientation,
                                           std::vector<double>& x_init /* [N][3] */)
{
    (void)backward;  // reference quirk (SURVEY App. C.2): the flipped yaw is computed and discarded -> no effect
    const int n_init = (int)initial_plan.size();
    const int N = cfg.n;
    if (n_init < 2 || N < 2) return false;
    const double tf_ref = (double)(N - 1) * cfg.dt_ref;
    const double dt_init = tf_ref / (double)(n_init - 1);
    std::vector<double> ts(n_init);
    std::vector<PoseSE2> ps(n_init);
    ts[0] = 0.0; ps[0] = x0;
    double t = dt_init;
    for (int i = 1; i < n_init - 1; ++i, t += dt_init)
    {
        PoseSE2 p = initial_plan[i];
        if (estimate_orientation)
            p.theta = std::atan2(initial_plan[i + 1].y - initial_plan[i].y, initial_plan[i + 1].x - initial_plan[i].x);
        ts[i] = t; ps[i] = p;
    }
    ts[n_init - 1] = tf_ref; ps[n_init - 1] = xf;
    x_init.assign((size_t)N * 3, 0.0);
    int seg = 1;
    for (int k = 0; k < N; ++k)
    {
        const double tk = (double)k * cfg.dt_ref;
        while (seg < n_init - 1 && ts[seg] < tk) ++seg;
        const double dtd = ts[seg] - ts[seg - 1];
        double f = dtd > 0 ? (tk - ts[seg - 1]) / dtd : 0.0;
        if (f > 1.0) f = 1.0;
        x_init[3 * k + 0] = ps[seg - 1].x + f * (ps[seg].x - ps[seg - 1].x);
        x_init[3 * k + 1] = ps[seg - 1].y + f * (ps[seg].y - ps[seg - 1].y);
        x_init[3 * k + 2] = interpolate_angle(ps[seg - 1].theta, ps[seg].theta, f);
    }
    return true;
}

class Controller
{
 public:
    Controller() = default;
    ~Controller() { if (_h) mpcb200_destroy(_h); }
    Controller(const Controller&) = delete;
    Controller& operator=(const Controller&) = delete;

    // Controller::configure (inc/controller.h:61-63): obstacles / via-points are held by pointer and must outlive the controller.
    bool configure(const mpcb200_config& cfg, const ControllerParams& params, const std::vector<Obstacle>* obstacles,
                   const std::vector<PoseSE2>* via_points, int device = 0)
    {
        if (_h) { mpcb200_destroy(_h); _h = nullptr; }
        _cfg = cfg; _params = params; _obstacles = obstacles; _via_points = via_points;
        _n_ref = cfg.n;
        _adapt = params.grid_adaptation && cfg.variable_dt;
        // with grid adaptation the handle is sized for the largest horizon and starts at grid_size_ref
        mpcb200_config cap = cfg;
        if (_adapt && params.max_grid_size > cap.n) cap.n = params.max_grid_size;
        const int K = params.multistart_candidates > 1 ? params.multistart_candidates : 1;
        int rc = mpcb200_create(&cap, K, device, &_h);
        if (rc != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::configure(): %s\n", mpcb200_last_error(nullptr));
            _h = nullptr;
            return false;
        }
        if (!setHorizon(_n_ref)) return false;
        if (_has_limits && !applyRobotLimits()) return false;
        if (!applyRobotGeometryAndModel()) return false;
        if (_has_weights && !applyRobotWeights()) return false;
        _ocp_seq = 0; _grid_empty = true; _ocp_successful = false;
        return true;
    }

    // Runtime limits of this robot (mpcb200_set_robot_limits with one record): u_lb[2], u_ub[2], du_lb[2], du_ub[2] and
    // min_obstacle_dist in place of the configuration's (a speed-limit zone, a payload, people nearby); with multistart they
    // cover all its candidates.  The next step warm-starts under the new values.  They survive reset(), grid adaptation and a
    // new configure(); false (and the previous limits kept) when the record is not valid for the configuration (mpcb200.h).
    bool setRobotLimits(const double limits[MPCB200_LIMIT_WORDS])
    {
        if (_h && mpcb200_set_robot_limits(_h, 1, limits) != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::setRobotLimits(): %s\n", mpcb200_last_error(_h));
            return false;
        }
        for (int i = 0; i < MPCB200_LIMIT_WORDS; ++i) _limits[i] = limits[i];
        _has_limits = true;
        return true;
    }
    // back to the configuration's limits
    void clearRobotLimits()
    {
        if (_h) mpcb200_set_robot_limits(_h, 0, nullptr);
        _has_limits = false;
    }

    // Runtime geometry of this robot (mpcb200_set_robot_geometry with one record, MPCB200_GEO_* words): the wheelbase or the
    // bicycle's lengths and the footprint's values in place of the configuration's (a cart picked up, a tool extended).  The robot
    // and footprint types stay the configuration's.  This is the footprint change of the reference without a reconfigure: the next
    // step warm-starts under the new values.  They survive reset(), grid adaptation and a new configure(); false (and the previous
    // geometry kept) when the record is not valid for the configuration (mpcb200.h).
    bool setRobotGeometry(const double geometry[MPCB200_GEOMETRY_WORDS])
    {
        if (_h && mpcb200_set_robot_geometry(_h, 1, geometry) != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::setRobotGeometry(): %s\n", mpcb200_last_error(_h));
            return false;
        }
        for (int i = 0; i < MPCB200_GEOMETRY_WORDS; ++i) _geometry[i] = geometry[i];
        _has_geometry = true;
        return true;
    }
    // back to the configuration's geometry
    void clearRobotGeometry()
    {
        if (_h) mpcb200_set_robot_geometry(_h, 0, nullptr);
        _has_geometry = false;
    }

    // Runtime model of this robot (mpcb200_set_robot_model with one record): its robot_type and footprint_type (MPCB200_ROBOT_*,
    // MPCB200_FOOTPRINT_*) in place of the configuration's -- the reference's robot/type and footprint_model/type without a
    // reconfigure, e.g. a circular robot that picks up a cart and gets a polygon.  The solves then run the generic kernel key.  The
    // robot's geometry (setRobotGeometry, else the configuration's values) must be valid for the new types, so a footprint-type
    // change goes geometry first (a record holding the words of the old and the new footprint, e.g. a radius and a polygon), then
    // model.  The next step warm-starts from the previous plan under the new model.  The model survives reset(), grid adaptation
    // and a new configure(); false (and the previous model kept) when the pair is refused (mpcb200.h).
    bool setRobotModel(int robot_type, int footprint_type)
    {
        const double model[MPCB200_MODEL_WORDS] = {(double)robot_type, (double)footprint_type};
        if (_h && mpcb200_set_robot_model(_h, 1, model) != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::setRobotModel(): %s\n", mpcb200_last_error(_h));
            return false;
        }
        _model[0] = model[0]; _model[1] = model[1];
        _has_model = true;
        return true;
    }
    // back to the configuration's types; false (and the model kept) when the robot's geometry record is not valid for them
    bool clearRobotModel()
    {
        if (_h && mpcb200_set_robot_model(_h, 0, nullptr) != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::clearRobotModel(): %s\n", mpcb200_last_error(_h));
            return false;
        }
        _has_model = false;
        return true;
    }

    // Runtime objective weights of this robot (mpcb200_set_robot_weights with one record, MPCB200_WGT_* words): Q, R, Qf and the
    // via-point weights in place of the configuration's (a heavier heading or terminal weight near the goal, smoother control with
    // a load).  The objective and its terms stay the configuration's.  The next step warm-starts under the new values.  They
    // survive reset(), grid adaptation and a new configure(); false (and the previous weights kept) when the record is not valid
    // for the configuration (mpcb200.h).
    bool setRobotWeights(const double weights[MPCB200_WEIGHT_WORDS])
    {
        if (_h && mpcb200_set_robot_weights(_h, 1, weights) != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::setRobotWeights(): %s\n", mpcb200_last_error(_h));
            return false;
        }
        for (int i = 0; i < MPCB200_WEIGHT_WORDS; ++i) _weights[i] = weights[i];
        _has_weights = true;
        return true;
    }
    // back to the configuration's weights
    void clearRobotWeights()
    {
        if (_h) mpcb200_set_robot_weights(_h, 0, nullptr);
        _has_weights = false;
    }

    // StructuredOptimalControlProblem::setPreviousControlInput (called by the planner before step, src/mpc_local_planner_ros.cpp:384)
    void setPreviousControlInput(const double u_prev[2], double dt) { _u_prev[0] = u_prev[0]; _u_prev[1] = u_prev[1]; _u_prev_dt = dt; }

    // Controller::step(start, goal, ...) (src/controller.cpp:102-109)
    bool step(const PoseSE2& start, const PoseSE2& goal, const Twist& vel, double dt, double t, TimeSeries* u_seq, TimeSeries* x_seq)
    {
        std::vector<PoseSE2> plan(2);
        plan.front() = start; plan.back() = goal;
        return step(plan, vel, dt, t, u_seq, x_seq);
    }

    // Controller::step(initial_plan, ...) (src/controller.cpp:111-179)
    bool step(const std::vector<PoseSE2>& initial_plan, const Twist& vel, double dt, double t, TimeSeries* u_seq, TimeSeries* x_seq)
    {
        (void)vel; (void)dt; (void)t;  // SE2 models take the full state from the start pose (inc/systems/base_robot_se2.h:93-101)
        if (!_h)
        {
            std::fprintf(stderr, "Controller must be configured before invoking step().\n");
            return false;
        }
        if (initial_plan.size() < 2)
        {
            std::fprintf(stderr, "Controller::step(): initial plan must contain at least two poses.\n");
            return false;
        }
        const PoseSE2 start = initial_plan.front(), goal = initial_plan.back();
        // re-init policy (src/controller.cpp:152-158)
        if (_params.force_reinit_num_steps > 0 && _ocp_seq % _params.force_reinit_num_steps == 0) _grid_empty = true;
        if (!_grid_empty)
        {
            const double dx = goal.x - _last_goal.x, dy = goal.y - _last_goal.y;
            if (std::sqrt(dx * dx + dy * dy) > _params.force_reinit_new_goal_dist ||
                std::fabs(normalize_theta(goal.theta - _last_goal.theta)) > _params.force_reinit_new_goal_angular)
                _grid_empty = true;
        }
        unsigned char reinit = 0;
        const double* x_init_ptr = nullptr;
        if (_grid_empty)
        {
            // FullDiscretizationGridBaseSE2::clear() forgets the adapted grid size: initialisation uses grid_size_ref again
            // (full_discretization_grid_base_se2.cpp:153,526-536)
            if (!setHorizon(_n_ref)) return false;
        }
        else if (_adapt)
        {
            // FiniteDifferencesVariableGridSE2::adaptGridTimeBasedSingleStep (finite_differences_variable_grid_se2.cpp:99-121),
            // called at the start of the grid update of a non-empty grid (full_discretization_grid_base_se2.cpp:52-56)
            const int n = _cfg.n, n_min = _params.min_grid_size < 3 ? 3 : _params.min_grid_size;
            int n_max = 0;
            mpcb200_get_horizon(_h, nullptr, &n_max);
            if (_params.max_grid_size < n_max) n_max = _params.max_grid_size;
            if (_last_dt > _cfg.dt_ref * (1.0 + _params.dt_hyst_ratio) && n < n_max) { if (!setHorizon(n + 1)) return false; }
            else if (_last_dt < _cfg.dt_ref * (1.0 - _params.dt_hyst_ratio) && n > n_min) { if (!setHorizon(n - 1)) return false; }
        }
        if (_grid_empty)
        {
            const bool backward = _params.allow_init_with_backward_motion &&
                                  ((goal.x - start.x) * std::cos(start.theta) + (goal.y - start.y) * std::sin(start.theta)) < 0;
            if (initial_plan.size() > 2)
            {
                generateInitialStateTrajectory(_cfg, start, goal, initial_plan, backward, _params.global_plan_overwrite_orientation, _x_init);
                x_init_ptr = _x_init.data();
            }
            reinit = 1;
        }
        const double x0[3] = {start.x, start.y, start.theta}, xf[3] = {goal.x, goal.y, goal.theta};
        // obstacles / via-points are read at every step (the caller mutates its containers between steps)
        std::vector<int> otype; std::vector<double> oparams; int ocount = 0;
        mpcb200_obstacles ob{0, nullptr, nullptr, nullptr};
        if (_obstacles && !_obstacles->empty())
        {
            ocount = (int)_obstacles->size();
            otype.resize(ocount); oparams.resize((size_t)ocount * MPCB200_OBST_STRIDE);
            for (int i = 0; i < ocount; ++i)
            {
                const Obstacle& o = (*_obstacles)[i];
                otype[i] = o.type;
                double* p = &oparams[(size_t)i * MPCB200_OBST_STRIDE];
                p[0] = o.x0; p[1] = o.y0; p[2] = o.x1; p[3] = o.y1; p[4] = o.radius; p[5] = o.vx; p[6] = o.vy;
            }
            ob.max_per_instance = ocount; ob.count = &ocount; ob.type = otype.data(); ob.params = oparams.data();
        }
        std::vector<double> vposes; int vcount = 0;
        mpcb200_viapoints vp{0, nullptr, nullptr};
        if (_via_points && !_via_points->empty())
        {
            vcount = (int)_via_points->size();
            vposes.resize((size_t)vcount * 3);
            for (int i = 0; i < vcount; ++i) { vposes[3 * i] = (*_via_points)[i].x; vposes[3 * i + 1] = (*_via_points)[i].y; vposes[3 * i + 2] = (*_via_points)[i].theta; }
            vp.max_per_instance = vcount; vp.count = &vcount; vp.poses = vposes.data();
        }
        const int N = _cfg.n;
        _u.assign((size_t)N * 2, 0.0); _x.assign((size_t)N * 3, 0.0);
        int status = 0, iters = 0; double dt_out = 0, kkt = 0, secs = 0;
        const int K = _params.multistart_candidates;
        const int rc = K > 1 ? mpcb200_step_batch_multistart(_h, 1, K, _params.multistart_hysteresis, x0, xf, _u_prev, _u_prev_dt,
                                                             ocount ? &ob : nullptr, vcount ? &vp : nullptr, x_init_ptr, &reinit, _u.data(),
                                                             _x.data(), &dt_out, &status, &kkt, &iters, nullptr, &secs)
                             : mpcb200_step_batch(_h, 1, x0, xf, _u_prev, _u_prev_dt, ocount ? &ob : nullptr, vcount ? &vp : nullptr, x_init_ptr,
                                                  &reinit, _u.data(), _x.data(), &dt_out, &status, &kkt, &iters, &secs);
        if (rc != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller::step(): %s\n", mpcb200_last_error(_h));
            _ocp_successful = false;
        }
        else
        {
            // success iff the solver status is Converged or EarlyTerminated (SURVEY App. B.1).  EarlyTerminated covers the iteration
            // cap and the time budget (max_cpu_time): [EXT] Ipopt's Maximum_CpuTime_Exceeded is taken to map to EarlyTerminated like
            // Maximum_Iterations_Exceeded -- the mapping lives in corbo's Ipopt wrapper, which is not part of the reference tree.
            _ocp_successful = (status == MPCB200_STATUS_CONVERGED || status == MPCB200_STATUS_MAX_ITER || status == MPCB200_STATUS_MAX_TIME);
            // a failed solve (numerical error, invalid input) leaves no trajectory to warm-start from: the device keeps the
            // instance cold, and the grid counts as empty here (the reference's planner resets the controller after a failed step)
            _grid_empty = !_ocp_successful;
            if (u_seq) fill(*u_seq, _u, 2, N, dt_out);
            if (x_seq) fill(*x_seq, _x, 3, N, dt_out);
            _last_dt = dt_out; _last_status = status; _last_iters = iters; _last_kkt = kkt; _last_solve_time = secs;
        }
        if (_params.print_cpu_time) std::fprintf(stderr, "Cpu time: %.3f ms.\n", secs * 1e3);
        ++_ocp_seq;
        _last_goal = goal;
        return _ocp_successful;
    }

    // Controller::reset (inc/controller.h:104)
    void reset()
    {
        if (_h) mpcb200_reset(_h, nullptr, 1);
        _grid_empty = true;
    }

    bool isOptimizationSuccessful() const { return _ocp_successful; }
    int gridSize() const { return _cfg.n; }  // current number of grid points (getN())
    double lastDt() const { return _last_dt; }
    int lastStatus() const { return _last_status; }
    int lastIterations() const { return _last_iters; }
    double lastKktError() const { return _last_kkt; }
    double lastSolveTime() const { return _last_solve_time; }

 private:
    // resampleTrajectory(n) on the device (or just the new horizon for an empty grid); _cfg.n follows
    bool setHorizon(int n)
    {
        if (n == _cfg.n) { int cur = 0; mpcb200_get_horizon(_h, &cur, nullptr); if (cur == n) return true; }
        const int rc = mpcb200_resample(_h, n);
        if (rc != MPCB200_OK)
        {
            std::fprintf(stderr, "Controller: horizon change to %d grid points failed: %s\n", n, mpcb200_last_error(_h));
            return false;
        }
        _cfg.n = n;
        return true;
    }
    bool applyRobotLimits()
    {
        if (mpcb200_set_robot_limits(_h, 1, _limits) == MPCB200_OK) return true;
        std::fprintf(stderr, "Controller: robot limits: %s\n", mpcb200_last_error(_h));
        return false;
    }
    bool applyRobotGeometry()
    {
        if (mpcb200_set_robot_geometry(_h, 1, _geometry) == MPCB200_OK) return true;
        std::fprintf(stderr, "Controller: robot geometry: %s\n", mpcb200_last_error(_h));
        return false;
    }
    // the geometry and model records on a new handle: the geometry first when the handle's own types accept it, else the model
    // first (checked against the configuration's geometry values)
    bool applyRobotGeometryAndModel()
    {
        if (!_has_model) return !_has_geometry || applyRobotGeometry();
        const auto model = [&] { return mpcb200_set_robot_model(_h, 1, _model) == MPCB200_OK; };
        const auto geometry = [&] { return !_has_geometry || mpcb200_set_robot_geometry(_h, 1, _geometry) == MPCB200_OK; };
        if ((geometry() && model()) || (model() && geometry())) return true;
        std::fprintf(stderr, "Controller: robot model: %s\n", mpcb200_last_error(_h));
        return false;
    }
    bool applyRobotWeights()
    {
        if (mpcb200_set_robot_weights(_h, 1, _weights) == MPCB200_OK) return true;
        std::fprintf(stderr, "Controller: robot weights: %s\n", mpcb200_last_error(_h));
        return false;
    }
    static void fill(TimeSeries& ts, const std::vector<double>& v, int dim, int N, double dt)
    {
        ts.clear(); ts.dim = dim;
        ts.time.resize(N); ts.values = v;
        for (int k = 0; k < N; ++k) ts.time[k] = (double)k * dt;  // getStateAndControlTimeSeries, full_discretization_grid_base_se2.cpp:579-615
    }
    mpcb200_handle* _h = nullptr;
    mpcb200_config _cfg{};
    ControllerParams _params;
    const std::vector<Obstacle>* _obstacles = nullptr;
    const std::vector<PoseSE2>* _via_points = nullptr;
    double _u_prev[2] = {0, 0};
    double _u_prev_dt = 0.0;
    std::vector<double> _x_init, _u, _x;
    PoseSE2 _last_goal;
    int _ocp_seq = 0;
    int _n_ref = 0;       // grid/grid_size_ref
    bool _adapt = false;  // grid adaptation active (variable grid + grid_adaptation/enable)
    bool _grid_empty = true, _ocp_successful = false;
    double _last_dt = 0, _last_kkt = 0, _last_solve_time = 0;
    int _last_status = -1, _last_iters = 0;
    double _limits[MPCB200_LIMIT_WORDS] = {};
    bool _has_limits = false;   // setRobotLimits in effect
    double _geometry[MPCB200_GEOMETRY_WORDS] = {};
    bool _has_geometry = false; // setRobotGeometry in effect
    double _weights[MPCB200_WEIGHT_WORDS] = {};
    bool _has_weights = false;  // setRobotWeights in effect
    double _model[MPCB200_MODEL_WORDS] = {};
    bool _has_model = false;    // setRobotModel in effect
};

}  // namespace mpcb200
#endif
