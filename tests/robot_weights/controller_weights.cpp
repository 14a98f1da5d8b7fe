// controller_weights.cpp -- the C++ mirror with objective weights that change at run time (TEST INFRASTRUCTURE): a quadratic-form
// unicycle (cfg 2's weights, N = 30, fixed dt) whose control weights R grow eightfold from the second step on by
// Controller::setRobotWeights -- no reconfigure, so the later steps warm-start.  Beside it run a controller that keeps the
// configuration's weights ("plain") and one configured with the new weights ("heavy").  Per step it prints whether the
// controller's plan equals the plain one's bit for bit; after the steps it resets the controller and the heavy one and prints
// whether their next (cold) plans are bit for bit equal, which holds only when the weights survived reset().
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/mpcb200_controller.hpp"

static bool same(const mpcb200::TimeSeries& a, const mpcb200::TimeSeries& b)
{
    return a.values.size() == b.values.size() && std::memcmp(a.values.data(), b.values.data(), a.values.size() * sizeof(double)) == 0;
}

int main()
{
    mpcb200_config cfg;
    mpcb200_default_config(&cfg);
    cfg.n = 30; cfg.variable_dt = 0; cfg.dt_ref = 0.3;
    cfg.xf_fixed[0] = cfg.xf_fixed[1] = cfg.xf_fixed[2] = 0;
    cfg.objective = MPCB200_OBJ_QUADRATIC_FORM;
    const double q[3] = {2.0, 2.0, 0.25}, r[2] = {0.1, 0.05}, qf[3] = {10.0, 10.0, 0.5};
    for (int i = 0; i < 3; ++i) { cfg.Q[4 * i] = q[i]; cfg.Qf[4 * i] = qf[i]; }
    for (int i = 0; i < 2; ++i) cfg.R[3 * i] = r[i];
    cfg.terminal_cost = 1;
    cfg.min_obstacle_dist = 0.2; cfg.k_max_obstacles_per_stage = 3;
    cfg.tol = 1e-8;
    double weights[MPCB200_WEIGHT_WORDS] = {};
    for (int i = 0; i < 9; ++i) { weights[MPCB200_WGT_Q + i] = cfg.Q[i]; weights[MPCB200_WGT_QF + i] = cfg.Qf[i]; }
    for (int i = 0; i < 4; ++i) weights[MPCB200_WGT_R + i] = 8.0 * cfg.R[i];
    mpcb200_config heavy_cfg = cfg;
    for (int i = 0; i < 4; ++i) heavy_cfg.R[i] = weights[MPCB200_WGT_R + i];

    std::vector<mpcb200::Obstacle> obstacles(2);
    obstacles[0].x0 = 2; obstacles[0].y0 = 0.6;
    obstacles[1].x0 = 3.5; obstacles[1].y0 = 1.8;
    std::vector<mpcb200::PoseSE2> via_points;
    mpcb200::ControllerParams params;
    mpcb200::Controller controller, plain, heavy;
    if (!controller.configure(cfg, params, &obstacles, &via_points) || !plain.configure(cfg, params, &obstacles, &via_points) ||
        !heavy.configure(heavy_cfg, params, &obstacles, &via_points))
        return 2;
    mpcb200::PoseSE2 x0, xf;
    xf.x = 5; xf.y = 2; xf.theta = 0;
    mpcb200::TimeSeries u, x, pu, px, hu, hx;
    for (int i = 0; i < 3; ++i)
    {
        if (i == 1 && !controller.setRobotWeights(weights)) return 2;
        if (!controller.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &u, &x)) return 1;
        if (!plain.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &pu, &px)) return 1;
        std::printf("step %d status %d iters %d same_as_plain %d\n", i, controller.lastStatus(), controller.lastIterations(),
                    (int)(same(u, pu) && same(x, px)));
        x0.x = x.values[3]; x0.y = x.values[4]; x0.theta = x.values[5];
    }
    controller.reset();
    heavy.reset();
    if (!controller.step(x0, xf, mpcb200::Twist(), 0.05, 0.2, &u, &x)) return 1;
    if (!heavy.step(x0, xf, mpcb200::Twist(), 0.05, 0.2, &hu, &hx)) return 1;
    if (!plain.step(x0, xf, mpcb200::Twist(), 0.05, 0.2, &pu, &px)) return 1;
    std::printf("after reset status %d same_as_heavy %d same_as_plain %d\n", controller.lastStatus(), (int)(same(u, hu) && same(x, hx)),
                (int)(same(u, pu) && same(x, px)));
    return 0;
}
