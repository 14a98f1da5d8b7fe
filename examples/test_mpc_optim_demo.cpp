// ROS-free twin of the reference's only standalone driver, test_mpc_optim_node
// (mpc_local_planner/src/test_mpc_optim_node.cpp:59-131): fixed start (0,0,0) -> goal (5,2,0), three point obstacles,
// unicycle minimum-time OCP with the parameters of mpc_local_planner/cfg/test_mpc_optim_node.yaml, re-solved in a loop
// through the mpc_local_planner::Controller mirror (include/mpcb200_controller.hpp) on top of the C ABI.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../include/mpcb200_controller.hpp"

int main(int argc, char** argv)
{
    const int steps = argc > 1 ? std::atoi(argv[1]) : 3;
    // grid/variable_grid/grid_adaptation/enable (True in test_mpc_optim_node.yaml:54-58, with dt_hyst_ratio 0.1 and at most 50
    // grid points): 1 = the horizon follows the optimal dt one grid point per step, 0 (default here) = fixed N = 20
    const bool adapt = argc > 2 && std::atoi(argv[2]) != 0;
    mpcb200_config cfg;
    mpcb200_default_config(&cfg);  // unicycle, N = 20, dt_ref = 0.3, minimum_time, xf fixed, point footprint, d_min 0.5
    // solver/ipopt/max_cpu_time in seconds (default -1: no limit); a step stopped by it still succeeds (EarlyTerminated)
    if (argc > 3) cfg.max_cpu_time = std::atof(argv[3]);
    cfg.k_max_obstacles_per_stage = 3;
    cfg.tol = 1e-8;
    std::vector<mpcb200::Obstacle> obstacles(3);
    obstacles[0].x0 = -3; obstacles[0].y0 = 1;   // test_mpc_optim_node.cpp:67-69
    obstacles[1].x0 = 6;  obstacles[1].y0 = 2;
    obstacles[2].x0 = 4;  obstacles[2].y0 = 0.1;
    std::vector<mpcb200::PoseSE2> via_points;
    mpcb200::Controller controller;
    mpcb200::ControllerParams params;
    params.grid_adaptation = adapt;
    if (!controller.configure(cfg, params, &obstacles, &via_points)) return 2;
    mpcb200::PoseSE2 x0, xf;
    xf.x = 5; xf.y = 2; xf.theta = 0;  // test_mpc_optim_node.cpp:105-106
    mpcb200::TimeSeries u_seq, x_seq;
    for (int i = 0; i < steps; ++i)
    {
        const bool ok = controller.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &u_seq, &x_seq);
        const int n = controller.gridSize();
        std::printf("step %d ok %d status %d iters %d dt %.9f u0 %.9f %.9f xN %.6f %.6f %.6f kkt %.2e n %d\n", i, (int)ok, controller.lastStatus(),
                    controller.lastIterations(), controller.lastDt(), u_seq.values[0], u_seq.values[1], x_seq.values[3 * (n - 1)],
                    x_seq.values[3 * (n - 1) + 1], x_seq.values[3 * (n - 1) + 2], controller.lastKktError(), n);
        if (!ok) return 1;
    }
    return 0;
}
