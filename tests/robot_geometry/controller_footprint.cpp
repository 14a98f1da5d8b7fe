// controller_footprint.cpp -- the C++ mirror with a footprint that grows at run time (TEST INFRASTRUCTURE): the demo's scene with a
// circular footprint of radius 0.1, enlarged to 0.35 from the second step on by Controller::setRobotGeometry -- no reconfigure,
// so the later steps warm-start.  Per step it prints the radius in effect, the status and iterations, the smallest clearance of
// the plan (distance of the circle to the nearest point obstacle) and the iterations of a cold solve of the same step by a
// controller configured with that radius.
#include <cmath>
#include <cstdio>
#include <vector>

#include "../../include/mpcb200_controller.hpp"

int main()
{
    mpcb200_config cfg;
    mpcb200_default_config(&cfg);   // unicycle, N = 20, minimum time, xf fixed, d_min 0.5
    cfg.k_max_obstacles_per_stage = 3;
    cfg.tol = 1e-8;
    cfg.footprint_type = MPCB200_FOOTPRINT_CIRCULAR;
    cfg.footprint_params[0] = 0.1;
    std::vector<mpcb200::Obstacle> obstacles(3);
    obstacles[0].x0 = -3; obstacles[0].y0 = 1;
    obstacles[1].x0 = 6;  obstacles[1].y0 = 2;
    obstacles[2].x0 = 4;  obstacles[2].y0 = 0.1;
    std::vector<mpcb200::PoseSE2> via_points;
    mpcb200::ControllerParams params;
    mpcb200::Controller controller;
    if (!controller.configure(cfg, params, &obstacles, &via_points)) return 2;
    mpcb200::PoseSE2 x0, xf;
    xf.x = 5; xf.y = 2; xf.theta = 0;
    mpcb200::TimeSeries u_seq, x_seq;
    double radius = cfg.footprint_params[0];
    for (int i = 0; i < 4; ++i)
    {
        if (i == 1)   // a cart picked up: the circle grows, everything else stays
        {
            radius = 0.35;
            double geometry[MPCB200_GEOMETRY_WORDS] = {};
            geometry[MPCB200_GEO_FOOTPRINT] = radius;
            if (!controller.setRobotGeometry(geometry)) return 2;
        }
        const bool ok = controller.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &u_seq, &x_seq);
        if (!ok) return 1;
        const int n = controller.gridSize();
        double clearance = 1e300;
        for (int k = 1; k < n; ++k)
            for (const auto& o : obstacles)
                clearance = std::fmin(clearance, std::hypot(x_seq.values[3 * k] - o.x0, x_seq.values[3 * k + 1] - o.y0) - radius);
        // the same step solved cold by a controller configured with this radius
        mpcb200_config cold_cfg = cfg;
        cold_cfg.footprint_params[0] = radius;
        mpcb200::Controller cold;
        if (!cold.configure(cold_cfg, params, &obstacles, &via_points)) return 2;
        mpcb200::TimeSeries cu, cx;
        if (!cold.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &cu, &cx)) return 1;
        std::printf("step %d radius %.2f status %d iters %d clearance %.9f cold_iters %d\n", i, radius, controller.lastStatus(),
                    controller.lastIterations(), clearance, cold.lastIterations());
    }
    return 0;
}
