// controller_model.cpp -- the C++ mirror with a footprint type that changes at run time (TEST INFRASTRUCTURE): the demo's scene
// with a circular robot of radius 0.1 that picks up a cart from the second step on -- a polygon footprint, set by
// Controller::setRobotGeometry (a record holding the radius and the polygon) and then Controller::setRobotModel, with no
// reconfigure, so the later steps warm-start.  Per step it prints the footprint type in effect, the status and iterations, the
// smallest clearance of the plan (distance of the footprint to the nearest point obstacle) and the iterations of a cold solve of
// the same step by a controller configured with that footprint.
#include <cmath>
#include <cstdio>
#include <vector>

#include "../../include/mpcb200_controller.hpp"

static const double CART[4][2] = {{-0.15, -0.2}, {0.35, -0.2}, {0.35, 0.2}, {-0.15, 0.2}};

// distance of point (px, py) to the footprint of a robot at pose (x, y, theta): a circle, or the cart polygon (> 0 outside)
static double footprint_distance(int footprint, double radius, double x, double y, double theta, double px, double py)
{
    if (footprint == MPCB200_FOOTPRINT_CIRCULAR) return std::hypot(px - x, py - y) - radius;
    const double c = std::cos(theta), s = std::sin(theta);
    const double lx = c * (px - x) + s * (py - y), ly = -s * (px - x) + c * (py - y);   // the point in the robot frame
    double d = 1e300;
    bool inside = true;
    for (int i = 0; i < 4; ++i)
    {
        const double* a = CART[i];
        const double* b = CART[(i + 1) % 4];
        const double ex = b[0] - a[0], ey = b[1] - a[1];
        double t = ((lx - a[0]) * ex + (ly - a[1]) * ey) / (ex * ex + ey * ey);
        t = t < 0 ? 0 : (t > 1 ? 1 : t);
        d = std::fmin(d, std::hypot(lx - a[0] - t * ex, ly - a[1] - t * ey));
        inside = inside && (ex * (ly - a[1]) - ey * (lx - a[0])) > 0;   // counter-clockwise vertices
    }
    return inside ? -d : d;
}

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
    int footprint = MPCB200_FOOTPRINT_CIRCULAR;
    for (int i = 0; i < 4; ++i)
    {
        if (i == 1)   // a cart picked up: geometry first (the radius still valid for the circle), then the footprint type
        {
            footprint = MPCB200_FOOTPRINT_POLYGON;
            double geometry[MPCB200_GEOMETRY_WORDS] = {};
            geometry[MPCB200_GEO_FOOTPRINT] = cfg.footprint_params[0];
            geometry[MPCB200_GEO_N_POLY] = 4;
            for (int v = 0; v < 4; ++v) { geometry[MPCB200_GEO_POLY_XY + 2 * v] = CART[v][0]; geometry[MPCB200_GEO_POLY_XY + 2 * v + 1] = CART[v][1]; }
            if (!controller.setRobotGeometry(geometry)) return 2;
            if (!controller.setRobotModel(MPCB200_ROBOT_UNICYCLE, footprint)) return 2;
        }
        const bool ok = controller.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &u_seq, &x_seq);
        if (!ok) return 1;
        const int n = controller.gridSize();
        double clearance = 1e300;
        for (int k = 1; k < n; ++k)
            for (const auto& o : obstacles)
                clearance = std::fmin(clearance, footprint_distance(footprint, cfg.footprint_params[0], x_seq.values[3 * k],
                                                                    x_seq.values[3 * k + 1], x_seq.values[3 * k + 2], o.x0, o.y0));
        // the same step solved cold by a controller configured with this footprint
        mpcb200_config cold_cfg = cfg;
        cold_cfg.footprint_type = footprint;
        cold_cfg.n_poly = 4;
        for (int v = 0; v < 4; ++v) { cold_cfg.poly_xy[2 * v] = CART[v][0]; cold_cfg.poly_xy[2 * v + 1] = CART[v][1]; }
        mpcb200::Controller cold;
        if (!cold.configure(cold_cfg, params, &obstacles, &via_points)) return 2;
        mpcb200::TimeSeries cu, cx;
        if (!cold.step(x0, xf, mpcb200::Twist(), 0.05, 0.05 * i, &cu, &cx)) return 1;
        std::printf("step %d footprint %d status %d iters %d clearance %.9f cold_iters %d\n", i, footprint, controller.lastStatus(),
                    controller.lastIterations(), clearance, cold.lastIterations());
    }
    return 0;
}
