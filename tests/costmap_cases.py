"""Random costmaps of the costmap-conversion, solver-chain and pose-feasibility tests."""
import numpy as np


def random_costmap(rng, W, H, density=0.01):
    cost = rng.choice(np.array([0, 1, 100, 253, 255], dtype=np.uint8), size=(H, W))   # free, inflated, inscribed, unknown
    cost[rng.random((H, W)) < density] = 254                                          # costmap_2d::LETHAL_OBSTACLE
    cost[:, W - 1] = 254; cost[H - 1, :] = 254   # the reference's loops stop one cell short of both upper edges
    return cost


def costmap_scene(B, density, seed, ahead=3.0):
    """robots on random costmaps, goals 3 m ahead, the cells around start and goal cleared"""
    rng = np.random.default_rng(seed)
    W, H, res = 200, 160, 0.05
    cost = np.stack([random_costmap(rng, W, H, density) for _ in range(B)])
    cost[:, :, W - 1] = 0; cost[:, H - 1, :] = 0
    origin = rng.uniform(-3, 3, (B, 2))
    pose = np.concatenate([origin + rng.uniform(2.5, 4.5, (B, 2)), rng.uniform(-np.pi, np.pi, (B, 1))], axis=1)
    goal = pose.copy(); goal[:, 0] += ahead * np.cos(pose[:, 2]); goal[:, 1] += ahead * np.sin(pose[:, 2])
    yy, xx = np.mgrid[0:H, 0:W]
    for b in range(B):
        cx, cy = origin[b, 0] + (xx + 0.5) * res, origin[b, 1] + (yy + 0.5) * res
        for p in (pose[b], goal[b]):
            cost[b][(cx - p[0]) ** 2 + (cy - p[1]) ** 2 < 0.7 ** 2] = 0
    return cost, origin, res, pose, goal


def feasibility_cases(rng, n_cases, W=80, H=70, res=0.05, n=14):
    """costmaps with lethal, unknown and inscribed cells and noisy pose trajectories across them: (cost, origin, poses)"""
    out = []
    for c in range(n_cases):
        cost = np.zeros((H, W), dtype=np.uint8)
        cost[rng.random((H, W)) < 0.004] = 254
        cost[rng.random((H, W)) < 0.01] = 255
        cost[rng.random((H, W)) < 0.01] = 253
        origin = rng.uniform(-1, 1, 2)
        start = origin + rng.uniform(0.3, 0.8, 2)
        goal = origin + np.array([W * res, H * res]) - rng.uniform(-0.2, 0.8, 2)   # sometimes leaves the map
        t = np.linspace(0, 1, n)[:, None]
        xy = start + t * (goal - start) + rng.normal(0, 0.02, (n, 2))
        th = np.arctan2(goal[1] - start[1], goal[0] - start[0]) + np.cumsum(rng.normal(0, 0.25, n))
        out.append((cost, origin, np.column_stack([xy, th])))
    return out
