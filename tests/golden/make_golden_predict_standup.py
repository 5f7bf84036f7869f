"""Golden vectors for the standup boxes the reference's axis-aligned NMS compares (mg_head.py:1009-1017:
center_to_corner_box2d, then corner_to_standup_nd; det3d/core/bbox/box_torch_ops.py:11-19,220-281,349-407).  Run in the
development container (needs /root/reference):

    python tests/golden/make_golden_predict_standup.py

The reference functions are lifted from their source file with `ast` (the module imports compiled extensions that are
not installed) and executed as they are; only the data is stored."""
import ast
import os

import numpy as np
import torch

REF = "/root/reference/det3d/core/bbox/box_torch_ops.py"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "predict_standup.npz")
NAMES = ("torch_to_np_dtype", "corners_nd", "rotation_2d", "center_to_corner_box2d", "corner_to_standup_nd")


def lift(path, names):
    src = open(path).read()
    nodes = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in names]
    ns = {"torch": torch, "np": np, "tstack": torch.stack}
    exec(compile(ast.Module(body=nodes, type_ignores=[]), path, "exec"), ns)
    return ns


def main():
    ns = lift(REF, NAMES)
    rng = np.random.default_rng(11)
    n = 1000
    centers = rng.uniform(-60.0, 60.0, size=(n, 2)).astype(np.float32)
    dims = rng.uniform(0.2, 12.0, size=(n, 2)).astype(np.float32)
    angles = rng.uniform(-7.0, 7.0, size=n).astype(np.float32)
    special = np.float32([0.0, -0.0, np.pi / 2, -np.pi / 2, np.pi, -np.pi, np.pi / 4, 3 * np.pi / 4, 2 * np.pi, 1e-7])
    angles[: special.shape[0]] = special
    corners = ns["center_to_corner_box2d"](torch.from_numpy(centers), torch.from_numpy(dims), torch.from_numpy(angles))
    standup = ns["corner_to_standup_nd"](corners)
    np.savez_compressed(OUT, centers=centers, dims=dims, angles=angles, corners=corners.numpy(), standup=standup.numpy())
    print("wrote", OUT, n, "boxes")


if __name__ == "__main__":
    main()
