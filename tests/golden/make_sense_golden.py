"""Writes tests/golden/sense_reference.npz: the reference's own depth renderer (oracle/_ref/libref_depth.so, built by oracle/depth.mk from
local_sensing/src/depth_render.cu) on the scenes and poses of sense_oracle.golden_cases(), with the default camera. Each pose's
double[16] camera-from-world is the one the library defines (sense_oracle.pose); the reference kernel takes it as render_pose does.
Needs an H100 and the library; run once from the repository root: python tests/golden/make_sense_golden.py"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "implicit-sdf-planner_b200", "py"))
import isdf_b200 as I  # noqa: E402
import sense_oracle as SO  # noqa: E402


def main():
    p = I.sense_params()
    out = {}
    names = []
    for name, (xyz, pos, quat) in SO.golden_cases().items():
        T = np.array([SO.pose(pos[q], quat[q], np.array(p.cam_to_body[:]))[1] for q in range(len(pos))])
        out[f"{name}/xyz"], out[f"{name}/pos"], out[f"{name}/quat"], out[f"{name}/T"] = xyz, pos, quat, T
        out[f"{name}/depth"] = SO.ref_render(xyz, T, p)
        names.append(name)
    np.savez_compressed(os.path.join(HERE, "sense_reference.npz"), names=np.array(names), **out)
    print("wrote", os.path.join(HERE, "sense_reference.npz"), {n: out[f"{n}/depth"].shape for n in names})


if __name__ == "__main__":
    main()
