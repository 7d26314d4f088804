"""CPU: the fp64 reference robot (tests/robot_ref.py) checked against independent restatements, and the fp32 error of
the package's eager forward kinematics measured against it -- the error the GPU tolerances of
tests/test_gpu_robot_fp64.py are derived from."""
import xml.etree.ElementTree as ET

import numpy as np
import pytest
import torch

import primitive_ref as pr
import robot_ref as rr
from test_gpu_robot_fp64 import (CHAINS, build_robot, fk_bound, joint_values, point_bound, tessellated_box,
                                 write_chain)
from test_host import MIXED_URDF


def _oracle_chain_fp64(text, end):
    """The oracle's pytorch_kinematics restatement in fp64, its joint origins and axes taken from the URDF in fp64
    (the restatement rounds them to fp32 when it parses)."""
    from oracle import tp_pytorch_kinematics as opk
    chain = opk.build_serial_chain_from_urdf(text, end).to(dtype=torch.float64)
    joints = {j.get("name"): j for j in ET.fromstring(text).findall("joint")}
    for f in chain._frames:
        je = joints.get(f.joint.name)
        if je is None:
            continue
        o = je.find("origin")
        m = torch.eye(4, dtype=torch.float64)
        if o is not None:
            m[:3, :3] = opk.rpy_to_matrix([float(v) for v in o.get("rpy", "0 0 0").split()])
            m[:3, 3] = torch.tensor([float(v) for v in o.get("xyz", "0 0 0").split()], dtype=torch.float64)
        f.joint.offset = opk.Transform3d(matrix=m)
        ax = je.find("axis")
        a = torch.tensor([float(v) for v in ax.get("xyz").split()] if ax is not None else [1.0, 0, 0],
                         dtype=torch.float64)
        f.joint.axis = a / a.norm()
    return chain


@pytest.mark.parametrize("kind", ["test_host_mixed"] + CHAINS)
def test_fk_equals_the_oracle_restatement_in_fp64(tmp_path, kind):
    if kind == "test_host_mixed":
        text, end = MIXED_URDF, "tool"
        q = np.random.default_rng(0).uniform(-3, 3, (9, 3)).astype(np.float32)
    else:
        urdf, end, _ = write_chain(kind, tmp_path)
        text = open(urdf).read()
        q = joint_values(rr.RefRobot(text, end, path_prefix=None), text, 50, seed=1)
    ref = rr.RefRobot(text, end, path_prefix=None)
    frames = ref.frames(q)
    out = _oracle_chain_fp64(text, end).forward_kinematics(torch.from_numpy(q).double(), end_only=False)
    assert list(out) == ref.names
    for f, name in enumerate(ref.names):
        np.testing.assert_allclose(frames[:, f], out[name].get_matrix().numpy(), rtol=0, atol=1e-12, err_msg=name)


def test_primitive_links_equal_primitive_ref_on_the_product_descriptors(tmp_path):
    """The URDF numbers -> link SDF mapping (box size / 2, cylinder length / 2, sphere radius) against the package's
    descriptors of the same visuals through tests/primitive_ref.py: equal up to the fp32 rounding of the extents."""
    robot, ref, _ = build_robot("mixed", tmp_path, device="cpu")
    assert len(ref.links) == len(robot.sdf.sdfs) == 8
    assert [l.kind for l in ref.links] == ["box", "cylinder", "box", "sphere", "cylinder", "box", "sphere",
                                           "cylinder"]
    q = np.random.default_rng(3).uniform(-0.3, 0.3, (20_000, 3))
    for link, s in zip(ref.links, robot.sdf.sdfs):
        d = s.native_desc("cpu")
        v, g, _, _ = link.evaluate(q)
        rv, rg = pr.primitive_ref(d, q)
        assert np.abs(v - rv).max() < 1e-8
        decided = pr.second_gap(d, q) > 1e-6
        # the extents differ by their fp32 rounding (< 1e-8 here), which turns the outside gradient by up to that / |v|
        tol = 1e-9 + 1e-7 / np.abs(rv)
        assert decided.mean() > 0.99 and (np.abs(g - rg).max(1) <= tol)[decided].all()


def test_mesh_distance_equals_the_box_on_a_tessellated_box():
    """Brute-force point-triangle distance of the tessellated box against box_ref: values everywhere, gradients
    wherever neither rule has a tie (the box's inside-rule axes, the mesh's faces of different sides)."""
    size = np.array([0.3, 0.12, 0.2])
    v, f = tessellated_box(3)
    link = rr.Link(0, np.eye(4), "mesh", vertices=v * size, faces=f)
    rng = np.random.default_rng(4)
    q = np.concatenate([rng.uniform(-1, 1, (20_000, 3)) * size,                          # inside and near
                        rng.uniform(-1, 1, (5_000, 3)) * size * 0.51,                      # mostly inside
                        rng.normal(size=(5_000, 3)) * 2])                                  # far
    val, g, gap, _ = link.evaluate(q)
    bv, bg = pr.box_ref(size / 2, q)
    np.testing.assert_allclose(val, bv, rtol=0, atol=1e-13)
    e = np.sort(np.abs(q) - size / 2, axis=1)
    clear = (gap > 0) & ((bv > 0) | (e[:, 2] - e[:, 1] > 1e-9))
    assert clear.mean() > 0.95 and (val < 0).mean() > 0.2 and (np.abs(val) < rr.MESH_SHELL).any()
    np.testing.assert_allclose(g[clear], bg[clear], rtol=0, atol=1e-9)


@pytest.mark.parametrize("kind", CHAINS)
def test_eager_fp32_fk_error_is_within_the_derived_bounds(tmp_path, kind):
    """The package's eager fp32 forward kinematics on the CPU against the fp64 reference: every entry of every
    object->link transform within fk_bound, every transformed point within point_bound, and the observed error at
    least a tenth of the bound (the bound is not loose by more than 10x)."""
    robot, ref, text = build_robot(kind, tmp_path, device="cpu")
    assert robot._fk_plan is None                         # the CPU has no native path
    q = joint_values(ref, text, 2000, seed=5)
    robot.set_joint_configuration(torch.from_numpy(q))
    S = len(ref.links)
    m = robot.object_to_link_frames.get_matrix().reshape(S, -1, 4, 4).double().numpy()
    mref = ref.object_to_link(q)
    reach = ref.reach(q)
    nf = np.array([l.frame + 1 for l in ref.links])[:, None]
    r_fk = (np.abs(m - mref)[..., :3, :].max((-1, -2)) / fk_bound(nf, reach)).max()
    p = np.random.default_rng(6).uniform(-1, 1, (64, 3)) * (1 + reach.max())
    p = p.astype(np.float32).astype(np.float64)
    dq = np.linalg.norm(np.einsum("saij,pj->sapi", m[..., :3, :3] - mref[..., :3, :3], p)
                        + (m - mref)[..., None, :3, 3], axis=-1)
    r_pt = (dq / point_bound(nf[..., None], reach[..., None], np.linalg.norm(p, axis=1))).max()
    print(f"{kind}: eager fp32 fk error / fk_bound = {r_fk:.3f}, point error / point_bound = {r_pt:.3f}")
    assert r_fk <= 1 and r_pt <= 1
    assert r_fk >= 0.1
