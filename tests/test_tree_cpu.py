"""CPU tier: kinematic trees (kinematics.Chain, build_chain_from_urdf) against the fp64 tree reference (tests/tree_ref.py).

1. The parser: frame order (depth-first pre-order, children in joint document order), joint order, parents and
   .children on robot_ref's mixed chain read as a tree (its side branch is a real branch), the hand and the gripper;
   every malformed tree raises ValueError.
2. The eager fp32 forward kinematics against fp64 within the tree's bound.
3. RobotSDF.joint_moves_link and self_collision_pairs on trees against the ancestor and path rules of the reference,
   and a Chain and a SerialChain of every serial URDF give equal masks.
4. The native plan: parents and save slots, pvb_fk_tree's refusals (a parents array that is not a pre-order, bad links
   and joint columns), the shared walk (pvb_device.cuh fk_walk, host build) against fp64, and the serial walk and the
   tree walk on the same chain giving identical bits."""
import ctypes

import numpy as np
import pytest
import torch

import hostsim_lib
import robot_ref
import workloads
from robot_ref import CHAINS, fk_bound, joint_values, write_chain
from tree_ref import RefTree, build_tree, write_tree


def _chain(text):
    import pytorch_volumetric_b200 as pv
    return pv.build_chain_from_urdf(text)


# ---------------------------------------------------------------- 1. the parser
def test_mixed_chain_read_as_a_tree(tmp_path):
    path, _ = robot_ref.write_mixed(str(tmp_path))
    c = _chain(open(path).read())
    names = c.get_frame_names(exclude_fixed=False)
    # the side branch hangs off l4; its joint comes last in the document, after l5's
    assert names == ["base", "l1", "l2", "l3", "l4", "l5", "l6", "l7", "l8", "l9", "side"]
    assert c.frame_parents() == [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 4]
    assert [f.name for f in c.find_frame("l4").children] == ["l5", "side"]
    assert c.find_frame("side").children == [] and c.find_frame("l4").joint.joint_type == "prismatic"
    assert c.get_joint_parameter_names() == ["j_l1", "j_l2", "j_l4", "j_l5", "j_l6", "j_l8", "j_l9", "j_side"]
    assert c.get_frame_names() == ["l1", "l2", "l4", "l5", "l6", "l8", "l9", "side"]
    assert c.n_joints == 8
    with pytest.raises(ValueError):
        c.forward_kinematics(torch.zeros(8), end_only=True)


def test_hand_and_gripper_structure(tmp_path):
    c = _chain(open(workloads.write_hand(str(tmp_path / "h"))).read())
    names = c.get_frame_names(exclude_fixed=False)
    assert len(names) == 23 and c.n_joints == 21
    palm = names.index("palm")
    assert [f.name for f in c.find_frame("palm").children] == [f"finger{i}_knuckle" for i in range(4)] + ["thumb_base"]
    parents = c.frame_parents()
    for child in c.find_frame("palm").children:
        assert parents[names.index(child.name)] == palm
    assert c.find_frame("thumb_base").joint.joint_type == "fixed"
    joints = c.get_joint_parameter_names()
    assert joints[:2] == ["wrist_pitch", "wrist_roll"] and joints[-3:] == ["thumb_flex1", "thumb_flex2", "thumb_flex3"]
    assert joints[2:6] == ["finger0_abduct", "finger0_flex1", "finger0_flex2", "finger0_flex3"]
    g = _chain(open(workloads.write_gripper_tree(str(tmp_path / "g"))).read())
    assert g.get_frame_names(exclude_fixed=False) == ["base", "link1", "link2", "palm", "finger_a", "finger_a_tip",
                                                      "finger_b1", "finger_b2"]
    assert g.frame_parents() == [-1, 0, 1, 2, 3, 4, 3, 6]
    assert g.get_joint_parameter_names() == ["j1", "j2", "j3", "finger_a_slide", "finger_b_base", "finger_b_tip"]
    assert workloads.tree_configurations(workloads.write_gripper_tree(str(tmp_path / "g2")), 7).shape == (7, 6)


_LINKS = '<link name="a"/><link name="b"/><link name="c"/>'
_J = '<joint name="{n}" type="revolute"><parent link="{p}"/><child link="{c}"/></joint>'


@pytest.mark.parametrize("body,what", [
    (_LINKS + _J.format(n="j1", p="a", c="b"), "two roots"),
    (_LINKS + _J.format(n="j1", p="a", c="b") + _J.format(n="j2", p="b", c="c") + _J.format(n="j3", p="c", c="a"),
     "no root"),
    (_LINKS + _J.format(n="j1", p="a", c="b") + _J.format(n="j2", p="a", c="c") + _J.format(n="j3", p="b", c="c"),
     "two parents"),
    (_LINKS + _J.format(n="j1", p="a", c="b") + _J.format(n="j2", p="b", c="d"), "missing child"),
    (_LINKS + _J.format(n="j1", p="a", c="b") + _J.format(n="j2", p="x", c="c"), "missing parent"),
    ('<link name="a"/><link name="b"/><link name="c"/><link name="d"/>' + _J.format(n="j1", p="a", c="b") +
     _J.format(n="j2", p="c", c="d") + _J.format(n="j3", p="d", c="c"), "cycle off the root"),
])
def test_malformed_trees_raise(body, what):
    with pytest.raises(ValueError):
        _chain(f'<robot name="r">{body}</robot>')


# ---------------------------------------------------------------- 2. eager forward kinematics
@pytest.mark.parametrize("kind", ["mixed", "hand", "gripper", "tree64", "tree65"])
def test_eager_fk_against_fp64(tmp_path, kind):
    robot, ref, text = build_tree(kind, tmp_path, device="cpu")
    assert robot._fk_plan is None
    assert robot.frame_names == ref.names and robot.chain.frame_parents() == ref.parents
    q = joint_values(ref, text, 500, seed=3)
    robot.set_joint_configuration(torch.from_numpy(q))
    S = len(ref.links)
    m = robot.object_to_link_frames.get_matrix().reshape(S, -1, 4, 4).double().numpy()
    err = np.abs(m - ref.object_to_link(q))[..., :3, :].max((-1, -2))
    bound = fk_bound(ref.path_frames()[:, None], ref.reach(q))
    print(f"{kind}: eager fk error / bound max {(err / bound).max():.3f}")
    assert (err <= bound).all()


# ---------------------------------------------------------------- 3. the structure masks
@pytest.mark.parametrize("kind", ["mixed", "hand", "gripper", "tree64"])
def test_masks_follow_the_tree(tmp_path, kind):
    robot, ref, _ = build_tree(kind, tmp_path, device="cpu")
    assert np.array_equal(robot.joint_moves_link().numpy(), ref.moves())
    assert np.array_equal(robot.self_collision_pairs().numpy(), ref.pairs())


@pytest.mark.parametrize("kind", CHAINS + ["write_arm"])
def test_serial_urdfs_give_the_serial_masks(tmp_path, kind):
    import pytorch_volumetric_b200 as pv
    if kind == "write_arm":
        urdf, end = workloads.write_arm(str(tmp_path))
        prim = False
    else:
        urdf, end, prim = write_chain(kind, tmp_path)
    text = open(urdf).read()
    serial = pv.RobotSDF(pv.build_serial_chain_from_urdf(text, end).to(dtype=torch.float64), path_prefix=str(tmp_path),
                         primitive_visuals=prim)
    if kind.startswith("mixed"):        # the side branch: a tree of the same URDF has one more frame and joint
        text = text.replace(text[text.index('<link name="side">'):text.index("</robot>")], "")
    tree = pv.RobotSDF(pv.build_chain_from_urdf(text).to(dtype=torch.float64), path_prefix=str(tmp_path),
                       primitive_visuals=prim)
    assert tree.frame_names == serial.frame_names and tree.joint_names == serial.joint_names
    assert torch.equal(tree.joint_moves_link(), serial.joint_moves_link())
    assert torch.equal(tree.self_collision_pairs(), serial.self_collision_pairs())


# ---------------------------------------------------------------- 4. the native plan and the shared walk
def _slots(parents):
    n = len(parents)
    p = np.ascontiguousarray(parents, dtype=np.int32)
    load, save = np.empty(n, np.int8), np.empty(n, np.int8)
    n_saves = ctypes.c_int(-1)
    bad = hostsim_lib.lib().simfk_tree_slots(hostsim_lib._p(p), ctypes.c_int(n), hostsim_lib._p(load),
                                             hostsim_lib._p(save), ctypes.byref(n_saves))
    return bad, load, save, n_saves.value


def test_save_slots(tmp_path):
    # the gripper: the palm (frame 3) saves, finger_b1 (frame 6) reloads it
    bad, load, save, n = _slots([-1, 0, 1, 2, 3, 4, 3, 6])
    assert bad == -1 and n == 1
    assert save.tolist() == [-1, -1, -1, 0, -1, -1, -1, -1] and load.tolist() == [-1] * 6 + [0, -1]
    # a chain saves nothing
    bad, load, save, n = _slots(list(range(-1, 31)))
    assert bad == -1 and n == 0 and (load == -1).all() and (save == -1).all()
    # every tree: a frame whose parent is not the frame before reloads the parent's slot; slots on one root path are
    # distinct, so no frame overwrites a pose an open branch still needs; at most the depth is live
    for kind in ("mixed", "hand", "tree64"):
        ref = RefTree(open(write_tree(kind, tmp_path / kind)[0]).read(), path_prefix=None)
        bad, load, save, n = _slots(ref.parents)
        assert bad == -1 and n <= max(ref.depth)
        for f, p in enumerate(ref.parents):
            if f > 0 and p != f - 1:
                assert load[f] == save[p] >= 0
            else:
                assert load[f] == -1
            path_slots = [save[a] for a in ref.root_path(f) if save[a] >= 0]
            assert len(path_slots) == len(set(path_slots))
        assert n == (save.max() + 1 if (save >= 0).any() else 0)


@pytest.mark.parametrize("parents,bad", [
    ([0, 0, 1], 0),                   # the root has a parent
    ([-1, -1, 1], 1),                 # a second root
    ([-1, 1, 1], 1),                  # its own parent
    ([-1, 0, 3, 0], 2),               # a parent after the frame
    ([-1, 0, 1, 0, 2], 4),            # frame 4's parent 2 is neither frame 3 nor one of its ancestors
    ([-1, 0, 0, 1], 3),               # frame 3 returns to frame 1's subtree after frame 2 left it
])
def test_pre_order_violations_are_refused(built_lib, parents, bad):
    from pytorch_volumetric_b200 import _native as nat
    assert _slots(parents)[0] == bad
    n = len(parents)
    frames = (nat.FkFrame * n)()
    links = (nat.FkLink * 1)()
    p = (ctypes.c_int32 * n)(*parents)
    rc = built_lib.pvb_fk_tree(frames, p, n, links, 1, None, 0, 0, None, None)
    assert rc == hostsim_lib.PVB_ERR_INVALID
    assert f"frame {bad} ".encode() in built_lib.pvb_last_error()


def test_entry_point_refusals(built_lib):
    from pytorch_volumetric_b200 import _native as nat
    n = 4
    frames = (nat.FkFrame * n)()
    frames[1].joint_type, frames[1].q_index = nat.FK_REVOLUTE, 0
    parents = (ctypes.c_int32 * n)(-1, 0, 1, 1)

    def links(*spec):
        arr = (nat.FkLink * len(spec))()
        for k, (frame, slot) in enumerate(spec):
            arr[k].frame, arr[k].slot = frame, slot
        return arr

    def call(lk, n_joints=1, n_frames=n, out=None, n_cfg=0, q=None):
        return built_lib.pvb_fk_tree(frames, parents, n_frames, lk, len(lk), q, n_cfg, n_joints, out, None)

    assert call(links((0, 0), (2, 1), (3, 2))) == 0
    for bad in (links((2, 0), (0, 1)),            # not sorted by frame
                links((0, 0), (1, 0)),            # one slot twice
                links((0, 0), (1, 2)),            # a slot past n_links
                links((0, 0), (4, 1))):           # a frame past n_frames
        assert call(bad) == hostsim_lib.PVB_ERR_INVALID and b"distinct slots" in built_lib.pvb_last_error()
    assert call(links((0, 0)), n_joints=0) == hostsim_lib.PVB_ERR_INVALID
    assert b"frame 1 reads joint value 0 of 0" in built_lib.pvb_last_error()
    assert call(links((0, 0)), n_frames=65) == hostsim_lib.PVB_ERR_INVALID
    q = np.zeros(1, np.float32)
    assert call(links((0, 0)), out=1 << 12 | 4, n_cfg=1, q=q.ctypes.data) == hostsim_lib.PVB_ERR_INVALID
    assert b"16-byte aligned" in built_lib.pvb_last_error()


def _walk(frames, parents, links, q):
    """Host walk (simfk_serial when parents is None, simfk_tree otherwise) -> [n_links, A, 4, 4] fp32."""
    A, J = q.shape
    q = np.ascontiguousarray(q, dtype=np.float32)
    out = np.zeros((len(links) * A, 4, 4), np.float32)
    if parents is None:
        hostsim_lib.lib().simfk_serial(frames, len(frames), links, len(links), hostsim_lib._p(q), A, J,
                                       hostsim_lib._p(out))
    else:
        assert hostsim_lib.lib().simfk_tree(frames, parents, len(frames), links, len(links), hostsim_lib._p(q), A, J,
                                            hostsim_lib._p(out)) == -1
    return out.reshape(len(links), A, 4, 4)


def _links_of(robot):
    """RobotSDF's pvb_fk_link array for its chain (the packing _make_fk_plan does on a CUDA device)."""
    from pytorch_volumetric_b200 import _native as nat
    frame_of = {f.link.name: i for i, f in enumerate(robot.chain._frames)}
    inv = robot._mesh_from_link.to(torch.float32)
    order = sorted(range(len(robot.sdf_to_link_name)), key=lambda s: frame_of[robot.sdf_to_link_name[s]])
    links = (nat.FkLink * len(order))()
    for k, s in enumerate(order):
        for e in range(12):
            links[k].mesh_from_link[e] = float(inv[s, e // 4, e % 4])
        links[k].frame, links[k].slot = frame_of[robot.sdf_to_link_name[s]], s
    return links


@pytest.mark.parametrize("kind", ["mixed", "hand", "gripper", "tree64"])
def test_host_walk_against_fp64(tmp_path, kind):
    robot, ref, text = build_tree(kind, tmp_path, device="cpu")
    frames, parents = robot.chain.native_fk_frames()
    assert list(parents) == ref.parents
    q = joint_values(ref, text, 300, seed=8)
    m = _walk(frames, parents, _links_of(robot), q).astype(np.float64)
    err = np.abs(m - ref.object_to_link(q))[..., :3, :].max((-1, -2))
    bound = fk_bound(ref.path_frames()[:, None], ref.reach(q))
    print(f"{kind}: host walk error / bound max {(err / bound).max():.3f}")
    assert (err <= bound).all() and (m[..., 3, :] == [0, 0, 0, 1]).all()


@pytest.mark.parametrize("kind", ["limit32", "arm", "prim_arm"])
def test_serial_plan_and_explicit_parents_give_identical_bits(tmp_path, kind):
    import pytorch_volumetric_b200 as pv
    urdf, end, prim = write_chain(kind, tmp_path)
    text = open(urdf).read()
    serial = pv.build_serial_chain_from_urdf(text, end)
    tree = pv.build_chain_from_urdf(text)
    robot = pv.RobotSDF(tree, path_prefix=str(tmp_path), primitive_visuals=prim)
    frames, parents = tree.native_fk_frames()
    assert list(parents) == list(range(-1, len(frames) - 1))
    s_frames = serial.native_fk_frames()
    assert bytes(s_frames) == bytes(frames)
    ref = robot_ref.RefRobot(text, end, primitive_visuals=prim, path_prefix=None)
    q = joint_values(ref, text, 200, seed=4)
    links = _links_of(robot)
    assert np.array_equal(_walk(s_frames, None, links, q), _walk(frames, parents, links, q))
