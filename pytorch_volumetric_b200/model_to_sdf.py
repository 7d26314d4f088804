"""RobotSDF: one SDF per link mesh, posed by batched forward kinematics, min over links in one fused kernel.

API mirror of the reference's src/pytorch_volumetric/model_to_sdf.py (RobotSDF :12-125,
cache_link_sdf_factory :128-133, aabb_to_ordered_end_points :136-171): same constructor arguments, attributes,
output shapes and state semantics.  `chain` is duck-typed on the pytorch_kinematics Chain surface listed in
kinematics.py; every query is a single pvb_composed_query launch.
"""
import logging
import math
import typing

import numpy as np
import torch

from . import sdf
from .transforms import Transform3d, invert_rigid, matrix_of

logger = logging.getLogger(__file__)


_PRIMITIVES = ("box", "cylinder", "sphere")


def _mesh_visuals(chain, frame_names, primitives=False):
    """(link name, visual) for every mesh visual along the chain -- and with `primitives` every box, cylinder and
    sphere visual -- in frame order; other geometry types are reported and skipped, like the reference does
    (model_to_sdf.py:41-56)."""
    for fname in frame_names:
        link = chain.find_frame(fname).link
        for vis in link.visuals:
            if vis.geom_type == "mesh" or (primitives and vis.geom_type in _PRIMITIVES):
                yield link.name, vis
            else:
                logger.warning("Cannot handle non-mesh link visual type %s for %s", vis, link.name)


def _primitive_sdf(vis):
    """BoxSDF / CylinderSDF / SphereSDF of a URDF primitive visual (pytorch_kinematics' geom_param conventions: box
    size [x, y, z], cylinder (radius, length), sphere radius)."""
    if vis.geom_type == "box":
        return sdf.BoxSDF(vis.geom_param)
    if vis.geom_type == "cylinder":
        radius, length = vis.geom_param
        return sdf.CylinderSDF(radius, length)
    radius = sdf._check_extent("sphere radius", vis.geom_param)
    return sdf.SphereSDF(radius)


def _primitive_surface(link_sdf, n, rng):
    """[n, 3] fp64 area-uniform samples of the surface of a BoxSDF, CylinderSDF or SphereSDF, in its own frame."""
    if isinstance(link_sdf, sdf.SphereSDF):
        d = rng.normal(size=(n, 3))
        return float(link_sdf.radius) * d / np.linalg.norm(d, axis=1, keepdims=True)
    u = rng.uniform(-1.0, 1.0, size=(n, 3))
    if isinstance(link_sdf, sdf.BoxSDF):
        h = np.asarray(link_sdf._half, dtype=np.float64)
        area = np.array([h[1] * h[2], h[0] * h[2], h[0] * h[1]])        # face pair normal to x, y, z
        axis = rng.choice(3, size=n, p=area / area.sum())
        out = u * h
        rows = np.arange(n)
        out[rows, axis] = np.where(rng.uniform(size=n) < 0.5, -1.0, 1.0) * h[axis]
        return out
    if isinstance(link_sdf, sdf.CylinderSDF):
        r, hl = float(link_sdf.radius), 0.5 * float(link_sdf.length)
        side, cap = 2.0 * np.pi * r * 2.0 * hl, np.pi * r * r          # side, one cap
        region = rng.choice(3, size=n, p=np.array([side, cap, cap]) / (side + 2.0 * cap))
        phi = rng.uniform(0.0, 2.0 * np.pi, size=n)
        rho = np.where(region == 0, r, r * np.sqrt(rng.uniform(size=n)))
        z = np.where(region == 0, u[:, 2] * hl, np.where(region == 1, hl, -hl))
        return np.stack([rho * np.cos(phi), rho * np.sin(phi), z], axis=1)
    raise ValueError(f"no analytic surface for {type(link_sdf).__name__}")


class RobotSDF(sdf.ObjectFrameSDF):
    """SDF of an articulated robot in its base frame.

    The joint configuration -- a single vector or an arbitrarily batched set of them -- is state: it is installed
    with `set_joint_configuration` and determines both the values and the leading shape of what `__call__` returns.
    """

    def __init__(self, chain, default_joint_config=None, path_prefix='',
                 link_sdf_cls: typing.Callable[[sdf.ObjectFactory], sdf.ObjectFrameSDF] = sdf.MeshSDF,
                 primitive_visuals=False):
        """
        :param chain: kinematic description; only mesh visuals become SDFs (and primitives, see primitive_visuals)
        :param default_joint_config: joint values installed at construction (zeros when None)
        :param path_prefix: directory the relative mesh paths of the description are resolved against
        :param link_sdf_cls: callable turning a link's ObjectFactory into its ObjectFrameSDF (mesh visuals only)
        :param primitive_visuals: EXTENSION (the reference skips them with a warning, which stays the default): box,
        cylinder and sphere visuals become BoxSDF / CylinderSDF / SphereSDF links, in frame / visual order with the
        mesh links and placed by their <origin> like them; the fused kernels evaluate them analytically
        """
        self.chain = chain
        self.dtype, self.device = chain.dtype, chain.device
        self.q = None
        self.configuration_batch = None
        self.object_to_link_frames = None
        self.joint_names = chain.get_joint_parameter_names()
        self.frame_names = chain.get_frame_names(exclude_fixed=False)

        visuals = list(_mesh_visuals(chain, self.frame_names, primitive_visuals))
        self.sdf_to_link_name = [name for name, _ in visuals]
        link_sdfs = []
        self._link_factories = []          # the MeshObjectFactory of every mesh link, None for primitives
        for name, vis in visuals:
            logger.info("%s offset %s", name, vis.offset)
            if vis.geom_type != "mesh":
                link_sdfs.append(_primitive_sdf(vis))
                self._link_factories.append(None)
                continue
            mesh_file, mesh_scale = vis.geom_param[0], vis.geom_param[1]
            factory = sdf.MeshObjectFactory(mesh_file, scale=mesh_scale, path_prefix=path_prefix)
            link_sdfs.append(link_sdf_cls(factory))
            self._link_factories.append(factory)
        self._surface_points = {}
        # visual origin of every mesh inside its link frame, stacked link-major
        self.offset_transforms = Transform3d(
            matrix=torch.cat([matrix_of(vis.offset) for _, vis in visuals]).to(device=self.device, dtype=self.dtype))
        # inverse of the visual offsets, once (general inverse: a scaled <visual><origin> is not rigid)
        self._mesh_from_link = self.offset_transforms.inverse().get_matrix()
        self.sdf: typing.Optional[sdf.ComposedSDF] = sdf.ComposedSDF(link_sdfs, None)
        self._fk_plan = self._make_fk_plan()
        self.set_joint_configuration(default_joint_config)

    #: set False to force the eager forward_kinematics of the chain object (what foreign pk chains always get)
    native_fk = True

    def _make_fk_plan(self):
        """(pvb_fk_frame[], pvb_fk_link[], parents) for the native forward kinematics when the chain is this package's
        SerialChain (pvb_fk_serial, parents None) or Chain (pvb_fk_tree, its int32 parents) in float32 on a CUDA device
        and within the entry point's limits; None otherwise (duck-typed pytorch_kinematics chains keep their own FK)."""
        from . import _native as nat
        from .kinematics import Chain, SerialChain
        tree = isinstance(self.chain, Chain)
        max_links = nat.FK_TREE_MAX_LINKS if tree else nat.FK_MAX_LINKS
        if not (tree or isinstance(self.chain, SerialChain)) or self.dtype != torch.float32 or \
                torch.device(self.device).type != "cuda" or not (1 <= len(self.sdf_to_link_name) <= max_links):
            return None
        packed = self.chain.native_fk_frames()
        if packed is None:
            return None
        frames, parents = packed if tree else (packed, None)
        frame_of = {f.link.name: i for i, f in enumerate(self.chain._frames)}
        inv = self._mesh_from_link.detach().to("cpu", torch.float32)
        if not bool((inv[:, 3] == torch.tensor([0.0, 0.0, 0.0, 1.0])).all()):
            return None                       # a projective visual offset: not an [A | t] matrix
        order = sorted(range(len(self.sdf_to_link_name)), key=lambda s: frame_of[self.sdf_to_link_name[s]])
        links = (nat.FkLink * len(order))()
        for k, s_idx in enumerate(order):
            for r in range(3):
                for c in range(4):
                    links[k].mesh_from_link[4 * r + c] = float(inv[s_idx, r, c])
            links[k].frame = frame_of[self.sdf_to_link_name[s_idx]]
            links[k].slot = s_idx
        return frames, links, parents

    # ------------------------------------------------------------------ state
    def set_joint_configuration(self, joint_config=None):
        """Install joint values of shape [*A, n_joints]; A (possibly empty) becomes the leading shape of results."""
        n_joints = len(self.joint_names)
        self._twists = None                   # joint twists of the installed configurations (collision_cost)
        if joint_config is None:
            joint_config = torch.zeros(n_joints, device=self.device, dtype=self.dtype)
        batched = joint_config.dim() > 1
        self.configuration_batch = tuple(joint_config.shape[:-1]) if batched else None
        if self.configuration_batch is not None:
            self.configuration_batch = torch.Size(self.configuration_batch)
        flat_q = joint_config.reshape(-1, n_joints) if batched else joint_config
        self.q = flat_q
        if self.native_fk and self._fk_plan is not None:
            # one kernel: FK along the chain or tree + (FK @ visual_offset)^-1 per mesh link, written link-major
            from . import _native as nat
            import ctypes
            frames, links, parents = self._fk_plan
            dev = nat.compute_device(self.device)
            with torch.cuda.device(dev):
                qd = flat_q.detach().reshape(-1, n_joints).to(device=dev, dtype=torch.float32).contiguous()
                n_cfg = qd.shape[0]
                out = torch.empty(len(links) * n_cfg, 4, 4, dtype=torch.float32, device=dev)
                tail = (ctypes.cast(links, ctypes.c_void_p), len(links), nat.ptr(qd), n_cfg, n_joints, nat.ptr(out),
                        nat.stream_ptr(dev))
                if parents is None:
                    nat.check(nat.lib().pvb_fk_serial(ctypes.cast(frames, ctypes.c_void_p), len(frames), *tail),
                              "pvb_fk_serial")
                else:
                    nat.check(nat.lib().pvb_fk_tree(ctypes.cast(frames, ctypes.c_void_p),
                                                    ctypes.cast(parents, ctypes.c_void_p), len(frames), *tail),
                              "pvb_fk_tree")
            self.object_to_link_frames = Transform3d(matrix=out)
            if self.sdf is not None:
                self.sdf.set_transforms(self.object_to_link_frames, batch_dim=self.configuration_batch)
            return
        poses = self.chain.forward_kinematics(flat_q, end_only=False)
        world_from_link = torch.stack([matrix_of(poses[name]) for name in self.sdf_to_link_name])   # (S, |A|, 4, 4)
        n_links, n_cfg = world_from_link.shape[:2]
        mesh_from_link = self._mesh_from_link.to(world_from_link)                                   # (S, 4, 4)
        # base frame -> mesh frame of each link: (FK @ visual_offset)^-1, link-major like the reference's stack
        mesh_from_world = mesh_from_link[:, None] @ invert_rigid(world_from_link)
        self.object_to_link_frames = Transform3d(matrix=mesh_from_world.reshape(n_links * n_cfg, 4, 4))
        if self.sdf is not None:
            self.sdf.set_transforms(self.object_to_link_frames, batch_dim=self.configuration_batch)

    # ---------------------------------------------------------------- queries
    def __call__(self, points_in_object_frame):
        """points [*B, N, 3] in the robot frame -> (values [*A, *B, N], gradients [*A, *B, N, 3])."""
        return self.sdf(points_in_object_frame)

    def paired(self, points_in_object_frame):
        """Every installed joint configuration at its own points: points [*A, *B, N, 3] in the robot frame ->
        (values [*A, *B, N], gradients [*A, *B, N, 3]), entry [a, ...] = configuration a at points[a, ...]
        (ComposedSDF.paired)."""
        return self.sdf.paired(points_in_object_frame)

    def swept(self, points_in_object_frame, return_argmin=False):
        """The minimum over every installed joint configuration at every point (the SDF of the swept volume):
        points [*B, N, 3] in the robot frame -> (values [*B, N], gradients [*B, N, 3]) and, with return_argmin, the
        first configuration attaining it (flat index into A) and its link, a position in `sdf_to_link_name`
        (ComposedSDF.swept)."""
        return self.sdf.swept(points_in_object_frame, return_argmin=return_argmin)

    def clearance(self, points_in_object_frame, return_argmin=False):
        """For every installed joint configuration, the minimum over the points of every segment (the robot's
        clearance to a cloud): points [*B, N, 3] in the robot frame -> (values [*A, *B], gradients [*A, *B, 3]) and,
        with return_argmin, the first point attaining it (index into N) and its link, a position in
        `sdf_to_link_name` (ComposedSDF.clearance)."""
        return self.sdf.clearance(points_in_object_frame, return_argmin=return_argmin)

    def paired_clearance(self, points_in_object_frame, return_argmin=False):
        """Every installed joint configuration against its own cloud: points [*A, *B, N, 3] in the robot frame ->
        (values [*A, *B], gradients [*A, *B, 3]) and, with return_argmin, the first point attaining the minimum (index
        into N) and its link, a position in `sdf_to_link_name` (ComposedSDF.paired_clearance)."""
        return self.sdf.paired_clearance(points_in_object_frame, return_argmin=return_argmin)

    def link_surface_points(self, num_points=256, seed=0):
        """[S, num_points, 3] points on the surface of every link, each in its link's own (mesh or primitive) frame,
        in the robot's dtype and on its device; cached per (num_points, seed).  Mesh links: sample_mesh_points on the
        link's mesh (kept in memory, never written to a cache file); box, cylinder and sphere links: seeded
        area-uniform samples of the analytic surface."""
        hit = self._surface_points.get((num_points, seed))
        if hit is None:
            per_link = []
            for s, (link_sdf, factory) in enumerate(zip(self.sdf.sdfs, self._link_factories)):
                if factory is not None:
                    pts = sdf.sample_mesh_points(factory, num_points, seed=seed, name=factory.name, device=self.device,
                                                 cache={})[0]
                else:
                    pts = torch.from_numpy(_primitive_surface(link_sdf, num_points, np.random.default_rng([seed, s])))
                per_link.append(pts.to(device=self.device, dtype=self.dtype))
            hit = self._surface_points[(num_points, seed)] = torch.stack(per_link)
        return hit

    def _link_paths(self):
        """(parents, paths): the parent of every frame of `frame_names` (-1 for the root), and for every link of
        `sdf_to_link_name` the frames from its own (a link's first frame) up to the root.  The parents are
        Chain.frame_parents(), or for any other chain the frame before (its frame order read as a serial chain)."""
        parents = getattr(self.chain, "frame_parents", None)
        parents = parents() if parents is not None else list(range(-1, len(self.frame_names) - 1))
        pos = {}
        for k, fname in enumerate(self.frame_names):
            pos.setdefault(self.chain.find_frame(fname).link.name, k)
        paths = []
        for name in self.sdf_to_link_name:
            f, path = pos[name], []
            while f >= 0:
                path.append(f)
                f = parents[f]
            paths.append(path)
        return parents, paths

    def self_collision_pairs(self):
        """The default `allowed` matrix of self_clearance, [S, S] bool: the pair (i, j) is tested when at least two
        movable joints lie on the tree path between the two links' frames, m(i) + m(j) - 2 m(lca(i, j)) >= 2, with m(f)
        the number of movable joints from the root up to frame f and lca the deepest frame both descend from.  That
        leaves out links on the same rigid body (one frame, or frames joined by fixed joints) and links one joint apart,
        which touch by design.  On a serial chain the lca is the shallower frame: |m(i) - m(j)| >= 2.  The structure is
        Chain.frame_parents(); any other chain is read as serial in frame order.  Other rules pass `allowed`
        explicitly."""
        parents, paths = self._link_paths()
        m = []
        for k, fname in enumerate(self.frame_names):
            movable = self.chain.find_frame(fname).joint.joint_type != "fixed"
            m.append((m[parents[k]] if parents[k] >= 0 else 0) + (1 if movable else 0))
        above = [set(p) for p in paths]
        S = len(paths)
        out = torch.zeros(S, S, dtype=torch.bool)
        for i in range(S):
            for j in range(S):
                lca = next(f for f in paths[j] if f in above[i])
                out[i, j] = m[paths[i][0]] + m[paths[j][0]] - 2 * m[lca] >= 2
        return out

    def self_clearance(self, link_points=None, allowed=None, return_argmin=False):
        """For every installed joint configuration, the smallest distance between the robot's own links: link_points
        [S, K, 3] (default: link_surface_points()) are posed with their links and tested against the links `allowed`
        [S, S] lets them (default: self_collision_pairs()).  Returns (values [*A], robot-frame gradients [*A, 3]) and,
        with return_argmin, the source link, point and target link, int64 [*A]; a negative value is a
        self-collision.  See ComposedSDF.self_clearance."""
        if link_points is None:
            link_points = self.link_surface_points()
        if allowed is None:
            allowed = self.self_collision_pairs()
        return self.sdf.self_clearance(link_points, allowed, return_argmin=return_argmin)

    def joint_twists(self):
        """[|A|, J, 6] fp64, J in `joint_names` order: (v_j, w_j) of every movable joint under the installed
        configurations, the robot-frame twist about the origin that a unit rate of q_j gives everything it moves.
        Revolute and continuous joints: w_j = R_f axis_j and v_j = -w_j x t_f, with (R_f, t_f) the pose of joint j's
        frame after its motion; prismatic joints: v_j = R_f axis_j, w_j = 0.  From the chain's forward_kinematics,
        computed on first use and kept until the configuration changes."""
        if self._twists is None:
            q = self.q.reshape(-1, len(self.joint_names))
            poses = self.chain.forward_kinematics(q, end_only=False)
            rows, names = [], []
            for fname in self.frame_names:
                frame = self.chain.find_frame(fname)
                jt = frame.joint.joint_type
                if jt == "fixed":
                    continue
                names.append(frame.joint.name)
                pose = matrix_of(poses[frame.link.name]).to(torch.float64)
                axis = torch.as_tensor(frame.joint.axis, dtype=torch.float64, device=pose.device)
                d = pose[:, :3, :3] @ (axis / axis.norm())
                if jt == "prismatic":
                    rows.append(torch.cat([d, torch.zeros_like(d)], dim=-1))
                else:
                    rows.append(torch.cat([-torch.linalg.cross(d, pose[:, :3, 3], dim=-1), d], dim=-1))
            assert names == list(self.joint_names), "joint twists must follow joint_names"
            self._twists = torch.stack(rows, dim=1) if rows else torch.zeros(q.shape[0], 0, 6, dtype=torch.float64)
        return self._twists

    def joint_moves_link(self):
        """[J, S] bool: joint j moves link s when j's frame is s's frame or one of its ancestors.  The structure is
        Chain.frame_parents(); any other chain is read as serial in frame order, where the ancestors of a frame are
        the frames before it (get_frame_names(exclude_fixed=False))."""
        _, paths = self._link_paths()
        joints = [k for k, fname in enumerate(self.frame_names)
                  if self.chain.find_frame(fname).joint.joint_type != "fixed"]
        above = [set(p) for p in paths]
        return torch.tensor([[j in up for up in above] for j in joints], dtype=torch.bool).reshape(len(joints),
                                                                                                   len(above))

    def collision_cost(self, points_in_object_frame, margin):
        """For every installed joint configuration and every segment of points [*B, N, 3] in the robot frame, the soft
        collision cost sum_p max(0, margin - d)^2 over the points within `margin` of the robot, and its derivative
        with respect to the joint values: returns (cost [*A, *B], joint_grad [*A, *B, J]) in the points' dtype and on
        their device, J in `joint_names` order.  dC/dq_j = sum over the links s that joint j moves of
        twist_grad[s] . (v_j, w_j): ComposedSDF.collision_cost's twist gradient through `joint_twists`, with the link
        gradients the query reports (for cached links, their gradient tables).  Not autograd: the gradient is an
        output of the query."""
        cost, twist = self.sdf.collision_cost(points_in_object_frame, margin)
        grad = self.joint_gradient(twist, self.joint_twists(), self.joint_moves_link())
        return cost, grad.to(cost.dtype)

    def paired_collision_cost(self, points_in_object_frame, margin):
        """Every installed joint configuration against its own cloud: points [*A, *B, N, 3] in the robot frame ->
        (cost [*A, *B], joint_grad [*A, *B, J]) in the points' dtype and on their device, J in `joint_names` order.
        Entry [a, b] is collision_cost of configuration a alone over points[a, b]: ComposedSDF.paired_collision_cost's
        twist gradient through joint_gradient(twist, joint_twists(), joint_moves_link()).  Not autograd: the gradient
        is an output of the query."""
        cost, twist = self.sdf.paired_collision_cost(points_in_object_frame, margin)
        grad = self.joint_gradient(twist, self.joint_twists(), self.joint_moves_link())
        return cost, grad.to(cost.dtype)

    def self_collision_cost(self, margin, link_points=None, allowed=None):
        """For every installed joint configuration, the soft self-collision cost between the robot's own links and its
        derivative with respect to the joint values: link_points [S, K, 3] (default: link_surface_points()) are posed
        with their links and tested against the links `allowed` [S, S] lets them (default: self_collision_pairs()),
        and every point within `margin` adds max(0, margin - d)^2.  Returns (cost [*A], joint_grad [*A, J]), J in
        `joint_names` order: ComposedSDF.self_collision_cost's twist gradient through joint_gradient(twist,
        joint_twists(), joint_moves_link()).  Not autograd: the gradient is an output of the query."""
        if link_points is None:
            link_points = self.link_surface_points()
        if allowed is None:
            allowed = self.self_collision_pairs()
        cost, twist = self.sdf.self_collision_cost(link_points, allowed, margin)
        grad = self.joint_gradient(twist, self.joint_twists(), self.joint_moves_link())
        return cost, grad.to(cost.dtype)

    def scene_clearance(self, scene, link_points=None, links=None, return_argmin=False):
        """For every installed joint configuration, the smallest distance from the robot's tested links to a static
        scene SDF in the robot frame (a CachedSDF of a scene mesh, primitives, or a ComposedSDF of them; place one
        with ComposedSDF([scene], T)): link_points [S, K, 3] (default: link_surface_points()) are posed with their
        links, and links [S] bool leaves out links not tested (a base resting on the table, say; default: all).
        Returns (values [*A], robot-frame scene gradients [*A, 3]) and, with return_argmin, the link (a position in
        `sdf_to_link_name`) and point, int64 [*A]; a negative value is a penetration.  See
        ComposedSDF.scene_clearance."""
        if link_points is None:
            link_points = self.link_surface_points()
        return self.sdf.scene_clearance(scene, link_points, links, return_argmin=return_argmin)

    def scene_collision_cost(self, scene, margin, link_points=None, links=None):
        """For every installed joint configuration, the soft collision cost of the robot's tested links against a
        static scene SDF and its derivative with respect to the joint values: link_points and links as in
        scene_clearance, and every posed point within `margin` of the scene adds max(0, margin - d)^2.  Returns
        (cost [*A], joint_grad [*A, J]), J in `joint_names` order: ComposedSDF.scene_collision_cost's twist gradient
        through joint_gradient(twist, joint_twists(), joint_moves_link()).  Not autograd: the gradient is an output of
        the query."""
        if link_points is None:
            link_points = self.link_surface_points()
        cost, twist = self.sdf.scene_collision_cost(scene, link_points, margin, links)
        grad = self.joint_gradient(twist, self.joint_twists(), self.joint_moves_link())
        return cost, grad.to(cost.dtype)

    @staticmethod
    def joint_gradient(twist, joint_twists, moves):
        """The Jacobian transpose of the robot's structure, which the [J, S] move mask encodes (joint_moves_link: joint
        j moves link s when j lies on s's path from the root): twist gradients [A, *B, S, 6] (configuration-major, A
        flat or not) and joint twists [A, J, 6] give [A, *B, J] in fp64, dC/dq_j = sum_s moves[j, s]
        twist[..., s, :] . joint_twists[a, j, :]."""
        jt = joint_twists.to(device=twist.device, dtype=torch.float64)
        tw = twist.to(torch.float64)
        lead = tw.shape[:-2]
        tw = tw.reshape(jt.shape[0], math.prod(lead) // jt.shape[0], *tw.shape[-2:])
        grad = torch.einsum("absk,js,ajk->abj", tw, moves.to(device=tw.device, dtype=torch.float64), jt)
        return grad.reshape(*lead, jt.shape[1])

    def surface_bounding_box(self, **kwargs):
        return self.sdf.surface_bounding_box(**kwargs)

    def link_bounding_boxes(self):
        """Corner points (8 x 3, robot frame) of every link's box under the installed configuration(s)."""
        world_from_mesh = Transform3d(matrix=sdf._affine_inverse(matrix_of(self.sdf.obj_frame_to_link_frame)))
        per_link = []
        for i, link_sdf in enumerate(self.sdf.sdfs):
            corners = aabb_to_ordered_end_points(np.asarray(link_sdf.surface_bounding_box(padding=0)))
            corners = torch.tensor(corners, device=world_from_mesh.device, dtype=world_from_mesh.dtype)
            per_link.append(world_from_mesh.transform_points(corners)[self.sdf.ith_transform_slice(i)])
        return torch.stack(per_link).squeeze()


class _CachedLinkFactory:
    """Picklable callable behind `cache_link_sdf_factory`."""

    def __init__(self, resolution, padding, kwargs):
        self.resolution, self.padding, self.kwargs = resolution, padding, kwargs

    def __call__(self, obj_factory: sdf.ObjectFactory):
        box = obj_factory.bounding_box(padding=self.padding)
        return sdf.CachedSDF(obj_factory.name, self.resolution, box, sdf.MeshSDF(obj_factory), **self.kwargs)


def cache_link_sdf_factory(resolution=0.01, padding=0.1, **kwargs):
    """`link_sdf_cls` that wraps every link mesh in a CachedSDF over its padded bounding box."""
    return _CachedLinkFactory(resolution, padding, kwargs)


def aabb_to_ordered_end_points(aabb, arrange_in_sequential_order=False):
    """8 corners of a (3,2) box, or (sequential order) a 16-point closed walk over its edges for line drawing."""
    lo, hi = aabb[:, 0], aabb[:, 1]
    if arrange_in_sequential_order:
        code = ["000", "100", "110", "010", "000", "001", "101", "100", "101", "111", "110", "111", "011", "010",
                "011", "001"]
    else:
        code = ["000", "100", "010", "001", "011", "101", "110", "111"]
    arr = [[(hi if c[k] == "1" else lo)[k] for k in range(3)] for c in code]
    if torch.is_tensor(aabb):
        return torch.tensor(arr, device=aabb.device, dtype=aabb.dtype)
    return np.array(arr)
