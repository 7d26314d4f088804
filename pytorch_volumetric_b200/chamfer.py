"""Points-to-mesh chamfer distance and the pose-set metrics built on it.

Mirrors the reference's src/pytorch_volumetric/chamfer.py: batch_chamfer_dist (:62-120) runs as one fused
kernel (transform -> unsigned nearest distance / table value -> square -> mean, pvb_chamfer);
pairwise_distance_chamfer (:20-59) and PlausibleDiversity (:130-195) are thin reductions on top of it.
"""
import ctypes
from typing import NamedTuple

import torch

from . import _native as nat
from .sdf import ObjectFactory, ObjectFrameSDF, sample_mesh_points
from .transforms import matrix_of, invert_rigid


def matrix_to_rotation_6d(m):
    return m[..., :2, :].clone().reshape(*m.shape[:-2], 6)


def pairwise_distance(world_to_link_tfs):
    m = matrix_of(world_to_link_tfs)
    cont_rep = torch.cat((m[:, :3, 3], matrix_to_rotation_6d(m[:, :3, :3])), dim=1)
    return torch.cdist(cont_rep, cont_rep)


def batch_chamfer_dist(world_to_object: torch.tensor, model_points_world_frame_eval: torch.tensor,
                       obj_factory: ObjectFactory = None, obj_sdf: ObjectFrameSDF = None, viewing_delay=0, scale=1000.,
                       print_err=False, vis=None):
    """
    Batched unidirectional chamfer distance between world-frame surface points and the object under B rigid
    transforms.
    :param world_to_object: B x 4 x 4 transformation matrices from world to object frame
    :param model_points_world_frame_eval: N x 3 points to evaluate the chamfer distance on
    :param obj_factory: object (mesh) to evaluate against
    :param obj_sdf: sdf of the object to evaluate against (faster, less accurate)
    :param scale: position-unit multiplier before squaring (1000: m -> mm)
    :return: B chamfer error per transform, mean over the N points of (scale * d)^2
    """
    if vis is not None:
        raise NotImplementedError("visualisation (vis=) is outside the query path; pass vis=None")
    desc = None
    if obj_sdf is not None:
        dev = nat.compute_device(world_to_object.device)
        desc = obj_sdf.native_desc(dev)
        if desc is None:
            # arbitrary ObjectFrameSDF: evaluate through its __call__ (chamfer.py:84-85)
            m = world_to_object
            pts = model_points_world_frame_eval
            pts_obj = pts @ m[:, :3, :3].transpose(-1, -2) + m[:, :3, 3].unsqueeze(1)
            d, _ = obj_sdf(pts_obj)
            return ((scale * d) ** 2).mean(dim=-1)
    elif obj_factory is not None:
        dev = nat.compute_device(world_to_object.device)
        desc = obj_factory.native_desc(dev)
    else:
        raise ValueError("Either obj_sdf or obj_factory must be given")

    B = world_to_object.shape[0]
    out_dtype, out_device = world_to_object.dtype, world_to_object.device
    if B == 0 or model_points_world_frame_eval.shape[0] == 0:       # mean over nothing: NaN, as torch's .mean()
        return torch.full((B,), float("nan"), dtype=out_dtype, device=out_device)
    with torch.cuda.device(dev):
        W = world_to_object.detach().to(device=dev, dtype=torch.float32).contiguous()
        p = nat.as_f32_points(model_points_world_frame_eval, dev)
        n = p.shape[0]
        L = nat.lib()
        out = torch.empty(B, dtype=torch.float32, device=dev)
        nblk = int(L.pvb_chamfer_workspace(n))
        sort_ws = nat.query_workspace(n, dev) if desc.kind == nat.PVB_KIND_MESH else None
        done = 0
        while done < B:     # the kernel takes at most 65535 transforms per launch
            nb = min(B - done, 65535)
            ws = torch.empty(nb * nblk, dtype=torch.float32, device=dev)
            nat.check(L.pvb_chamfer(ctypes.byref(desc), nat.ptr(W[done:]), nb, nat.ptr(p), n, float(scale),
                                    nat.ptr(ws), nat.ptr(out[done:]), nat.ptr(sort_ws),
                                    sort_ws.numel() if sort_ws is not None else 0, nat.stream_ptr(dev)),
                      "pvb_chamfer")
            done += nb
    return nat.deliver(out, out_device, out_dtype)


def pairwise_distance_chamfer(A_link_to_world_tfs, B_world_to_link_tfs=None,
                              obj_factory: ObjectFactory = None, obj_sdf: ObjectFrameSDF = None,
                              model_points_eval: torch.tensor = None, vis=None, scale=1000):
    """Chamfer distance of every pairing of two pose sets (reference chamfer.py:20-59).

    The composites B[p] @ A[b] (identity when the two poses agree; B defaults to the inverses of A) are evaluated in
    one `batch_chamfer_dist` launch, flat in p-major order.  The reference then returns `errors.view(len(A), len(B))`
    of that flat data (chamfer.py:49-58), which this function reproduces exactly: for equally sized pose sets -- the
    only case the reference's callers use -- entry [i, j] scores B[i] @ A[j]; for unequal sizes the view re-chunks
    the p-major data just like the reference does.
    """
    link_to_world = matrix_of(A_link_to_world_tfs)
    if model_points_eval is None:
        model_points_eval, _, _ = sample_mesh_points(obj_factory, num_points=500, name=obj_factory.name,
                                                     device=link_to_world.device)
    world_to_link = invert_rigid(link_to_world) if B_world_to_link_tfs is None else matrix_of(B_world_to_link_tfs)
    errors = _pairwise_chamfer(world_to_link, link_to_world, model_points_eval, obj_factory, obj_sdf, scale, vis)
    return errors.reshape(-1).view(link_to_world.shape[0], world_to_link.shape[0])


def _pairwise_chamfer(left, right, points, obj_factory, obj_sdf, scale, vis=None):
    """errors[i, j] = chamfer(left[i] @ right[j]) as an (len(left), len(right)) matrix."""
    composite = torch.einsum("bij,pjk->bpik", left, right)
    n_left, n_right = composite.shape[:2]
    errors = batch_chamfer_dist(composite.reshape(n_left * n_right, 4, 4), points, obj_factory=obj_factory,
                                obj_sdf=obj_sdf, viewing_delay=0, vis=vis, scale=scale)
    return errors.view(n_left, n_right)


class PlausibleDiversityReturn(NamedTuple):
    plausibility: torch.tensor
    coverage: torch.tensor
    most_plausible_per_estimated: torch.tensor
    most_covered_per_plausible: torch.tensor


class PlausibleDiversity:
    """Set divergence between estimated and plausible pose sets (reference chamfer.py:130-195), in squared scaled
    units: plausibility = mean over estimates of the best match among the plausible poses, coverage = mean over
    plausible poses of the best match among the estimates."""

    def __init__(self, obj_factory: ObjectFactory, model_points_eval: torch.tensor = None, num_model_points_eval=500,
                 obj_sdf: ObjectFrameSDF = None):
        self.obj_factory = obj_factory
        self.obj_sdf = obj_sdf
        if model_points_eval is None:
            model_points_eval = sample_mesh_points(obj_factory, num_points=num_model_points_eval,
                                                   name=obj_factory.name)[0]
        self.model_points_eval = model_points_eval

    def compute_tf_pairwise_error_per_batch(self, T_est_inv, T_p, scale=1000.):
        self.model_points_eval = self.model_points_eval.to(device=T_est_inv.device, dtype=T_est_inv.dtype)
        return _pairwise_chamfer(T_est_inv, T_p, self.model_points_eval, self.obj_factory, self.obj_sdf, scale)

    @staticmethod
    def do_evaluate_plausible_diversity_on_pairwise_chamfer_dist(errors_per_batch):
        per_estimate = errors_per_batch.min(dim=1)
        per_plausible = errors_per_batch.min(dim=0)
        return PlausibleDiversityReturn(per_estimate.values.mean(), per_plausible.values.mean(),
                                        per_estimate, per_plausible)

    def __call__(self, T_est_inv, T_p, bidirectional=False, scale=1000.):
        score = self.do_evaluate_plausible_diversity_on_pairwise_chamfer_dist
        forward = score(self.compute_tf_pairwise_error_per_batch(T_est_inv, T_p, scale=scale))
        if not bidirectional:
            return forward
        # with the roles of the two sets swapped, plausibility and coverage trade places
        backward = score(self.compute_tf_pairwise_error_per_batch(T_p, T_est_inv, scale=scale))
        return PlausibleDiversityReturn(plausibility=(forward.plausibility + backward.coverage) / 2,
                                        coverage=(forward.coverage + backward.plausibility) / 2,
                                        most_plausible_per_estimated=forward.most_plausible_per_estimated,
                                        most_covered_per_plausible=forward.most_covered_per_plausible)
