"""Host-side container of one LiDAR scan with the attribute and method names the reference's loops touch
(src/lidarFrame.py:10-57: index, num_point, points, pointsCos, pose, rays_d, rays_norm, rel_pose, sample_mask; get_* / set_rel_pose /
sample_rays) plus the per-iteration ray selection of src/utils/sample_util.py:4-19.  The selection stays on the CPU torch
generator on purpose: the same seed then picks the same rays as the reference (the fused loops also offer a device-side draw,
render_helpers._FrameBatch.select)."""
import torch
import torch.nn as nn

from .se3pose import OptimizablePose

POSE_OFFSET = 2000   # metres added to the translation of externally supplied poses (lidarFrame.py:18)
_TINY = 1e-9


def sample_rays(mask, num_samples, generator=None):
    """Boolean mask [B,H,W] with exactly `num_samples` True cells per batch entry, drawn without replacement with probability
    proportional to `mask` (Gumbel top-k, sample_util.py:4-19; the constants 1e-9 / 1e-7 are the reference's).  generator: a
    torch.Generator on the mask's device to draw from instead of torch's (None: the reference's draw, torch.rand_like)."""
    batch, height, width = mask.shape
    weights = (mask / (mask.sum() + _TINY)).reshape(batch, height * width)
    uniform = torch.rand(weights.shape, dtype=weights.dtype, device=weights.device, generator=generator)
    keys = torch.log(weights + _TINY) - torch.log(1e-7 - torch.log(uniform + 1e-7))
    chosen = keys.topk(num_samples, dim=-1).indices
    picked = torch.zeros_like(weights)
    picked.scatter_(-1, chosen, 1)
    return picked.reshape(batch, height, width) > 0


def _unit_directions(points):
    """(unit ray directions [N,1,3] fp32, ranges [N,1]); the 1e-8 guards the origin return (lidarFrame.py:48-52)."""
    ranges = points.norm(p=2, dim=-1, keepdim=True) + 1e-8
    return (points / ranges).unsqueeze(1).float(), ranges


class LidarFrame(nn.Module):
    """index: scan number; points: f32[N,3] in the sensor frame; pointsCos: f32[N] incidence cosines.  `pose` is either a 4x4
    matrix (numpy / tensor; gets POSE_OFFSET and becomes an OptimizablePose parameter) or, with new_keyframe=True, an
    OptimizablePose that is adopted as is."""

    def __init__(self, index, points, pointsCos, pose=None, new_keyframe=False):
        super().__init__()
        self.index, self.points, self.pointsCos = index, points, pointsCos
        self.num_point = len(points)
        if new_keyframe:
            self.pose = pose
        elif pose is not None:
            pose[:3, 3] += POSE_OFFSET        # in place, like the reference: the caller's matrix is shifted too
            self.pose = OptimizablePose.from_matrix(torch.tensor(pose, requires_grad=True, dtype=torch.float32))
        self.rel_pose = None
        self.sample_mask = None
        self.rays_d = self.get_rays()

    # --- pose views ------------------------------------------------------------------------------------------------
    def get_pose(self):
        return self.pose.matrix()

    def get_rotation(self):
        return self.pose.rotation()

    def get_translation(self):
        return self.pose.translation()

    def get_rel_pose(self):
        return self.rel_pose

    def set_rel_pose(self, rel_pose):
        self.rel_pose = rel_pose

    # --- scan data -------------------------------------------------------------------------------------------------
    def get_points(self):
        return self.points

    def get_pointsCos(self):
        return self.pointsCos

    @torch.no_grad()
    def get_rays(self):
        directions, self.rays_norm = _unit_directions(self.points)
        return directions

    @torch.no_grad()
    def sample_rays(self, N_rays, track=False, generator=None):
        """Draws this iteration's rays: sample_mask bool[N,1] with N_rays True (every point equally likely), from `generator` (a CPU
        torch.Generator) when one is given."""
        every_point = torch.ones((1, self.num_point, 1))
        self.sample_mask = sample_rays(every_point, N_rays, generator)[0]
