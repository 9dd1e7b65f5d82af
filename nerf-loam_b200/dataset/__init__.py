"""The reference's scan loaders (src/dataset/kitti.py, maicity.py) with the ground segmentation on the GPU (ground.py) in place of
the external Patchwork++ library.  `dataset.kitti.DataLoader` and `dataset.maicity.DataLoader` keep the reference's constructor and
methods; __getitem__ returns (index, points f32[N,3], pointcos f32[N], pose 4x4 or None) with CPU tensors, the ground points first.
The keyword `ground_params` (a ground.GroundParams, e.g. with the vertical filter on) sets the segmentation; None keeps its defaults.

The reference imports them as `import_module("dataset." + name)` (src/utils/import_util.py:4-6), so the seam is one line:

    sys.modules["dataset"] = nerfloam_b200.dataset

That import creates the submodules a second time, as `dataset.kitti`; they therefore import the package absolutely.
"""
import os.path as osp
from glob import glob

import numpy as np
import torch
from torch.utils.data import Dataset

__all__ = ["ScanLoader", "kitti", "maicity"]


class ScanLoader(Dataset):
    """A directory of velodyne/*.bin scans (float32 rows x, y, z, intensity) and an optional pose file of 3x4 rows."""
    scan_name = None            # format of a scan's file name under velodyne/
    pose_file = None
    remove_abnormal_z = False   # drop rows with z <= -3.0 before the depth gates

    def __init__(self, data_path, use_gt=False, max_depth=-1, min_depth=-1, ground_params=None):
        self.data_path = data_path
        self.ground_params = ground_params
        self.num_bin = len(glob(osp.join(self.data_path, "velodyne/*.bin")))
        self.use_gt = use_gt
        self.max_depth = max_depth
        self.min_depth = min_depth
        self.gt_pose = self.load_gt_pose() if use_gt else None

    def get_init_pose(self, frame):
        if self.gt_pose is not None:
            return np.concatenate((self.gt_pose[frame], [0, 0, 0, 1])).reshape(4, 4)
        return np.eye(4)

    def load_gt_pose(self):
        """The pose file's rows (3x4 row-major, one per scan) as f64[S,12]."""
        return np.loadtxt(osp.join(self.data_path, self.pose_file)).reshape(-1, 12)

    def read_points(self, index):
        """Scan `index` after the reference's filters (z > -3 where it applies, then the depth gates on |p|): float32 [M,4]."""
        path = osp.join(self.data_path, "velodyne", self.scan_name.format(index))
        points = np.fromfile(path, dtype=np.float32, count=-1).reshape([-1, 4])
        if self.remove_abnormal_z:
            points = points[points[:, 2] > -3.0]
        points_norm = np.linalg.norm(points[:, :3], axis=-1)
        point_mask = True
        if self.max_depth != -1:
            point_mask = (points_norm < self.max_depth) & point_mask
        if self.min_depth != -1:
            point_mask = (points_norm > self.min_depth) & point_mask
        if isinstance(point_mask, np.ndarray):
            points = points[point_mask]
        return points

    def load_points(self, index):
        """(points f32[N,3], pointcos f32[N]) as numpy: the ground points first, then the rest, each half in scan order."""
        import nerfloam_b200
        points, pointcos, _ = nerfloam_b200.ground.points_and_cos(self.read_points(index), self.ground_params)
        return points.cpu().numpy(), pointcos.cpu().numpy()

    def __len__(self):
        return self.num_bin

    def __getitem__(self, index):
        points, pointcos = self.load_points(index)
        pose = np.concatenate((self.gt_pose[index], [0, 0, 0, 1])).reshape(4, 4) if self.use_gt else None
        return index, torch.from_numpy(points).float(), torch.from_numpy(pointcos).float(), pose


def __getattr__(name):
    if name in ("kitti", "maicity"):
        import importlib
        return importlib.import_module("." + name, __name__)
    raise AttributeError(name)
