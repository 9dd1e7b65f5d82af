"""KITTI layout (src/dataset/kitti.py): velodyne/{:06d}.bin, poses_lidar.txt, rows with z <= -3 dropped."""
import nerfloam_b200


class DataLoader(nerfloam_b200.dataset.ScanLoader):
    scan_name = "{:06d}.bin"
    pose_file = "poses_lidar.txt"
    remove_abnormal_z = True
