"""MaiCity layout (src/dataset/maicity.py): velodyne/{:05d}.bin, poses.txt, no z filter."""
import nerfloam_b200


class DataLoader(nerfloam_b200.dataset.ScanLoader):
    scan_name = "{:05d}.bin"
    pose_file = "poses.txt"
