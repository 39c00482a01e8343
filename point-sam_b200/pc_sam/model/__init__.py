from .pc_sam import PointCloudSAM, PointCloudSAMHier, PointSAM, build_point_sam, build_point_sam_hier  # noqa: F401
