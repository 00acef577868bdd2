"""Training examples of labelled RGB-D frames (morefusion/datasets/rgbd_pose_estimation/base.py):
``RGBDPoseEstimationDatasetBase.get_example`` on the device, and a synthetic dataset over
``synthetic.make_pose_frame``.  ``visibility`` is built on request (``with_visibility``).

Per-class model data from CAD meshes (morefusion/datasets/ycb_video/models.py): ``MeshModels``,
the solid voxel grid, the SDF points and their signed distances built on the device from the
meshes a caller gives or ``MeshModels.from_directory`` reads in the YCB layout (DESIGN.md section
4.22).  Reading the YCB-Video / synthetic dataset frames and the image and mask augmentation are
not part of this package (DESIGN.md section 7)."""

from .mesh_models import MeshModels, read_obj  # noqa: F401
from .rgbd_pose_estimation import (  # noqa: F401
    MAX_INSTANCES, RGBDPoseEstimationDatasetBase, SyntheticRGBDPoseEstimationDataset, full_grids)
