"""Training examples of labelled RGB-D frames (morefusion/datasets/rgbd_pose_estimation/base.py):
``RGBDPoseEstimationDatasetBase.get_example`` on the device, and a synthetic dataset over
``synthetic.make_pose_frame``.  ``visibility`` is built on request (``with_visibility``).  Reading
the YCB-Video / synthetic dataset files and the image and mask augmentation are not part of this
package (DESIGN.md section 7)."""

from .rgbd_pose_estimation import (  # noqa: F401
    MAX_INSTANCES, RGBDPoseEstimationDatasetBase, SyntheticRGBDPoseEstimationDataset, full_grids)
