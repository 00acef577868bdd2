"""GPU: the occupancy server's render (``MultiInstanceOctreeMapping.render``) and the instance boxes
its scan keeps (``boxes``) bitwise against oracle/octomap_server_render.py over synthetic 640x480
multi-view sequences of 8 instances, rendered after every scan (tests/test_mapping_render_emu.py
runs the same kernels serially on the CPU)."""

import numpy as np
import pytest
import torch

from oracle import octomap_server_render as osr
from test_mapping_server_emu import pcd_of, pitch_of

pytestmark = pytest.mark.gpu


class GpuPair:
    def __init__(self, capacity=1 << 22):
        from morefusion_b200.contrib import MultiInstanceOctreeMapping
        self.ours = MultiInstanceOctreeMapping(capacity=capacity)
        self.trees, self.centres, self.boxes, self.server_trees = {}, {}, {}, set()

    def scan(self, label, pcd, T, classes, max_range):
        self.ours.integrate_scan(torch.as_tensor(label, device="cuda"), pcd, T, classes,
                                 max_range=max_range, background_pitch=0.01)
        osr.insert_scan(self.trees, self.centres, self.boxes, self.server_trees, label,
                        pcd.cpu().numpy(), T,
                        classes, pitch_of=pitch_of, max_range=max_range, background_pitch=0.01)

    def check(self, pcd, T, K):
        got = self.ours.boxes()
        assert set(got) == set(self.trees) - {-1}
        for i, b in got.items():
            want = np.stack(self.boxes.get(i, osr.DEFAULT_BBX))
            assert np.array_equal(b.view(np.uint32), want.view(np.uint32)), i
        label, depth = self.ours.render(pcd, T, K)
        assert label.is_cuda and depth.is_cuda
        again = self.ours.render(pcd, T, K)
        assert torch.equal(label, again[0]) and torch.equal(depth.view(torch.int32),
                                                            again[1].view(torch.int32))
        want = osr.render(self.trees, self.boxes, pcd.cpu().numpy(), T, K)
        assert np.array_equal(label.cpu().numpy(), want[0])
        assert np.array_equal(depth.cpu().numpy().view(np.uint32), want[1].view(np.uint32))
        return want


@pytest.mark.parametrize("n_views", [1, 3, 10])
def test_render_after_every_scan_matches_oracle(cuda_device, n_views):
    from morefusion_b200 import synthetic
    f = synthetic.make_rgbd_views(n_views, n_views, n_objects=8)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    pair = GpuPair()
    n_hit = 0
    for v in f["views"]:
        pcd = torch.as_tensor(pcd_of(v, f["K"]), device="cuda")
        pair.scan(v["label"], pcd, v["sensor_to_world"], classes, synthetic.VIEWS_MAX_RANGE)
        want = pair.check(pcd, v["sensor_to_world"], f["K"])
        n_hit += int((want[0] > 0).sum())
    assert n_hit > 1000
    assert set(np.unique(want[0]).tolist()) - {-2} <= set(classes)


def test_render_while_the_table_grows(cuda_device):
    """The hash table starts small and grows mid-sequence; boxes and render stay exact."""
    from morefusion_b200 import synthetic
    f = synthetic.make_rgbd_views(11, 3, n_objects=8)
    classes = dict(zip(f["instance_ids"].tolist(), f["class_ids"].tolist()))
    pair = GpuPair(capacity=1 << 17)
    caps = []
    for v in f["views"]:
        pcd = torch.as_tensor(pcd_of(v, f["K"]), device="cuda")
        pair.scan(v["label"], pcd, v["sensor_to_world"], classes, -1.0)
        pair.ours._check()
        caps.append(pair.ours._cap)
        pair.check(pcd, v["sensor_to_world"], f["K"])
    assert caps[0] < caps[-1]
