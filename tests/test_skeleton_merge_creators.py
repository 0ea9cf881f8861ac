"""create_unsharded_skeleton_merge_tasks without a GPU: the prefix enumeration for magnitudes 1-3, __len__,
the provenance appended after iteration, the import surface and the skeleton info's mip.  No kernel runs."""
import numpy as np
import pytest

import igneous_b200
from igneous_b200 import task_creation as tc
from igneous_b200 import tasks
from igneous_b200._compat import CloudVolume


def _layer(tmp_path):
  path = "file://" + str(tmp_path / "seg")
  info = CloudVolume.create_new_info(1, "segmentation", np.uint64, "raw", (4, 4, 40), (0, 0, 0), (64, 64, 16),
                                     (64, 64, 16))
  CloudVolume(path, info=info).commit_info()
  return path


@pytest.mark.parametrize("magnitude,want", [
  (1, [str(p) for p in range(1, 10)]),
  (2, ["%d:" % p for p in range(1, 10)] + [str(p) for p in range(10, 100)]),
  (3, ["%d:" % p for p in range(1, 100)] + [str(p) for p in range(100, 1000)]),
])
def test_prefixes_len_and_provenance(tmp_path, magnitude, want):
  path = _layer(tmp_path)
  it = tc.create_unsharded_skeleton_merge_tasks(path, crop=2, magnitude=magnitude, dust_threshold=7,
                                                max_cable_length=50, tick_threshold=9, delete_fragments=True)
  assert len(it) == 10 ** magnitude
  assert not CloudVolume(path).provenance.processing
  got = list(it)
  assert [str(t.prefix) for t in got] == want
  t = got[0]
  assert (t.crop, t.dust_threshold, t.tick_threshold, t.max_cable_length, t.delete_fragments) == (2, 7, 9, 50.0, True)
  # every label 1..10^4 is matched by exactly one prefix
  for segid in [1, 9, 10, 99, 100, 999, 1000, 12345, 2 ** 40 + 7]:
    name = "%d:0-1_0-1_0-1" % segid
    assert sum(name.startswith(str(p)) for p in want) == 1, segid
  method = CloudVolume(path).provenance.processing[-1]["method"]
  assert method == {"task": "UnshardedSkeletonMergeTask", "cloudpath": path, "crop": 2, "dust_threshold": 7,
                    "tick_threshold": 9, "delete_fragments": True, "max_cable_length": 50}


def test_import_surface_and_defaults():
  assert igneous_b200.UnshardedSkeletonMergeTask is tasks.UnshardedSkeletonMergeTask
  assert tc.create_unsharded_skeleton_merge_tasks is not None
  t = tasks.UnshardedSkeletonMergeTask("file:///x", "1:")
  assert (t.crop, t.dust_threshold, t.max_cable_length, t.tick_threshold, t.delete_fragments) == \
      (0, 4000, None, 6000, False)
  from igneous_b200 import kimimaro
  assert callable(kimimaro.postprocess) and callable(kimimaro.merge_fragments)
  assert kimimaro.merge_fragments({}) == {}  # a prefix without fragments needs no device


def test_skeleton_meta_mip(tmp_path):
  path = _layer(tmp_path)
  vol = CloudVolume(path)
  assert vol.skeleton.meta.mip == 0
  vol.info["skeletons"] = "skeletons_mip_2"
  vol.commit_info()
  vol = CloudVolume(path)
  vol.skeleton.meta.info["mip"] = 2
  vol.skeleton.meta.commit_info()
  assert CloudVolume(path).skeleton.meta.mip == 2
