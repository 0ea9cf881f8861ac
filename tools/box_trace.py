import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from igneous_b200 import zmesh
from oracle import oracle as O
data = np.zeros((64, 64, 64), dtype=np.uint32, order="F")
data[1:-1, 1:-1, 1:-1] = 1
m = zmesh.Mesher((1, 1, 1)); m.mesh(data)
got = m.get(1, reduction_factor=100, max_error=40, voxel_centered=False)
print("gpu faces", len(got.faces))
tl, tv = O.marching_cubes(data)
os.environ["ORC_SIMP_TRACE"] = "1"
want, rounds = O.simplify_welded(O.WeldedMeshes(tl, tv), (1, 1, 1), 100, 40.0, False)
print("oracle faces", len(want[1][1]), "rounds", rounds)
