"""The marching-cubes table uses, in every case, exactly the cube edges whose two corners differ in
the case's bits.  The mesher's weld relies on it: it places a label's vertices on every lattice
edge with that label on one side and another label on the other, without looking at triangles."""
import numpy as np

import mcref


def test_every_case_uses_exactly_the_edges_with_differing_corner_bits():
  tri, ntri = mcref.mc_tables()
  ends = mcref.edge_corners()
  for case in range(256):
    row = tri[case]
    assert (row[3 * ntri[case]:] == -1).all() and (row[:3 * ntri[case]] >= 0).all()
    used = set(int(e) for e in row[:3 * ntri[case]])
    differ = {e for e, (a, b) in enumerate(ends) if ((case >> a) & 1) != ((case >> b) & 1)}
    assert used == differ, case


def test_edge_corner_map_is_bourkes():
  # Bourke's edge list: 0-1, 1-2, 2-3, 3-0, 4-5, 5-6, 6-7, 7-4, 0-4, 1-5, 2-6, 3-7
  want = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
  assert [tuple(sorted(e)) for e in mcref.edge_corners()] == [tuple(sorted(e)) for e in want]
