"""The serial C oracle of hole filling (oracle_fill/) against the numpy transcription
(tests/fillref.py), and the fastmorph shim's argument errors.  No GPU."""
import numpy as np
import pytest

import fillref as F
import oracle_fill as C


@pytest.mark.parametrize("name", sorted(F.kats()))
def test_oracle_equals_numpy_on_kats(name):
  X = F.kats()[name]
  for level in (1, 2, 3, 4, 12, 13, 50, 103):
    got, want = C.fill_level(X, level), F.fill_level(X, level)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), level
  for p in (40, 60):
    got, want = C.fill_holes(X, p=p), F.fill_holes(X, p=p)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), p


@pytest.mark.parametrize("shape,seed", [((40, 36, 33), 1), ((65, 33, 17), 2), ((40, 1, 30), 3), ((1, 37, 29), 4),
                                        ((64, 64, 64), 5), ((33, 40, 1), 6)])
def test_oracle_equals_numpy_on_random_volumes(shape, seed):
  X = F.random_volume(shape, seed)
  for level in (1, 2, 3, 4, 50, 103):
    got, want = C.fill_level(X, level), F.fill_level(X, level)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), level


def test_oracle_dilation_equals_numpy():
  rng = np.random.default_rng(0)
  for shape in ((5, 5, 5), (33, 17, 9), (70, 1, 13)):
    X = rng.integers(0, 5, size=shape).astype(np.uint16)
    X[rng.random(shape) < 0.5] = 0
    assert np.array_equal(C.dilate(X), F.dilate(X))


def test_fastmorph_shim_argument_errors():
  """Refused before any device work, so no GPU is needed."""
  from igneous_b200 import fastmorph
  X = np.zeros((4, 4, 4), np.uint32)
  with pytest.raises(NotImplementedError):
    fastmorph.dilate(X, mode=fastmorph.Mode.grey)
  with pytest.raises(NotImplementedError):
    fastmorph.dilate(X, background_only=False)
  with pytest.raises(NotImplementedError):
    fastmorph.fill_holes_v2(X, return_crackle=True)
  with pytest.raises(ValueError):
    fastmorph.fill_holes_v2(X, merge_threshold=0.995)
  for bad in (X.astype(np.float32), X.astype(np.int32), X.astype(np.int64)):
    with pytest.raises(NotImplementedError):
      fastmorph.fill_holes_v2(bad)
    with pytest.raises(NotImplementedError):
      fastmorph.dilate(bad)
  with pytest.raises(ValueError):
    fastmorph.fill_holes_v2(np.zeros((2, 2, 2, 2), np.uint32))
