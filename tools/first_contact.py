#!/usr/bin/env python3
"""First-contact probes (SURVEY.md 8(c), "run once against the real wheels, then freeze the
enum defaults").  The reference's arithmetic lives in tinybrain / cc3d / zmesh / fastremap,
which are absent from the build image; the oracle restates their documented behaviour and
marks the rules it had to recall as "parity unpinned".  Run this script in ANY environment
where those wheels import:

    python tools/first_contact.py [--out tests/golden]

For every probe it prints which of the oracle's candidate rules the wheel follows, writes the
wheel's outputs to tests/golden/upstream_*.npz (tests/test_golden.py picks them up and holds
both the oracle and the GPU path to them), and exits non-zero if a frozen default of the
product (igneous_b200.tinybrain.DEFAULT_ROUNDING, the corner convention of the mode rule, the
marching-cubes winding, cc3d's numbering order) disagrees with the wheel.  Without the wheels it
reports which probes could not run and exits 0.
"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def try_import(name):
  try:
    return importlib.import_module(name)
  except Exception as e:  # noqa: BLE001 - any import failure means "wheel absent"
    return None


def probe_averaging(tb, O, out, report):
  """2x2 blocks (0,1,1,1) 0.75, (0,0,1,1) 0.5, (1,1,2,2) 1.5 and a ramp through 5 mips."""
  blocks = np.array([[0, 1, 1, 1], [0, 0, 1, 1], [1, 1, 2, 2], [254, 255, 255, 255]], dtype=np.uint8)
  img = np.zeros((2, 2 * len(blocks), 1), dtype=np.uint8, order="F")
  for i, b in enumerate(blocks):
    img[:, 2 * i:2 * i + 2, 0] = b.reshape(2, 2)
  got = np.asarray(tb.downsample_with_averaging(img, (2, 2, 1), num_mips=1)[0]).ravel()
  cands = {"floor": [0, 0, 1, 254], "half_up": [1, 1, 2, 255], "half_even": [1, 0, 2, 255]}
  rule = [k for k, v in cands.items() if list(got) == v]
  ramp = (np.add.outer(np.arange(64), np.arange(64)) % 251).astype(np.uint8)[:, :, None]
  ramp = np.asfortranarray(ramp)
  up = [np.asarray(m) for m in tb.downsample_with_averaging(ramp, (2, 2, 1), num_mips=5)]
  np.savez_compressed(os.path.join(out, "upstream_avg_pool.npz"), blocks=img, blocks_out=got, ramp=ramp,
                      **{"ramp_mip%d" % (i + 1): m for i, m in enumerate(up)})
  mode = None
  for name, r in (("floor", 0), ("half_up", 1), ("half_even", 2)):
    mine = O.downsample_with_averaging(ramp, (2, 2, 1), num_mips=5, rounding=r)
    if all(np.array_equal(a, b) for a, b in zip(mine, up)):
      mode = name
  report["averaging"] = {"block_rule": rule, "five_mip_ramp_matches_oracle_rounding": mode}
  from igneous_b200 import tinybrain as mine_tb, _shim
  names = {_shim.ROUND_FLOOR: "floor", _shim.ROUND_HALF_UP: "half_up", _shim.ROUND_HALF_EVEN: "half_even"}
  return mode is not None and names[mine_tb.DEFAULT_ROUNDING] == mode


def probe_mode(tb, O, out, report):
  kats = {(1, 1, 2, 3): 1, (1, 2, 1, 3): 1, (1, 2, 2, 3): 2, (1, 2, 3, 3): 3, (1, 2, 3, 4): 4, (1, 1, 2, 2): 1,
          (1, 2, 2, 1): 2, (0, 0, 5, 5): 0}
  ok = True
  res = {}
  for (a, b, c, d), want in kats.items():
    img = np.asfortranarray(np.array([[a, c], [b, d]], dtype=np.uint32)[:, :, None])  # img[x, y]
    got = int(np.asarray(tb.downsample_segmentation(img, (2, 2, 1), num_mips=1)[0]).ravel()[0])
    res[str((a, b, c, d))] = got
    ok = ok and got == want
  rng = np.random.default_rng(0)
  odd = np.asfortranarray(rng.integers(0, 4, size=(7, 5, 3)).astype(np.uint32))
  up_odd = [np.asarray(m) for m in tb.downsample_segmentation(odd, (2, 2, 1), num_mips=2)]
  up_sparse = [np.asarray(m) for m in tb.downsample_segmentation(odd, (2, 2, 1), num_mips=2, sparse=True)]
  np.savez_compressed(os.path.join(out, "upstream_mode_pool.npz"), odd=odd,
                      **{"odd_mip%d" % (i + 1): m for i, m in enumerate(up_odd)},
                      **{"sparse_mip%d" % (i + 1): m for i, m in enumerate(up_sparse)})
  mine = O.downsample_segmentation(odd, (2, 2, 1), num_mips=2)
  mine_s = O.downsample_segmentation(odd, (2, 2, 1), num_mips=2, sparse=True)
  odd_ok = all(np.array_equal(a, b) for a, b in zip(mine, up_odd))
  sparse_ok = all(np.array_equal(a, b) for a, b in zip(mine_s, up_sparse))
  report["mode"] = {"tie_break_kats": res, "kats_match": ok, "odd_extent_matches_oracle": odd_ok,
                    "sparse_matches_oracle": sparse_ok}
  return ok and odd_ok and sparse_ok


def probe_cc3d(cc3d, fastremap, O, out, report):
  rng = np.random.default_rng(1)
  vol = rng.integers(0, 3, size=(9, 8, 7)).astype(np.uint32)
  f = np.asfortranarray(vol)
  c = np.ascontiguousarray(vol)
  lf = np.asarray(cc3d.connected_components(f, connectivity=6, out_dtype=np.uint64))
  lc = np.asarray(cc3d.connected_components(c, connectivity=6, out_dtype=np.uint64))
  mine = O.connected_components(f)
  report["cc3d"] = {"f_order_numbering_equals_oracle": bool(np.array_equal(lf, mine)),
                    "c_order_numbering_equals_f_order": bool(np.array_equal(lf, lc)),
                    "equal_after_renumber": bool(np.array_equal(fastremap.renumber(lf.copy())[0],
                                                                fastremap.renumber(mine.copy())[0]))}
  np.savez_compressed(os.path.join(out, "upstream_cc3d.npz"), vol=f, labels_f=lf, labels_c=lc)
  return report["cc3d"]["equal_after_renumber"]


def probe_zmesh(zmesh, O, out, report):
  data = np.zeros((64, 64, 64), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 1  # the reference's own mesh test volume (test/test_tasks.py:413-415)
  m = zmesh.Mesher((1, 1, 1))
  m.mesh(data)
  raw = m.get(1, reduction_factor=0, voxel_centered=False)
  v, f = np.asarray(raw.vertices, np.float64), np.asarray(raw.faces)
  vol6 = np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum()
  vc = m.get(1, reduction_factor=0, voxel_centered=True)
  simp = m.get(1, reduction_factor=100, max_error=40, voxel_centered=True)
  tl, tv = O.marching_cubes(data)
  cv1, cf1 = O.canonicalise_mesh(raw.vertices, raw.faces)
  wv, wf = O.mesh_for_label(tl, tv, 1, resolution=(1, 1, 1), voxel_centered=False)
  cv2, cf2 = O.canonicalise_mesh(wv, wf)
  report["zmesh"] = {"faces": int(len(f)), "vertices": int(len(v)), "outward_winding": bool(vol6 > 0),
                     "voxel_centered_shift": [float(x) for x in (np.asarray(vc.vertices).min(0) - v.min(0))],
                     "canonical_mesh_equals_oracle": bool(np.array_equal(cv1, cv2) and np.array_equal(cf1, cf2)),
                     "faces_after_x100": int(len(simp.faces)), "vertices_after_x100": int(len(simp.vertices))}
  np.savez_compressed(os.path.join(out, "upstream_zmesh_box.npz"), vertices=raw.vertices, faces=raw.faces,
                      simp_vertices=simp.vertices, simp_faces=simp.faces)
  return report["zmesh"]["canonical_mesh_equals_oracle"] and report["zmesh"]["outward_winding"]


def probe_cseg(cseg, O, out, report):
  """compressed_segmentation wheel: is the oracle's (and therefore the device codec's) byte stream the
  one the wheel writes, and does each side decode the other's stream?"""
  rng = np.random.default_rng(3)
  vols = {"u32": np.asfortranarray(rng.integers(0, 6, size=(40, 33, 17)).astype(np.uint32)),
          "u64": np.asfortranarray((rng.integers(0, 9, size=(16, 16, 16)).astype(np.uint64) << np.uint64(33)))}
  res = {}
  ok = True
  for name, v in vols.items():
    theirs = bytes(cseg.compress(v, block_size=(8, 8, 8), order="F"))
    mine = O.cseg_encode(v[..., np.newaxis], (8, 8, 8)).tobytes()
    back = np.asarray(cseg.decompress(mine, v.shape, dtype=v.dtype, block_size=(8, 8, 8), order="F")).reshape(v.shape)
    mine_back = O.cseg_decode(np.frombuffer(theirs, dtype=np.uint32), v.shape + (1,), v.dtype, (8, 8, 8))[..., 0]
    res[name] = {"bytes_identical": theirs == mine, "wheel_decodes_ours": bool(np.array_equal(back, v)),
                 "we_decode_wheel": bool(np.array_equal(mine_back, v))}
    ok = ok and res[name]["wheel_decodes_ours"] and res[name]["we_decode_wheel"]
    np.savez_compressed(os.path.join(out, "upstream_cseg_%s.npz" % name), vol=v, stream=np.frombuffer(theirs, dtype=np.uint8))
  report["compressed_segmentation"] = res
  return ok


def probe_fastmorph(fm, out, report):
  """fastmorph.dilate / fill_holes_v2 on the hole-filling test volumes (tests/fillref.py): records
  the wheel's outputs and whether they follow the rule of DESIGN.md "Hole filling".  That rule
  is this project's own until the recorded outputs pin it, so a difference is reported, not failed."""
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  import fillref as F
  res, arrays = {}, {}
  for name, X in sorted(F.kats().items()):
    for level in (1, 2, 3, 4, 13):
      X0 = np.asarray(fm.dilate(X, mode=fm.Mode.multilabel, background_only=True, parallel=1)) if level >= 3 else X
      filled, holes = fm.fill_holes_v2(X0, fix_borders=level >= 2, parallel=1,
                                       merge_threshold=1.0 if level <= 3 else 1.0 - 0.01 * (level - 3))
      filled, holes = np.asarray(filled), np.asarray(holes)
      want_f, want_h = F.fill_level(X, level)
      res["%s@%d" % (name, level)] = {"dilate_equals_rule": bool(level < 3 or np.array_equal(X0, F.dilate(X))),
                                      "filled_equals_rule": bool(np.array_equal(filled, want_f)),
                                      "holes_equals_rule": bool(np.array_equal(holes, want_h))}
      arrays["%s_l%d_filled" % (name, level)] = filled
      arrays["%s_l%d_holes" % (name, level)] = holes
    arrays[name] = X
  np.savez_compressed(os.path.join(out, "upstream_fastmorph.npz"), **arrays)
  report["fastmorph"] = res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden"))
  args = ap.parse_args()
  os.makedirs(args.out, exist_ok=True)
  from oracle import oracle as O
  O.build()
  mods = {n: try_import(n) for n in ("tinybrain", "cc3d", "zmesh", "fastremap", "compressed_segmentation",
                                     "fastmorph")}
  report = {"wheels": {n: (getattr(m, "__version__", "present") if m else None) for n, m in mods.items()}}
  verdicts = {}
  if mods["tinybrain"]:
    verdicts["averaging"] = probe_averaging(mods["tinybrain"], O, args.out, report)
    verdicts["mode"] = probe_mode(mods["tinybrain"], O, args.out, report)
  if mods["cc3d"] and mods["fastremap"]:
    verdicts["cc3d"] = probe_cc3d(mods["cc3d"], mods["fastremap"], O, args.out, report)
  if mods["zmesh"]:
    verdicts["zmesh"] = probe_zmesh(mods["zmesh"], O, args.out, report)
  if mods["compressed_segmentation"]:
    verdicts["compressed_segmentation"] = probe_cseg(mods["compressed_segmentation"], O, args.out, report)
  if mods["fastmorph"]:
    probe_fastmorph(mods["fastmorph"], args.out, report)
  report["agrees_with_frozen_defaults"] = verdicts
  report["not_run"] = [k for k, n in (("averaging", "tinybrain"), ("mode", "tinybrain"), ("cc3d", "cc3d"),
                                      ("zmesh", "zmesh"), ("compressed_segmentation", "compressed_segmentation"),
                                      ("fastmorph", "fastmorph")) if not mods[n]]
  with open(os.path.join(args.out, "first_contact_report.json"), "w") as f:
    json.dump(report, f, indent=1)
  print(json.dumps(report, indent=1))
  sys.exit(0 if all(verdicts.values()) else 1)


if __name__ == "__main__":
  main()
