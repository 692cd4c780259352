"""Writes tests/golden/relink.npz: the reference's single-video tracklet re-linking (single_video_reid.py preprocess /
reid / save_new_track, run on the CPU) on the synthetic video of tests/relink_inputs.py, with the real torchreid
extractors: osnet_x1_0 loaded with synth_osnet_state(4321) and resnet101 with synth_resnet101_reid_state(2468).

The driver's module-level imports that are absent here or need TF are stubbed with MagicMock (as
make_golden_tmot.py:reid_pairs does); expand_tlwh / tlwh_intersection / valid_box are taken out of the reference's
utils.py with `ast` (utils.py imports TF).  `args` is SimpleNamespace(debug=False).

For each parameter set of relink_inputs.RUNS the file holds, as one JSON string per run:
  * the candidates preprocess returned for both classes, and after reid (rows [id, start, end, dist], sorted);
  * the reference's needed_track_boxes (key -> boxes, in its order) and the box indices of each key's valid crops;
  * the margins of every decision (see below);
and the bytes of both merged track files that save_new_track wrote.

Margins: a GPU distance differs from the CPU one in the last bits of ~70-100 layers of fp32, so the generator asserts
that no decision sits close to a tie.  For every compared query: each gap between two of its sorted distances, and the
distance of each to the threshold, is at least MARGIN relative to the larger value.  The smallest of each is recorded.
Run: python tests/golden/make_golden_relink.py
"""
import ast
import json
import os
import sys
import tempfile
import types
from types import SimpleNamespace
from unittest.mock import MagicMock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
OUT = os.path.join(HERE, "relink.npz")
MARGIN = 0.02

sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import relink_inputs as ri  # noqa: E402


def reference_utils():
    src = open(os.path.join(REF, "utils.py")).read()
    tree = ast.parse(src)
    keep = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("expand_tlwh", "tlwh_intersection",
                                                                                  "valid_box")]
    mod = types.ModuleType("utils")
    mod.np = np
    exec(compile(ast.Module(body=keep, type_ignores=[]), "utils.py", "exec"), mod.__dict__)
    mod.parse_meva_clip_name = MagicMock()
    mod.sec2time = MagicMock()
    return mod


def load_driver():
    sys.modules["utils"] = reference_utils()
    for m in ("enqueuer_thread", "diva_io", "diva_io.video", "moviepy", "moviepy.editor", "matplotlib"):
        sys.modules.setdefault(m, MagicMock())
    sys.path.insert(0, REF)
    import single_video_reid as svr
    svr.args = SimpleNamespace(debug=False)
    return svr


def extractors():
    import torch
    from torchreid.feature_extractor import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_osnet_state, synth_resnet101_reid_state
    out = []
    for name, size, state in (("osnet_x1_0", (256, 128), synth_osnet_state(4321)),
                              ("resnet101", (128, 256), synth_resnet101_reid_state(2468))):
        ext = FeatureExtractor(name, model_path="", image_size=size, device="cpu", verbose=False)
        sd = ext.model.state_dict()
        for k, v in state.items():
            sd[k].copy_(torch.from_numpy(v))
        ext.model.load_state_dict(sd)
        ext.model.eval()
        out.append(ext)
    return out


def cand_json(c):
    return [[float(q), [[float(v) for v in row] for row in c[q]]] for q in c]


class Spy(object):
    """The frame iterator: yields the video's batches and, when the driver's loop asks for the frame after the last,
    copies the driver's needed_track_boxes and the valid crops' box indices out of its frame."""

    def __init__(self, video):
        self.video = video
        self.needed = None
        self.valid = None

    def __iter__(self):
        for f in range(len(self.video)):
            yield [(self.video[f], 1.0, f)]
        fr = sys._getframe(1)
        while "needed_track_box_imgs" not in fr.f_locals:
            fr = fr.f_back
        self.needed = [[k, [[float(x) for x in b] for b in v]] for k, v in fr.f_locals["needed_track_boxes"].items()]
        self.valid = {k: sorted(int(i) for i in v) for k, v in fr.f_locals["needed_track_box_imgs"].items()}


def margins(cands, thr):
    gap, to_thr = np.inf, np.inf
    for q in cands:
        d = [float(r[-1]) for r in cands[q]]
        for i in range(len(d)):
            to_thr = min(to_thr, abs(d[i] - thr) / max(abs(d[i]), abs(thr)))
            for j in range(i + 1, len(d)):
                gap = min(gap, abs(d[i] - d[j]) / max(abs(d[i]), abs(d[j])))
    return gap, to_thr


def main():
    svr = load_driver()
    p_ext, v_ext = extractors()
    video = ri.frames()
    tmp = tempfile.mkdtemp()
    pf = ri.write_track_file(os.path.join(tmp, "p.txt"), ri.track_rows("p"))
    vf = ri.write_track_file(os.path.join(tmp, "v.txt"), ri.track_rows("v"))
    data = {}
    for r, (box_num, gap, method) in enumerate(ri.RUNS):
        _, p_data, p_cand = svr.preprocess(pf, ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
        _, v_data, v_cand = svr.preprocess(vf, ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
        before = {"p": cand_json(p_cand), "v": cand_json(v_cand)}
        spy = Spy(video)
        thr = ri.THRESHOLD[method]
        new_p, new_v = svr.reid((spy, len(video)), p_ext, v_ext, p_data, p_cand, v_data, v_cand,
                                feature_box_num=box_num, feature_box_gap=gap, reject_dist_thres=thr,
                                compare_method=method)
        print("run %d (%s): person %s" % (r, method, {q: [(row[0], round(float(row[-1]), 3)) for row in p_cand[q]]
                                                      for q in p_cand}))
        print("             vehicle %s" % {q: [(row[0], round(float(row[-1]), 3)) for row in v_cand[q]] for q in v_cand})
        g_p, t_p = margins(p_cand, thr)
        g_v, t_v = margins(v_cand, thr)
        print("  margins: gap %.4f / %.4f, to threshold %.4f / %.4f" % (g_p, g_v, t_p, t_v))
        if os.environ.get("PROBE") is None:
            assert min(g_p, g_v, t_p, t_v) >= MARGIN, "a decision is too close to a tie"
        out_dir = os.path.join(tmp, "run%d" % r)
        svr.save_new_track("Person", new_p, out_dir, "video.mp4")
        svr.save_new_track("Vehicle", new_v, out_dir, "video.mp4")
        for cat in ("Person", "Vehicle"):
            raw = open(os.path.join(out_dir, "video.mp4", cat, "video.txt"), "rb").read()
            data["run%d_%s" % (r, cat)] = np.frombuffer(raw, np.uint8)
        info = {"params": [box_num, gap, thr, method], "before": before,
                "after": {"p": cand_json(p_cand), "v": cand_json(v_cand)},
                "needed": spy.needed, "valid": spy.valid, "new_ids": {"p": sorted(new_p), "v": sorted(new_v)},
                "margins": {"gap": min(g_p, g_v), "threshold": min(t_p, t_v)}}
        data["run%d_json" % r] = np.asarray(json.dumps(info))
    np.savez_compressed(OUT, **data)
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
