"""Host-side timing of the TMOT association loop (no GPU involved): the native JDE tracker (csrc/tmot.cpp) against the
reference's tmot.multitracker.JDETracker on the same synthetic sequence, both with a CPU embedding distance (the native
one through the cost_fn hook with scipy's cdist -- what the reference calls).  Shows what moving the per-track Python loops
into native code buys on its own; on the GPU the embedding distance additionally moves to the tensor cores.
Needs /root/reference (authoring container only).  Usage: python tools/host_jde_bench.py [n_objects] [frames]"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def main():
    n_obj = int(sys.argv[1]) if len(sys.argv) > 1 else 100
    frames = int(sys.argv[2]) if len(sys.argv) > 2 else 60
    import make_golden_tmot as mg
    mg.install_stubs()
    from scipy.spatial.distance import cdist
    from tmot.multitracker import JDETracker as RefTracker
    from tmot.basetrack import BaseTrack
    from object_detection_tracking_b200.tmot import JDETracker, _IdGroup
    rng = np.random.default_rng(0)
    D = 256
    proto = rng.standard_normal((n_obj, D)).astype(np.float32)
    pos = rng.uniform(50, 1800, (n_obj, 2))
    vel = rng.uniform(-6, 6, (n_obj, 2))
    seq = [[(np.concatenate([pos[o] + vel[o] * f, [40., 90.]]), 0.9,
             proto[o] + 0.1 * rng.standard_normal(D).astype(np.float32)) for o in range(n_obj)] for f in range(frames + 5)]

    def run(make):
        trk = make()
        ids = []
        for f in range(5):
            trk.update([(a.copy(), b, c.copy()) for a, b, c in seq[f]])
        t0 = time.perf_counter()
        for f in range(5, 5 + frames):
            ids.append(sorted(t.track_id for t in trk.update([(a.copy(), b, c.copy()) for a, b, c in seq[f]])))
        return (time.perf_counter() - t0) / frames * 1e3, ids

    BaseTrack._count = 0
    ref_ms, ref_ids = run(lambda: RefTracker(0.5))
    nat_ms, nat_ids = run(lambda: JDETracker(0.5, id_group=_IdGroup(), cost_fn=lambda a, b: cdist(a.astype(np.float64), b.astype(np.float64))))
    print(json.dumps(dict(what="jde_association_host_only", objects=n_obj, frames=frames, feature_dim=D,
                          reference_ms_per_frame=round(ref_ms, 3), native_ms_per_frame=round(nat_ms, 3),
                          speedup=round(ref_ms / nat_ms, 2), identical_track_ids=ref_ids == nat_ids,
                          host="authoring container (no GPU), %d cores" % (os.cpu_count() or 0),
                          note="embedding distance = scipy cdist on the CPU in both arms")))


if __name__ == "__main__":
    main()
