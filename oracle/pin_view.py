"""Pin the agent's debug view (oracle/view_ref.py) against the REFERENCE and write tests/golden/agent_view.npz.  Every other golden
is left untouched.

Runs only where the reference sources and cv2 are readable.  It imports the unmodified team_code_v2/lav_agent_fast.py
(leaderboard.autoagents, agents.navigation and carla come from oracle/refshim) and calls LAVAgent.visualize on a stub ``self``
that holds the config attributes it reads (min_x, max_x, min_y, max_y, pixels_per_meter, cmd_thresh; lav_agent_fast.py:71-72),
once per seeded case of oracle.view_ref.view_case (no detections and 15, scores at fp32 0.2 and one ulp either side, boxes partly
off the image, a target past pixel 255, points on the bin edges and the last edge, commands 4 and 5, ...).  matplotlib is not
installed where this runs: matplotlib.cm.get_cmap('jet') is served by view_ref's restatement of matplotlib's jet
(LinearSegmentedColormap of _jet_data, N = 256, Colormap.__call__), which is therefore not pinned by this script.  It checks
view_ref.case_frame against every frame and stores the seed, the case kinds and the reference's frames (the inputs are
regenerated from the seed).

    python oracle/pin_view.py
"""
import os
import sys
import types

import numpy as np
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("LAV_REFERENCE", "/root/reference")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "refshim"))
sys.path.insert(0, os.path.join(REF, "team_code_v2"))

from oracle import view_ref as V  # noqa: E402

SEED = 2026
GOLD = os.path.join(ROOT, "tests", "golden", "agent_view.npz")
VIEW_KEYS = ("min_x", "max_x", "min_y", "max_y", "pixels_per_meter", "cmd_thresh")


class _Jet:
    """matplotlib Colormap.__call__ on a scalar: (r, g, b, a) of the row view_ref.jet_index picks."""

    def __init__(self):
        self.lut = V.jet_rgba()

    def __call__(self, x):
        return tuple(float(v) for v in self.lut[int(V.jet_index(x))])


def main():
    import matplotlib.cm
    import torch
    matplotlib.cm.get_cmap = lambda name: _Jet() if name == "jet" else None
    from lav_agent_fast import LAVAgent
    full = yaml.safe_load(open(os.path.join(REF, "team_code_v2", "config.yaml")))
    s = types.SimpleNamespace(**{k: full[k] for k in VIEW_KEYS})
    frames = []
    for kind in V.VIEW_KINDS:
        c = V.view_case(SEED, kind)
        ref = LAVAgent.visualize(s, c["rgb"], c["tel"], torch.from_numpy(c["points"]), c["pred_bra"], c["sig_bev"], c["plan"],
                                 c["cast_locs"], c["cast_cmds"], [[], c["boxes"]], [float(v) for v in c["tgt"]], c["cmd"],
                                 c["spd"], c["steer"], c["throt"], c["brake"])
        mine = V.case_frame(c, s.pixels_per_meter, s.cmd_thresh)
        bad = int((ref != mine).any(-1).sum())
        print(f"{kind:>11}: {len(c['boxes']):2d} boxes, {bad} pixels differ")
        assert bad == 0, kind
        frames.append(ref)
    np.savez_compressed(GOLD, seed=SEED, kinds=np.array(V.VIEW_KINDS), frames=np.stack(frames),
                        config=np.array([full[k] for k in VIEW_KEYS], dtype=np.float64))
    print(f"wrote {GOLD} ({os.path.getsize(GOLD) / 1e3:.0f} kB)")


if __name__ == "__main__":
    main()
