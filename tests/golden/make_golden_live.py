"""Stored outputs of the REAL reference modules for the comparisons that used to need a reference checkout at test time
(tests/test_oracle_golden.py::test_oracle_vs_live_reference, tests/test_s3fd_oracle.py::test_oracle_against_live_reference,
tests/test_abi.py::test_reference_citations_in_the_header_resolve).

    python tests/golden/make_golden_live.py <reference checkout>

writes tests/golden/live_ref.npz (network outputs on the seeded weights / inputs those tests use) and
tests/golden/reference_lines.json (line count of every .py file of the reference, by path relative to its root)."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import s3fd_oracle as S  # noqa: E402
from oracle import w2l_oracle as O  # noqa: E402


def main(ref):
    sys.path.insert(0, ref)
    from models import SyncNet_color, Wav2Lip, Wav2Lip_disc_qual
    sys.path.insert(0, HERE)
    import make_golden_s3fd as G
    G.REF = os.path.join(ref, "face_detection", "detection", "sfd")
    out = {}
    with torch.no_grad():
        sd = O.make_state_dict("generator", 3)
        m = Wav2Lip(); m.load_state_dict(sd, strict=True); m.eval()
        mel, face = O.make_generator_inputs(1, 5)
        out["gen_out"] = m(mel, face).numpy()
        sd = O.make_state_dict("syncnet", 3)
        s = SyncNet_color(); s.load_state_dict(sd, strict=True); s.eval()
        mel, face = O.make_syncnet_inputs(2, 5)
        a, v = s(mel, face)
        out["sync_a"], out["sync_v"] = a.numpy(), v.numpy()
        sd = O.make_state_dict("disc", 3)
        d = Wav2Lip_disc_qual(); d.load_state_dict(sd, strict=True); d.eval()
        out["disc_out"] = d(O.make_disc_inputs(1, 5, 5)).numpy()
        net = G.load_reference()["net_s3fd"].s3fd()
        net.load_state_dict(S.make_state_dict(3), strict=True)
        net.eval()
        for i, o in enumerate(net(S.preprocess(S.make_images(1, 70, 90, seed=5)))):
            out[f"s3fd_o{i}"] = o.numpy()
    np.savez_compressed(os.path.join(HERE, "live_ref.npz"), **out)
    lines = {}
    for dp, _dn, fn in os.walk(ref):
        for f in fn:
            if f.endswith(".py"):
                p = os.path.join(dp, f)
                lines[os.path.relpath(p, ref)] = sum(1 for _ in open(p, errors="replace"))
    with open(os.path.join(HERE, "reference_lines.json"), "w") as f:
        json.dump(dict(sorted(lines.items())), f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1])
