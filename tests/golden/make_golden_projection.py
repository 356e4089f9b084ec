"""Records the unmodified reference cube-map transformers (habitat_baselines/common/obs_transformers.py
CubeMap2Equirect, CubeMap2Fisheye, Equirect2CubeMap) on small seeded inputs, with torch's CPU grid_sample, into
tests/golden/projection.pt.  Each case keeps the reference converter's own table (from its grids) and depth factors
next to its output: their last bits follow the recording host's torch.sqrt (DESIGN §8.2b), so the GPU tests feed
these tables to the kernel and hold it to these bytes whatever host runs them.  torch.sqrt of a probe is kept too, so
the CPU tests can tell whether their host rounds it the same way.  Run from the repository root:
    python tests/golden/make_golden_projection.py
"""
import logging
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from oracle import ref_shim  # noqa: E402
from projection_reference import GOLDEN_CASES, golden_faces, sqrt_probe_input, table_from_grids  # noqa: E402


def main():
    ref_shim.install()
    if "habitat.core.logging" not in sys.modules:
        sys.modules["habitat.core.logging"] = types.ModuleType("habitat.core.logging")
        sys.modules["habitat.core.logging"].logger = logging.getLogger("habitat")
    import habitat_baselines.common.obs_transformers as m

    rec = {"cpu_capability": torch.backends.cpu.get_cpu_capability(), "torch": str(torch.__version__),
           "sqrt_probe": torch.sqrt(sqrt_probe_input())}
    make = {"c2e": lambda k, hw, _: m.CubeMap2Equirect(k, hw),
            "c2f": lambda k, hw, fish: m.CubeMap2Fisheye(k, hw, *fish),
            "e2c": lambda k, hw, _: m.Equirect2CubeMap(k, hw)}
    for name, (kind, out_hw, fish, key, shape, dtype) in GOLDEN_CASES.items():
        obs = golden_faces(name)
        t = make[kind](list(obs), out_hw, fish)
        out = t({k: v.clone() for k, v in obs.items()})[f"{key}_0"]
        conv = t.converter
        is_depth = key == "depth"
        zf = lambda z: None if z is None or not is_depth else z[:, 0].contiguous()  # noqa: E731
        # the faces are regenerated from their seed; the sum checks that they were
        rec[name] = {"faces_sum": sum(float(v.double().sum()) for v in obs.values()), "out": out.contiguous(),
                     "table": table_from_grids(conv.grids), "n_in": conv.input_len,
                     "in_zf": zf(conv.input_zfactor), "out_zf": zf(conv.output_zfactor)}
    torch.save(rec, os.path.join(ROOT, "tests", "golden", "projection.pt"))


if __name__ == "__main__":
    main()
