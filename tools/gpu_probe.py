"""Pins the wgmma shared-memory descriptor encodings on the GPU by running the raw GEMM probe for every
shared-memory layout and tile width in its own process, and writes the result table as JSON to the path given as the
only argument (default: hb200_probe.json in the system temporary directory).

    python tools/gpu_probe.py [OUT.json]
"""
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = [(layout, n, k) for layout in (0, 1, 2) for (n, k) in ((32, 64), (64, 128), (16, 192), (128, 576))]


def one(layout, n, k):
    import torch
    import habitat_lab_b200 as hb
    from habitat_lab_b200 import ops

    hb.load()
    torch.manual_seed(layout * 100 + n + k)
    m = 256
    a = torch.randn(m, k, device="cuda").to(torch.bfloat16)
    b = torch.randn(n, k, device="cuda").to(torch.bfloat16)
    d = torch.zeros(m, n, device="cuda")
    if layout == 2:
        ops.umma_gemm_probe(a.t().contiguous(), b.t().contiguous(), d, m, n, k, 2)
    else:
        ops.umma_gemm_probe(a, b, d, m, n, k, layout)
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t()
    err = (d - ref).abs().max().item()
    print(json.dumps({"layout": layout, "n": n, "k": k, "max_abs_err": err, "ref_max": ref.abs().max().item()}))


if __name__ == "__main__":
    if len(sys.argv) == 4:
        one(int(sys.argv[1]), int(sys.argv[2]), int(sys.argv[3]))
        sys.exit(0)
    out = []
    for layout, n, k in CASES:
        try:
            p = subprocess.run([sys.executable, __file__, str(layout), str(n), str(k)], capture_output=True,
                               text=True, timeout=180)
            line = [l for l in p.stdout.splitlines() if l.startswith("{")]
            if line:
                out.append(json.loads(line[-1]))
            else:
                out.append({"layout": layout, "n": n, "k": k, "error": (p.stderr or p.stdout)[-400:]})
        except subprocess.TimeoutExpired:
            out.append({"layout": layout, "n": n, "k": k, "error": "timeout"})
        print(out[-1], flush=True)
    path = sys.argv[1] if len(sys.argv) == 2 else os.path.join(tempfile.gettempdir(), "hb200_probe.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print("wrote", path)
