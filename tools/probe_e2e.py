#!/usr/bin/env python3
"""PCIe probe (pinned H2D / D2H alone and together) and an e2e sweep over slice count / K1 variant for the host-buffer path."""
import json, os, subprocess, sys, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

def pcie():
    n = 2 << 30
    h1 = torch.empty(n, dtype=torch.uint8).pin_memory(); h2 = torch.empty(n, dtype=torch.uint8).pin_memory()
    d1 = torch.empty(n, dtype=torch.uint8, device="cuda"); d2 = torch.empty(n, dtype=torch.uint8, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    def t(fn):
        torch.cuda.synchronize(); t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); return time.perf_counter() - t0
    def h2d():
        with torch.cuda.stream(s1): d1.copy_(h1, non_blocking=True)
    def d2h():
        with torch.cuda.stream(s2): h2.copy_(d2, non_blocking=True)
    def both(): h2d(); d2h()
    for f in (h2d, d2h, both): t(f)
    r = {"h2d_GBps": n / t(h2d) / 1e9, "d2h_GBps": n / t(d2h) / 1e9}
    tb = t(both); r["both_GBps_each"] = n / tb / 1e9
    print(json.dumps(r))

if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "pcie":
        pcie(); sys.exit(0)
    subprocess.run([sys.executable, __file__, "pcie"])
    for k1 in ("", "lut"):
        for S in (8, 16, 32):
            env = dict(os.environ, SWC_HOST_SLICES=str(S))
            if k1: env["SWC_DEFLATE_K1"] = k1
            out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "3", "--units", "65536", "--no-cpu", "--e2e-steps", "4"],
                                 env=env, capture_output=True, text=True).stdout.strip().splitlines()
            try:
                d = json.loads(out[-1]); print("K1=%s S=%d e2e %.2f GB/s" % (k1 or "auto", S, d["e2e"]["value"]))
            except Exception as e:
                print("K1=%s S=%d failed: %s" % (k1 or "auto", S, out[-3:]))
