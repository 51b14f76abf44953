"""TEST INFRASTRUCTURE (oracle).  Generates tests/golden/*.pt by EXECUTING THE UNMODIFIED REFERENCE
(/root/reference/distrifuser/modules/pp/*.py, models/distri_sdxl_unet_pp.py, models/naive_patch_sdxl.py,
utils.py:112-199) on CPU under gloo, through the diffusers stub.  Runs only in the build container (the reference
tree does not exist on the GPU box); the vectors it writes are committed.

    python -m oracle.make_golden [--only chain|unet|naive] [--case NAME]
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "diffusers_stub"))

from oracle import harness, naive_patch, workloads  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["chain", "unet", "naive"], default=None)
    ap.add_argument("--case", default=None)
    a = ap.parse_args()
    os.makedirs(GOLDEN, exist_ok=True)
    if a.only in (None, "chain"):
        for case in workloads.CHAIN_CASES:
            if a.case and case.name != a.case:
                continue
            t0 = time.time()
            outs = harness.run_chain(case, impl="reference")
            src = "reference modules @ /root/reference, gloo, fp32"
            path = os.path.join(GOLDEN, f"{case.name}.pt")
            torch.save({"case": case.__dict__, "outs": outs, "source": src}, path)
            if os.path.getsize(path) > 1 << 20:              # fixtures stay below 1 MiB a file: one file per rank instead
                os.unlink(path)
                for r, rank_outs in enumerate(outs):
                    torch.save({"case": case.__dict__, "rank": r, "outs": rank_outs, "source": src},
                               os.path.join(GOLDEN, f"{case.name}.rank{r}.pt"))
            print(f"{case.name}: {time.time() - t0:.1f}s", flush=True)
    if a.only in (None, "unet"):
        for case in workloads.UNET_CASES:
            if a.case and case.name != a.case:
                continue
            t0 = time.time()
            outs = harness.run_unet(case, impl="reference")
            torch.save({"case": case.__dict__, "outs": [o.clone() for o in outs],
                        "source": "reference DistriUNetPP @ /root/reference over oracle/diffusers_stub, gloo, fp32"},
                       os.path.join(GOLDEN, f"unet_{case.name}.pt"))
            print(f"unet_{case.name}: {time.time() - t0:.1f}s  std={outs[-1].std():.4f}", flush=True)
    if a.only in (None, "naive"):
        for case in naive_patch.NAIVE_CASES:
            if a.case and case.name != a.case:
                continue
            t0 = time.time()
            outs = harness.run_unet(case, impl="reference")
            torch.save({"case": case.__dict__, "outs": [o.clone() for o in outs],
                        "source": "reference NaivePatchUNet @ /root/reference over oracle/diffusers_stub, gloo, fp32"},
                       os.path.join(GOLDEN, f"{case.name}.pt"))
            print(f"{case.name}: {time.time() - t0:.1f}s  std={outs[-1].std():.4f}", flush=True)


if __name__ == "__main__":
    main()
