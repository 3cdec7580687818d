"""Record tests/golden/sd20_registry.json: the parameter registry of the SD-2.0 engine (U-Net, VAE encoder and decoder at their
benchmark sizes), one [name, shape] entry per registry slot, in registry order.  StableDiffusion.__init__ draws the seeded
stand-in weights in this order, so the order decides what the seeded workload computes; tests/test_sd_fullsize_gpu.py holds the
engine to it.  The registry is read from a planned engine, so this needs the GPU.
    python tests/golden/make_golden_sd_registry.py"""
import importlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "sd20_registry.json")


def main():
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    eng = sdm.SDEngine(sdm.sd20_unet_cfg(), sdm.sd_vae_cfg(), "cuda")
    rows = [json.dumps([n, list(s)]) for n, s in zip(eng.names, eng.shapes)]
    with open(OUT, "w") as f:
        f.write("[\n" + ",\n".join(rows) + "\n]\n")
    print(f"wrote {OUT}: {len(rows)} entries")


if __name__ == "__main__":
    main()
