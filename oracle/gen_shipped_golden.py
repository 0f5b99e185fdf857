"""TEST INFRASTRUCTURE -- fixtures of the reference's two shipped trained models, for tests/test_shipped_models.py.
Runs the UNMODIFIED reference on CPU (oracle/ref_harness.py) and writes

    tests/golden/shipped/{barbershop_k4,pavillon_k16}/   the shipped export directories byte for byte: config.ini and
                                                         dataset_info.txt as they are, each model{0,1}.onnx as raw parts
                                                         of at most 1 MB, manifest.json with every file's size and sha256
    tests/golden/weights_barbershop/                     the Barbershop networks' initialisers (as weights_pavillon)
    tests/golden/barber_k4_t0.15.npz                     the reference's stages for the trained Barbershop networks at
    tests/golden/barber_k16_t0.5.npz                     the shipped setting and at a ragged, mostly uncapped one

    python oracle/gen_shipped_golden.py

Running it twice writes identical bytes.
"""
import hashlib
import json
import os
import shutil
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh          # noqa: E402
from oracle import adanerf_oracle as orc      # noqa: E402
from oracle.gen_golden import OUT, RX, meta, save, stage_case  # noqa: E402
from adanerf_b200.onnx_weights import read_onnx_initializers  # noqa: E402

SHIPPED = {"barbershop_k4": os.path.join("adanerf_real_time_viewer", "sample"),
           "pavillon_k16": os.path.join("adanerf_real_time_viewer", "sample_pavillon_16")}
TEXT_FILES = ("config.ini", "dataset_info.txt")
MODEL_FILES = ("model0.onnx", "model1.onnx")
PART_BYTES = 1_000_000
# a pose inside the Barbershop view cell (half extents 0.75, 0.75, 0.2) that is not its centre, looking along the floor
BARBER_POSE_OFF = [0.3, -0.2, 0.08]
BARBER_ROT = orc.rotation_yaw(35.0) @ RX
# the shipped setting, and one where sample counts are ragged: every ray of the trained sampling net has 17 or more cells
# >= 0.05, so K = 8 / thr 0.05 would cap them all, while at K = 16 / thr 0.5 a fifth are capped, a third fall back to the
# arg-max cell and the rest take 2..15 samples
BARBER_CASES = [("barber_k4_t0.15", 4, 0.15, True), ("barber_k16_t0.5", 16, 0.5, False)]


def copy_export_dir(name, rel):
    src = os.path.join(rh.REF_ROOT, rel)
    dst = os.path.join(OUT, "shipped", name)
    if os.path.isdir(dst):
        shutil.rmtree(dst)
    os.makedirs(dst)
    manifest = {}
    for f in TEXT_FILES + MODEL_FILES:
        with open(os.path.join(src, f), "rb") as fh:
            data = fh.read()
        entry = dict(size=len(data), sha256=hashlib.sha256(data).hexdigest())
        if f in MODEL_FILES:
            entry["parts"] = []
            for i in range(0, len(data), PART_BYTES):
                part = f"{f}.part{i // PART_BYTES}"
                with open(os.path.join(dst, part), "wb") as fh:
                    fh.write(data[i:i + PART_BYTES])
                entry["parts"].append(part)
        else:
            with open(os.path.join(dst, f), "wb") as fh:
                fh.write(data)
        manifest[f] = entry
    manifest = dict(source=rel.replace(os.sep, "/"), files=manifest)
    with open(os.path.join(dst, "manifest.json"), "w") as fh:
        json.dump(manifest, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(f"wrote {dst}")


def barbershop():
    d = os.path.join(rh.REF_ROOT, SHIPPED["barbershop_k4"])
    w0 = read_onnx_initializers(os.path.join(d, "model0.onnx"))
    w1 = read_onnx_initializers(os.path.join(d, "model1.onnx"))
    save("weights_barbershop.npz", meta=meta(source="adanerf_real_time_viewer/sample/model{0,1}.onnx initialisers"),
         **{"sd0/" + k: v for k, v in w0.items()}, **{"sd1/" + k: v for k, v in w1.items()})
    sd0 = {k: torch.from_numpy(v) for k, v in w0.items()}
    sd1 = {k: torch.from_numpy(v) for k, v in w1.items()}
    for name, K, thr, keep_x1 in BARBER_CASES:
        stage_case(name, "barbershop", orc.SCENE_BARBERSHOP, sd0, sd1, K, thr, 256, 2503, BARBER_POSE_OFF, BARBER_ROT,
                   keep_x1)


def main():
    assert rh.available(), "needs the reference checkout (ADANERF_REFERENCE)"
    torch.set_num_threads(8)
    for name, rel in SHIPPED.items():
        copy_export_dir(name, rel)
    barbershop()


if __name__ == "__main__":
    main()
