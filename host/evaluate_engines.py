#!/usr/bin/env python
"""Both engines of the reference's evaluation loop (/root/reference/test_inference.py:130-175), batched.

test_inference.py scores every test image twice: with the C engine (`lib.Inference()` on the int8-scaled image) and with the
Python emulator (`np.argmax(quantized_model.inference_quantized(x))`, test_inference.py:153-154), and prints both accuracies and
the number of images on which the two disagree.  host/test_inference_batched.py prints the C-engine half; this driver runs it
unchanged and then the emulator on the GPU on the same float images, held in device memory:

    labels_py = bnm_emulate_batch_device(model, float images)     # one kernel for FC models up to 64 wide

and adds the reference's other lines: "Mispredictions Py", "Overall accuracy Python" and "Mismatches between engines".
Arguments and data as for host/test_inference_batched.py.

There is no CPU fallback: without a CUDA device the engine raises.
"""
import argparse
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _c_driver():
    spec = importlib.util.spec_from_file_location("test_inference_batched", os.path.join(ROOT, "host", "test_inference_batched.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def evaluate(model, images_f32, labels, out=print):
    """The C-engine report of host/test_inference_batched.py, then the emulator's lines; returns the counters of both."""
    import torch
    from bitnetmcu_b200.engine import Engine
    res = _c_driver().evaluate(model, images_f32, labels, out=out)
    eng = Engine(model)
    x = torch.from_numpy(np.ascontiguousarray(images_f32, dtype=np.float32).reshape(-1, eng.img_bytes)).cuda()
    lab = torch.empty(x.shape[0], dtype=torch.int32, device=x.device)
    eng.inference_quantized_device(x, None, lab)          # test_inference.py:153-154, whole set at once
    predicted_py = lab.cpu().numpy().astype(np.int64)     # synchronises torch's current stream
    eng.close()
    n = res["n"]
    correct_py = int((predicted_py == labels).sum())
    mismatch = int((predicted_py != res["predicted"].astype(np.int64)).sum())
    res.update(correct_py=correct_py, predicted_py=predicted_py, mismatch=mismatch)
    out(f"Mispredictions Py: {n - correct_py}")
    out(f"Overall accuracy Python: {correct_py / max(n, 1) * 100} %")
    out(f"Mismatches between engines: {mismatch} ({mismatch / max(n, 1) * 100}%)")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", default="BitNetMCU_model.h", help="model header (exportquant.py output) or .bnm blob")
    ap.add_argument("--data", required=True, help=".npz with images/labels, or a directory with the MNIST t10k idx files")
    args = ap.parse_args()
    drv = _c_driver()
    model = drv.load_model(args.model)
    side = int(round(model.img_bytes ** 0.5))
    x, y = drv.load_dataset(args.data, side)
    print(f"model: {model.describe()}")
    evaluate(model, x, y)


if __name__ == "__main__":
    main()
