#!/usr/bin/env python
"""Top-k accuracy of the C engine, batched: the evaluation of host/test_inference_batched.py plus one line.

host/test_inference_batched.py prints the reference's C-engine summary ("size of test data", "Mispredictions C", "Overall
accuracy C").  This driver runs it unchanged, then asks the engine for each image's K best classes on the same int8-scaled
images (bnm_infer_topk: ranked by logit, ties to the lower class, no logits written or copied back) and adds

    Top-K accuracy C: x %

the share of images whose label is among those K classes.  Models with more than 10 classes (EMNIST letters: 26 or 37,
balanced: 47) are usually reported this way.  Arguments and data as for host/test_inference_batched.py, plus --topk K
(1 <= K <= min(classes, 16), default 5).

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


def evaluate(model, images_f32, labels, k, out=print):
    """The C-engine report of host/test_inference_batched.py, then the top-k line; returns its counters and correct_topk_c."""
    from bitnetmcu_b200.engine import Engine
    res = _c_driver().evaluate(model, images_f32, labels, out=out)
    eng = Engine(model)
    classes, _ = eng.topk(res["quantized"], k, want_scores=False)   # the same int8 images the report scored
    eng.close()
    n = res["n"]
    res["classes"] = classes
    res["correct_topk_c"] = int((classes.astype(np.int64) == np.asarray(labels, dtype=np.int64)[:, None]).any(axis=1).sum())
    out(f"Top-{k} accuracy C: {res['correct_topk_c'] / max(n, 1) * 100} %")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", default="BitNetMCU_model.h", help="model header (exportquant.py output) or .bnm blob")
    ap.add_argument("--data", required=True, help=".npz with images/labels, or a directory with the MNIST t10k idx files")
    ap.add_argument("--topk", type=int, default=5, metavar="K", help="classes per image (1 <= K <= min(classes, 16))")
    args = ap.parse_args()
    drv = _c_driver()
    model = drv.load_model(args.model)
    side = int(round(model.img_bytes ** 0.5))
    x, y = drv.load_dataset(args.data, side)
    print(f"model: {model.describe()}")
    evaluate(model, x, y, args.topk)


if __name__ == "__main__":
    main()
