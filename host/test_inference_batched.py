#!/usr/bin/env python
"""Batched counterpart of the reference's C-engine evaluation loop (/root/reference/test_inference.py:130-175).

The reference feeds the MNIST test set to `lib.Inference()` one image at a time: per image it flattens the normalised
16x16 float image, scales it to int8 (test_inference.py:140-141) and calls the DLL.  Here the whole set takes three calls:

    q      = bnm_quantize_images(float images)          # same float32 arithmetic, on the GPU, bit-identical
    logits, predicted = bnm_infer_batch(model, q)       # the fused sm_90a kernel
    accuracy = mean(predicted == labels)

and prints the reference's summary lines ("size of test data", "Mispredictions C", "Overall accuracy C").  The
engine-vs-engine comparison the reference prints ("Mismatches between engines") lives in tests/test_batched_driver.py,
where the same set is also pushed through the unmodified reference C code and must agree bit for bit.

Data (no dataset ships with the sandbox, so it has to be pointed at one):
    --data set.npz          arrays `images` float32 [n,16,16] | [n,256] (already resized + normalised like the reference's
                            transform: Resize(16,16), ToTensor, Normalize(0.1307, 0.3081)) and `labels` int [n]
    --data <dir>            a directory holding MNIST's t10k-images-idx3-ubyte[.gz] + t10k-labels-idx1-ubyte[.gz]; the
                            28x28 images are resized with antialiased bilinear interpolation and normalised as above
Model: a BitNetMCU_model.h written by exportquant.py (or this repo's packer), or a .bnm blob.

There is no CPU fallback: without a CUDA device the engine raises.
"""
import argparse
import gzip
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_idx(path):
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rb") as f:
        raw = f.read()
    magic, = struct.unpack(">I", raw[:4])
    ndim = magic & 0xFF
    dims = struct.unpack(">" + "I" * ndim, raw[4:4 + 4 * ndim])
    return np.frombuffer(raw, dtype=np.uint8, offset=4 + 4 * ndim).reshape(dims)


def find(dirname, stem):
    for name in (stem, stem + ".gz", stem.replace("-idx", ".idx"), stem.replace("-idx", ".idx") + ".gz"):
        p = os.path.join(dirname, name)
        if os.path.exists(p):
            return p
    raise FileNotFoundError(f"{stem}[.gz] not found in {dirname}")


def load_dataset(path, side=16):
    """-> float32 [n, side*side] normalised images, int64 [n] labels"""
    if os.path.isdir(path):
        import torch
        import torch.nn.functional as F
        imgs = load_idx(find(path, "t10k-images-idx3-ubyte")).astype(np.float32) / 255.0
        labels = load_idx(find(path, "t10k-labels-idx1-ubyte")).astype(np.int64)
        t = torch.from_numpy(imgs)[:, None]
        t = F.interpolate(t, size=(side, side), mode="bilinear", antialias=True, align_corners=False)
        x = ((t - 0.1307) / 0.3081).reshape(len(labels), -1).numpy()
        return np.ascontiguousarray(x, dtype=np.float32), labels
    z = np.load(path)
    x = np.asarray(z["images"], dtype=np.float32)
    return np.ascontiguousarray(x.reshape(x.shape[0], -1)), np.asarray(z["labels"]).astype(np.int64).reshape(-1)


def load_model(path):
    from bitnetmcu_b200.model import Model, parse_header
    return Model.load(path) if path.endswith(".bnm") else parse_header(path)


def evaluate(model, images_f32, labels, out=print):
    """Runs the set through the GPU engine; returns a dict with the reference's counters."""
    from bitnetmcu_b200.engine import Engine, quantize_images
    eng = Engine(model)
    q = quantize_images(images_f32)                       # test_inference.py:140-141, whole set at once
    logits, predicted = eng.infer(q)
    eng.close()
    n = len(labels)
    correct = int((predicted.astype(np.int64) == labels).sum())
    res = {"n": n, "correct_c": correct, "logits": logits, "predicted": predicted, "quantized": q}
    out(f"size of test data: {n}")
    out(f"Mispredictions C: {n - correct}")
    out(f"Overall accuracy C: {correct / max(n, 1) * 100} %")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--model", default="BitNetMCU_model.h", help="model header (exportquant.py output) or .bnm blob")
    ap.add_argument("--data", required=True, help=".npz with images/labels, or a directory with the MNIST t10k idx files")
    args = ap.parse_args()
    model = load_model(args.model)
    side = int(round(model.img_bytes ** 0.5))
    x, y = load_dataset(args.data, side)
    print(f"model: {model.describe()}")
    evaluate(model, x, y)


if __name__ == "__main__":
    main()
