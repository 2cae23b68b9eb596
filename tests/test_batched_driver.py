"""host/test_inference_batched.py -- the batched counterpart of the reference's evaluation loop
(/root/reference/test_inference.py:130-175; SURVEY.md 8f rank 1)."""
import gzip
import importlib.util
import os
import struct

import numpy as np
import pytest

from restate import scale_images

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _driver():
    spec = importlib.util.spec_from_file_location("test_inference_batched", os.path.join(ROOT, "host", "test_inference_batched.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _float_set(n_rep=40, seed=0):
    """Float images whose reference-style int8 scaling is known: the reference's ten test digits (golden/digits.npz, already
    +-127 int8) times a random positive scale per image -- scaling back by 127/max|x| returns the digit exactly."""
    z = np.load(os.path.join(GOLD, "digits.npz"))
    rng = np.random.default_rng(seed)
    imgs = np.tile(z["images"].astype(np.float32), (n_rep, 1))
    labels = np.tile(z["labels"].astype(np.int64), n_rep)
    # powers of two keep x * (127 / max|x|) exact, so the expected int8 image is the digit itself
    scale = np.exp2(rng.integers(-6, 4, size=(imgs.shape[0], 1))).astype(np.float32)
    return imgs * scale / np.float32(127.0) * np.float32(127.0), labels, np.tile(z["images"], (n_rep, 1))


def test_idx_and_npz_loaders(tmp_path):
    d = _driver()
    rng = np.random.default_rng(1)
    imgs = rng.integers(0, 256, size=(7, 28, 28), dtype=np.uint8)
    labels = rng.integers(0, 10, size=7, dtype=np.uint8)
    with gzip.open(tmp_path / "t10k-images-idx3-ubyte.gz", "wb") as f:
        f.write(struct.pack(">IIII", 0x00000803, 7, 28, 28) + imgs.tobytes())
    with open(tmp_path / "t10k-labels-idx1-ubyte", "wb") as f:
        f.write(struct.pack(">II", 0x00000801, 7) + labels.tobytes())
    x, y = d.load_dataset(str(tmp_path), 16)
    assert x.shape == (7, 256) and x.dtype == np.float32 and np.array_equal(y, labels)
    lo, hi = (0 - 0.1307) / 0.3081, (1 - 0.1307) / 0.3081
    assert x.min() >= lo - 1e-4 and x.max() <= hi + 1e-4           # Normalize(0.1307, 0.3081) of [0, 1] pixels
    np.savez(tmp_path / "set.npz", images=x.reshape(7, 16, 16), labels=y)
    x2, y2 = d.load_dataset(str(tmp_path / "set.npz"))
    assert np.array_equal(x2, x) and np.array_equal(y2, y)


def test_scaling_recipe_matches_reference_expression():
    """The CPU-side statement of test_inference.py:140-141 used as the expectation in the GPU test."""
    x, _, digits = _float_set(3)
    q = scale_images(x)
    # every shipped test digit has a +127 pixel, so the recipe returns the digit itself
    assert np.array_equal(q, digits)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["fc", "cnn"])
def test_batched_evaluation_matches_reference(which):
    d = _driver()
    from bitnetmcu_b200.model import Model
    model = Model.load(os.path.join(GOLD, "models", which + ".bnm"))
    x, labels, digits = _float_set(40)
    lines = []
    res = d.evaluate(model, x, labels, out=lines.append)
    assert np.array_equal(res["quantized"], digits)
    # "Mismatches between engines" (test_inference.py:166-175): the unmodified reference C code on the same int8 images
    from oracle.oracle import Oracle, Reference
    ref_logits, ref_labels = (Reference() if Reference.available() else Oracle()).infer(model, res["quantized"])
    assert np.array_equal(ref_labels, res["predicted"]) and np.array_equal(ref_logits, res["logits"])
    # the reference scores 10/10 on its own test digits with both shipped models (BitNetMCU_MNIST_test.c)
    assert res["n"] == 400 and res["correct_c"] == 400
    assert lines[0] == "size of test data: 400" and lines[1] == "Mispredictions C: 0" and lines[2] == "Overall accuracy C: 100.0 %"
