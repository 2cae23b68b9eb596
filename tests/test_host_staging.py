"""The host-buffer entries' staging.  The emulator's host entry runs the C engine's three-stream chunk pipeline, whose slot buffers
it shares with bnm_infer_batch and bnm_infer_topk at other element sizes.  The batched reference kernels and bnm_quantize_images
stage through stream-ordered temporaries on the library's own stream, so they never wait for another stream's work."""
import numpy as np
import pytest

from conftest import load_model
from restate import emulate, scale_images
from support import engine, lib, normal_images, run_emulator  # noqa: F401  (lib: fixture)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["fc", "cnn_48"])
@pytest.mark.parametrize("layers", [False, True])
def test_emulator_host_entry_shares_the_pipeline(lib, oracle, name, layers):
    """128-image chunks: the emulator's float chunks and the C engine's int8 and top-k chunks take turns in the same slot buffers"""
    from bitnetmcu_b200 import _lib
    m = load_model(name)
    e = engine(m, path=_lib.PATH_LAYERS if layers else _lib.PATH_AUTO)
    e.set_option(_lib.OPT_CHUNK_IMAGES, 128)
    x = normal_images(7 * 128 + 5, seed=21)
    want = emulate(m, x)
    assert np.array_equal(run_emulator(e, x)[0], want)
    imgs = np.random.default_rng(22).integers(-128, 128, size=(3000, m.img_bytes)).astype(np.int8)
    want_logits, want_labels = oracle.infer(m, imgs)
    want_classes = np.argsort(-want_logits.astype(np.int64), kind="stable", axis=1)[:, :5]
    for _ in range(2):
        assert np.array_equal(e.inference_quantized(x), want), "emulator host entry"
        logits, labels = e.infer(imgs)
        assert np.array_equal(logits, want_logits) and np.array_equal(labels, want_labels), "bnm_infer_batch"
        classes, scores = e.topk(imgs, 5)
        assert np.array_equal(classes, want_classes), "bnm_infer_topk classes"
        assert np.array_equal(scores, np.take_along_axis(want_logits, want_classes, axis=1)), "bnm_infer_topk scores"
    e.close()


@pytest.mark.gpu
def test_batched_entries_wait_for_their_own_stream_only(lib, oracle):
    """each batched entry returns its results while a kernel on another stream is still running"""
    import torch
    from bitnetmcu_b200 import engine as E
    rng = np.random.default_rng(23)
    n = 64
    act = rng.integers(-128, 128, size=(n, 256)).astype(np.int8)
    w = rng.integers(0, 2 ** 32, size=64 * 256 // 8, dtype=np.uint64).astype(np.uint32)   # 4bitsym, 256 -> 64
    x = rng.integers(-2 ** 20, 2 ** 20, size=(n, 64)).astype(np.int32)
    a16 = rng.integers(0, 1 << 12, size=(n, 256)).astype(np.int32)
    w9 = rng.integers(-128, 128, size=(n, 9)).astype(np.int8)
    f = rng.standard_normal((n, 256)).astype(np.float32)
    calls = {
        "processfclayer": (lambda: E.processfclayer(act, w, 4, 256, 64),
                           np.stack([oracle.fclayer(act[i], w, 4, 256, 64) for i in range(n)])),
        "relunorm": (lambda: E.relunorm(x)[0], np.stack([oracle.relunorm(x[i])[0] for i in range(n)])),
        "conv33relu": (lambda: E.conv33relu(a16, w9, 16), np.stack([oracle.conv33relu(a16[i], w9[i], 16) for i in range(n)])),
        "maxpool22": (lambda: E.maxpool22(a16, 16), np.stack([oracle.maxpool22(a16[i], 16) for i in range(n)])),
        "quantize_images": (lambda: E.quantize_images(f), scale_images(f)),
    }
    for what, (call, want) in calls.items():   # first calls load their kernels
        assert np.array_equal(call(), want), what
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(int(2.0 * 1.98e9))   # about two seconds at the H100's highest SM clock
        busy = torch.cuda.Event()
        busy.record(side)
    try:
        for what, (call, want) in calls.items():
            assert np.array_equal(call(), want), what
            assert not busy.query(), f"{what} waited for another stream's kernel"
    finally:
        side.synchronize()
