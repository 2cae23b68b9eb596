"""Pin the oracle (oracle/bitnet_oracle.c) against the reference: golden vectors made by the unmodified
reference kernels (tests/golden/make_golden.py), the reference's own label KAT, and random function-level comparisons against
outputs recorded from the reference itself (tests/golden/make_reference_vectors.py)."""
import json
import os
import zlib

import numpy as np
import pytest

from conftest import GOLDEN, load_model, model_names, xorshift_images
from golden import reference_cases as RC
from bitnetmcu_b200 import model as M
from bitnetmcu_b200 import pack as P


@pytest.mark.parametrize("name", model_names())
def test_oracle_matches_golden_logits(oracle, golden, digits, name):
    m = load_model(name)
    imgs, _ = digits
    lo, la = oracle.infer(m, imgs, threads=1)
    assert np.array_equal(lo, golden[name + "/digits_logits"])
    assert np.array_equal(la, golden[name + "/digits_labels"])
    xs = oracle.xorshift_images(256)
    lo, la = oracle.infer(m, xs, threads=2)
    assert np.array_equal(lo, golden[name + "/xs_logits"])
    assert np.array_equal(la, golden[name + "/xs_labels"])


def test_reference_label_kat(oracle, digits):
    """BitNetMCU_MNIST_test.c:17-40: predicted == label for both shipped models (config #1)."""
    imgs, labels = digits
    kat = json.load(open(os.path.join(GOLDEN, "kat.json")))
    assert kat["reference_labels"] == labels.tolist() == kat["dll_fc_labels"] == kat["dll_cnn_labels"]
    for name in ("fc", "cnn", "12k", "12k_FP130", "1k", "cnn_48", "cnn_32", "cnn_16", "binary160"):
        _, la = oracle.infer(load_model(name), imgs)
        assert la.tolist() == labels.tolist(), name


def test_survey_kats(oracle):
    """SURVEY.md 8c synthetic KAT: CRC-32 of the first 1000x10 logits, label sums."""
    kat = json.load(open(os.path.join(GOLDEN, "kat.json")))
    xs = oracle.xorshift_images(1000)
    assert xs[0, :8].tolist() == kat["xorshift_first_pixels"] == [122, -81, -96, -22, -45, 98, -104, 56]
    assert np.array_equal(xs[:4], xorshift_images(4))
    lo, la = oracle.infer(load_model("fc"), xs)
    assert lo[0].tolist() == kat["fc_xs_logits0"]
    assert "%08x" % zlib.crc32(lo.astype("<i4").tobytes()) == kat["fc_xs_crc32_first1000"] == "fc621bad"
    assert int(la.sum()) == kat["fc_xs_sum_labels_1000"] == 4064
    xs = oracle.xorshift_images(40000)
    _, la = oracle.infer(load_model("cnn"), xs)
    assert int(la.sum()) == kat["cnn_xs_sum_labels_40000"] == 303886


def test_relunorm_probed_vectors(oracle):
    """SURVEY.md 8a row a2, probed against the reference."""
    cases = [([127, 128, 255, 256, -3], [32, 32, 64, 64, 0], 3), ([255, 254, 253, 127, 1], [127, 127, 127, 64, 1], 0),
             ([1000, 509, 510, -1, 1], [125, 64, 64, 0, 0], 0), ([-5, -1, -7], [0, 0, 0], 1), ([5, 9, 9, 2], None, 1),
             ([], [], 255)]
    for x, want, pos in cases:
        out, p = oracle.relunorm(np.array(x, dtype=np.int32))
        assert p == pos
        if want is not None:
            assert out.tolist() == want


def test_decode_tables(oracle):
    """nibble/code -> weight tables of SURVEY.md 8a, through the packed-word decoder."""
    for enc, want in [(M.ENC_4BITSYM, [1, 3, 5, 7, 9, 11, 13, 15, -1, -3, -5, -7, -9, -11, -13, -15]),
                      (M.ENC_4BIT, [0, 1, 2, 3, 4, 5, 6, 7, -8, -7, -6, -5, -4, -3, -2, -1]),
                      (M.ENC_FP130, [1, 2, 4, 8, 16, 32, 64, 128, -1, -2, -4, -8, -16, -32, -64, -128])]:
        codes = np.arange(16, dtype=np.uint32).reshape(1, 16)
        dense = oracle.decode_fc(P.pack_codes(codes, 4), enc, 16, 1)
        assert dense[0].tolist() == want
        assert P.INT_LUT[enc].tolist() == want
    dense = oracle.decode_fc(P.pack_codes(np.tile(np.arange(4, dtype=np.uint32), 4).reshape(1, 16), 2), M.ENC_2BITSYM, 16, 1)
    assert dense[0, :4].tolist() == [1, 3, -1, -3]
    dense = oracle.decode_fc(np.array([0x80000001], dtype=np.uint32), M.ENC_BINARY, 32, 1)
    assert dense[0, 0] == 1 and dense[0, 1] == -1 and dense[0, 31] == 1
    dense = oracle.decode_fc(np.array([0x7F80FF01], dtype=np.uint32), M.ENC_8BIT, 4, 1)
    assert dense[0].tolist() == [127, -128, -1, 1]
    # NF4: zeros in the reference (inference.c:202); LUT only as the documented extension
    w = P.pack_codes(np.arange(16, dtype=np.uint32).reshape(1, 16), 4)
    assert not oracle.decode_fc(w, M.ENC_NF4, 16, 1).any()
    assert oracle.decode_fc(w, M.ENC_NF4, 16, 1, nf4_extension=True)[0].tolist() == P.NF4_INT_LUT.tolist()


def test_ternary_all_words(oracle):
    """Every one of the 65536 raw uint16 words decodes deterministically (0xFFFF -> all 0, 0x0000 -> all +1),
    and all 59049 trit codes round-trip through pack -> decode (SURVEY.md 8c)."""
    words = np.arange(65536, dtype=np.uint16)
    dense = oracle.decode_fc(words, M.ENC_TERNARY, 10, 65536)
    assert np.array_equal(dense, P.unpack_ternary(words, 65536, 10))
    assert not dense[0xFFFF].any() and (dense[0] == 1).all()
    idx = np.arange(59049)
    trits = np.stack([(idx // 3 ** (9 - j)) % 3 for j in range(10)], axis=1) - 1
    packed, n_in = P.pack_ternary(trits)
    assert n_in == 10
    assert np.array_equal(oracle.decode_fc(packed, M.ENC_TERNARY, 10, 59049), trits)


# ---- comparisons with the unmodified reference: its outputs for these seeded inputs were recorded by
# tests/golden/make_reference_vectors.py (tests/golden/reference_vectors.npz); the inputs are regenerated here

@pytest.fixture(scope="module")
def ref_vectors():
    return np.load(os.path.join(GOLDEN, "reference_vectors.npz"))


@pytest.mark.parametrize("enc", RC.FCLAYER_ENCS)
def test_fclayer_vs_reference(oracle, ref_vectors, enc):
    for key, (act, w, e, n_in, n_out) in RC.fclayer_cases([enc]):
        assert np.array_equal(oracle.fclayer(act, w, e, n_in, n_out), ref_vectors["fclayer/" + key])


def test_relunorm_vs_reference(oracle, ref_vectors):
    for key, x in RC.relunorm_cases():
        a, pa = oracle.relunorm(x)
        assert pa == int(ref_vectors["relunorm_pos/" + key]) and np.array_equal(a, ref_vectors["relunorm/" + key])


def test_conv_pool_vs_reference(oracle, ref_vectors):
    for key, (act, w, xy) in RC.conv_pool_cases():
        assert np.array_equal(oracle.conv33relu(act, w, xy, 4), ref_vectors["conv/" + key])
        if xy % 2 == 0:
            assert np.array_equal(oracle.maxpool22(act, xy), ref_vectors["pool/" + key])


@pytest.mark.parametrize("name", RC.WHOLE_MODELS)
def test_whole_model_vs_reference_random(oracle, ref_vectors, name):
    m = load_model(name)
    lo, la = oracle.infer(m, RC.whole_model_images(m))
    assert np.array_equal(lo, ref_vectors["model_logits/" + name]) and np.array_equal(la, ref_vectors["model_labels/" + name])
