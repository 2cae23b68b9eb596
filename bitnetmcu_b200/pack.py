"""Weight packer: the on-disk format either side of the hot path (SURVEY.md 8f rank 2).

Restates the packing half of ``export_to_hfile`` (/root/reference/exportquant.py:86-207) with its
two dtype defects avoided (SURVEY.md 8c):

* Binary and NF4 codes come out of ``np.where`` / ``np.argmin`` as int64; ``<<`` then promotes and
  ``.view(uint32)`` interleaves a zero word after every data word (exportquant.py:105,119,187).
  Here every code array is cast to ``uint32`` before shifting.
* the Ternary size check uses bpw = 1.6 (exportquant.py:97) and rejects first layers such as 256
  inputs; here ternary rows are simply padded to a multiple of 10 with zero trits
  (exportquant.py:132-137) and the padded size is what ``Lk_incoming_weights`` carries (166).

Two domains are used below:
  *levels*  -- the float grid the exporter sees (4bitsym: +-0.5..+-7.5, FP130: +-2^e, ...);
  *integer* -- what the C engine multiplies by (4bitsym: +-1..+-15 odd, ...; inference.c:96-201).
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

from . import model as M

NF4_LEVELS = np.array([-1.0, -0.6962, -0.5251, -0.3949, -0.2844, -0.1848, -0.0911, 0.0,
                       0.0796, 0.1609, 0.2461, 0.3379, 0.4407, 0.5626, 0.723, 1.0])  # exportquant.py:117-118
# integer NF4 extension table (round(127*level)); the reference C engine has no NF4 decode (inference.c:202)
NF4_INT_LUT = np.array([-127, -88, -67, -50, -36, -23, -12, 0, 10, 20, 31, 43, 56, 71, 92, 127], dtype=np.int32)

# code -> integer weight, index = code taken MSB-first (SURVEY.md 8a, probed against the reference)
INT_LUT = {
    M.ENC_BINARY: np.array([-1, 1], dtype=np.int32),
    M.ENC_2BITSYM: np.array([1, 3, -1, -3], dtype=np.int32),
    M.ENC_4BITSYM: np.array([1, 3, 5, 7, 9, 11, 13, 15, -1, -3, -5, -7, -9, -11, -13, -15], dtype=np.int32),
    M.ENC_4BIT: np.array([0, 1, 2, 3, 4, 5, 6, 7, -8, -7, -6, -5, -4, -3, -2, -1], dtype=np.int32),
    M.ENC_FP130: np.array([1, 2, 4, 8, 16, 32, 64, 128, -1, -2, -4, -8, -16, -32, -64, -128], dtype=np.int32),
    M.ENC_8BIT: np.concatenate([np.arange(0, 128), np.arange(-128, 0)]).astype(np.int32),
    M.ENC_NF4: NF4_INT_LUT,
}
CODE_BITS = {M.ENC_BINARY: 1, M.ENC_2BITSYM: 2, M.ENC_4BITSYM: 4, M.ENC_4BIT: 4, M.ENC_FP130: 4, M.ENC_NF4: 4,
             M.ENC_8BIT: 8}
QUANT_IDS = {"Binary": M.ENC_BINARY, "2bitsym": M.ENC_2BITSYM, "4bitsym": M.ENC_4BITSYM, "4bit": M.ENC_4BIT,
             "NF4": M.ENC_NF4, "8bit": M.ENC_8BIT, "FP130": M.ENC_FP130, "Ternary": M.ENC_TERNARY}


def encode_levels(quant_type: str, w: np.ndarray) -> np.ndarray:
    """Quantised weight *levels* -> codes (exportquant.py:104-126), always uint32."""
    w = np.asarray(w)
    if quant_type == "Binary":
        return np.where(w == -1, 0, 1).astype(np.uint32)
    if quant_type == "2bitsym":
        return ((w < 0).astype(np.uint32) << 1) | np.floor(np.abs(w)).astype(np.uint32)
    if quant_type == "4bitsym":
        return ((w < 0).astype(np.uint32) << 3) | np.floor(np.abs(w)).astype(np.uint32)
    if quant_type == "4bit":
        return np.floor(w).astype(np.int64).astype(np.uint32) & 15
    if quant_type == "NF4":
        return np.argmin(np.abs(w[..., np.newaxis] - NF4_LEVELS), axis=-1).astype(np.uint32)
    if quant_type == "8bit":
        return np.floor(w).astype(np.int64).astype(np.uint32) & 255
    if quant_type == "FP130":
        return ((w < 0).astype(np.uint32) << 3) | np.floor(np.log2(np.abs(w))).astype(np.uint32)
    raise ValueError(f"unsupported quantisation type {quant_type}")


def codes_from_int_weights(enc: int, w_int: np.ndarray) -> np.ndarray:
    """Engine-domain integer weights -> codes (inverse of INT_LUT); raises if a value is not representable."""
    lut = INT_LUT[enc]
    w_int = np.asarray(w_int, dtype=np.int64)
    order = np.argsort(lut)
    pos = np.searchsorted(lut[order], w_int)
    pos = np.clip(pos, 0, lut.size - 1)
    if not np.array_equal(lut[order][pos], w_int):
        raise ValueError(f"weights not representable in encoding {M.ENC_NAMES[enc]}")
    return order[pos].astype(np.uint32)


def pack_codes(codes: np.ndarray, bits: int) -> np.ndarray:
    """[n_out, n_in] codes -> uint32 words, first weight in the MSBs (exportquant.py:182-187).
    Rows must fill whole words: bits*n_in % 32 == 0 (exportquant.py:97)."""
    codes = np.asarray(codes, dtype=np.uint32)
    n_out, n_in = codes.shape
    if (bits * n_in) % 32:
        raise ValueError(f"incoming weights must pack to a 32-bit boundary: {n_in} x {bits} bits")
    per = 32 // bits
    c = codes.reshape(n_out, n_in // per, per)
    shifts = (32 - bits - np.arange(per, dtype=np.uint32) * bits).astype(np.uint32)
    return np.bitwise_or.reduce(c << shifts, axis=2).astype(np.uint32).reshape(-1)


def unpack_codes(words: np.ndarray, bits: int, n_out: int, n_in: int) -> np.ndarray:
    per = 32 // bits
    w = np.asarray(words, dtype=np.uint32).reshape(n_out, n_in // per, 1)
    shifts = (32 - bits - np.arange(per, dtype=np.uint32) * bits).astype(np.uint32)
    return ((w >> shifts) & np.uint32((1 << bits) - 1)).reshape(n_out, n_in)


def pack_ternary(trits: np.ndarray):
    """[n_out, n_in] in {-1,0,+1} -> (uint16 words [n_out * n_in_padded/10], n_in_padded).
    exportquant.py:127-157: trit +1 -> 0, -1 -> 1, 0 -> 2; base-3 MSB-first; ceil-scale to 16 bits."""
    t = np.asarray(trits, dtype=np.int64)
    n_out, n_in = t.shape
    pad = (-n_in) % 10
    if pad:
        t = np.pad(t, ((0, 0), (0, pad)))
    digits = np.where(t == 1, 0, np.where(t == -1, 1, 2)).astype(np.int64).reshape(n_out, -1, 10)
    value = np.zeros(digits.shape[:2], dtype=np.int64)
    for j in range(10):
        value = value * 3 + digits[:, :, j]
    packed = (value * 65536 + 59048) // 59049
    return packed.astype(np.uint16).reshape(-1), n_in + pad


def unpack_ternary(words: np.ndarray, n_out: int, n_in: int) -> np.ndarray:
    """uint16 words -> trits, by the engine's repeated *3 extraction (inference.c:116-136)."""
    c = np.asarray(words, dtype=np.uint32).reshape(n_out, n_in // 10).astype(np.uint64)
    out = np.zeros((n_out, n_in // 10, 10), dtype=np.int32)
    for j in range(10):
        c = c * 3
        out[:, :, j] = np.where(c & 0x20000, 0, np.where(c & 0x10000, -1, 1))
        c = c & 0xFFFF
    return out.reshape(n_out, n_in)


def decode_int_weights(layer: M.Layer, nf4_extension: bool = False) -> np.ndarray:
    """Packed FC layer -> dense engine-domain integer weights [n_out, n_in] (numpy restatement of the decode)."""
    enc = layer.bitperweight
    if enc == M.ENC_TERNARY:
        return unpack_ternary(layer.weights[: layer.n_out * (layer.n_in // 10)], layer.n_out, layer.n_in)
    if enc not in CODE_BITS or (enc == M.ENC_NF4 and not nf4_extension):
        return np.zeros((layer.n_out, layer.n_in), dtype=np.int32)
    bits = CODE_BITS[enc]
    codes = unpack_codes(layer.weights[: layer.n_out * layer.n_in * bits // 32], bits, layer.n_out, layer.n_in)
    return INT_LUT[enc][codes]


def fc_layer_from_codes(name: str, enc: int, codes: np.ndarray) -> M.Layer:
    n_out, n_in = codes.shape
    return M.Layer(kind=M.LAYER_FC, name=name, bitperweight=enc, n_in=n_in, n_out=n_out,
                   weights=pack_codes(codes, CODE_BITS[enc]))


def fc_layer_from_trits(name: str, trits: np.ndarray) -> M.Layer:
    words, n_in_padded = pack_ternary(trits)
    return M.Layer(kind=M.LAYER_FC, name=name, bitperweight=M.ENC_TERNARY, n_in=n_in_padded, n_out=trits.shape[0],
                   weights=words)


def fc_layer_from_levels(name: str, quant_type: str, levels: np.ndarray) -> M.Layer:
    """What export_to_hfile does for one BitLinear layer (exportquant.py:88-207)."""
    if quant_type == "Ternary":
        return fc_layer_from_trits(name, np.asarray(levels))
    return fc_layer_from_codes(name, QUANT_IDS[quant_type], encode_levels(quant_type, levels))


def random_fc_model(enc: int, widths: Sequence[int] = (256, 64, 64, 64, 10), seed: int = 0) -> M.Model:
    """FC model with uniformly random codes: every bit pattern is a legal weight in every encoding
    (SURVEY.md 8d, config 5), so this exercises the full decode tables."""
    rng = np.random.default_rng(seed)
    layers: List[M.Layer] = []
    for i in range(len(widths) - 1):
        n_in, n_out = widths[i], widths[i + 1]
        if enc == M.ENC_TERNARY:
            layers.append(fc_layer_from_trits(f"L{i + 1}", rng.integers(-1, 2, size=(n_out, n_in))))
        else:
            codes = rng.integers(0, 1 << CODE_BITS[enc], size=(n_out, n_in), dtype=np.uint32)
            layers.append(fc_layer_from_codes(f"L{i + 1}", enc, codes))
    m = M.Model(model_class=M.MODEL_FCMNIST, layers=layers, img_bytes=widths[0], source=f"random:{M.ENC_NAMES[enc]}:{seed}")
    m.validate()
    return m


def max_n_activations(model: M.Model) -> int:
    """MAX_N_ACTIVATIONS of a header: the size of BitMnistInference's stack buffers (BitNetMCU_MNIST_dll.c:49-50,96-97).
    The exporter writes the widest layer input (exportquant.py:64), but the driver also keeps each layer's outputs there and,
    for CNN models, uses the int32 buffer as 16x16 scratch and the int8 one as the channels x 4 int32 features: fewer than
    256 would overflow the stack of a 16-channel model."""
    fc = model.fc_layers
    return max([256, model.channels * 4] + [l.n_in for l in fc] + [l.n_out for l in fc])


def write_header(model: M.Model, path: str, runname: str = "bitnetmcu_b200") -> None:
    """Emit a reference-compatible ``BitNetMCU_model.h`` (exportquant.py:68-84,164-259)."""
    cls = "CNNMNIST" if model.model_class == M.MODEL_CNNMNIST else "FCMNIST"
    out = ["// Automatically generated header file", f"// Quantized model exported from {runname}",
           "// Generated by bitnetmcu_b200.pack.write_header (layout of exportquant.py)", "", "#include <stdint.h>", "",
           "#ifndef BITNETMCU_MODEL_H", "#define BITNETMCU_MODEL_H", "", f"#define MODEL_{cls}", "",
           f"#define NUM_LAYERS {len(model.layers)}", "",
           f"#define MAX_N_ACTIVATIONS {max_n_activations(model)}", ""]
    for l in model.layers:
        n = l.name
        if l.kind == M.LAYER_FC:
            tern = l.bitperweight == M.ENC_TERNARY
            out += [f"// Layer: {n}", f"// QuantType: {M.ENC_NAMES.get(l.bitperweight, '?')}", f"#define {n}_active",
                    f"#define {n}_bitperweight {l.bitperweight}", f"#define {n}_incoming_weights {l.n_in}",
                    f"#define {n}_outgoing_weights {l.n_out}"]
            per, fmt = (10, "0x%04x,") if tern else (8, "0x%08x,")
            out.append(f"const {'uint16_t' if tern else 'uint32_t'} {n}_weights[] = {{")
            w = l.weights.reshape(-1)
            out += ["\t" + "".join(fmt % int(v) for v in w[i:i + per]) for i in range(0, w.size, per)]
            out += ["};", ""]
        elif l.kind == M.LAYER_CONV33:
            out += [f"// Layer: {n} (Convolutional)", f"#define {n}_active", f"#define {n}_type BitConv2d",
                    f"#define {n}_in_channels {l.in_channels}", f"#define {n}_out_channels {l.n_out}",
                    f"#define {n}_incoming_x {l.n_in}", f"#define {n}_incoming_y {l.n_in}",
                    f"#define {n}_outgoing_x {l.n_in - 2}", f"#define {n}_outgoing_y {l.n_in - 2}",
                    f"#define {n}_kernel_size 3", f"#define {n}_stride 1", f"#define {n}_padding 0",
                    f"#define {n}_groups {l.groups}", f"#define {n}_bitperweight {l.bitperweight}",
                    f"const int8_t {n}_weights[] = {{"]
            w = l.weights.reshape(-1)
            out += ["\t" + "".join("%d," % int(v) for v in w[i:i + 16]) for i in range(0, w.size, 16)]
            out += ["};", ""]
        else:
            out += [f"#define {n}_active", f"#define {n}_type MaxPool2d", f"#define {n}_pool_size 2",
                    f"#define {n}_incoming_x {l.n_in}", f"#define {n}_incoming_y {l.n_in}",
                    f"#define {n}_outgoing_x {l.n_in // 2}", f"#define {n}_outgoing_y {l.n_in // 2}", ""]
    out += ["#endif", ""]
    with open(path, "w") as f:
        f.write("\n".join(out))
