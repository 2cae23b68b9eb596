"""The models the reference's own BitNetMCU_MNIST_dll.c is built for, once with the reference kernels and once with the
library's reference-named symbols (oracle/Makefile, target `dropin`), and their BitNetMCU_model.h headers (TEST
INFRASTRUCTURE).

    python dropin_headers.py --list               the model names, one line
    python dropin_headers.py <model> <path>       write <model>'s header to <path>

dll.c hard-codes its layer names (L1..L3 and an optional L4 for FC models, L2..L15 for CNN models), so only the fixtures
whose layers carry those names are listed.  A Ternary layer declares its inputs padded to a multiple of 10, and dll.c hands
it the previous layer's n_out bytes of an uninitialised stack buffer (or the caller's 256-byte image): a non-zero trit
past that width reads undefined bytes, and such a model is left out (reads_past_its_input)."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FC_MODELS = ["fc", "12k", "12k_FP130", "1k", "2bitsym96", "4bit64", "8bit64", "binary160", "ternary64", "rand_8bit64",
             "rand_binary64", "rand_fp130_64", "rand_nf4_64", "rand_ternary64"]
CNN_MODELS = ["cnn", "cnn_16", "cnn_16small", "cnn_32", "cnn_48", "cnn_letters"]


def load(name):
    from bitnetmcu_b200.model import Model
    return Model.load(os.path.join(ROOT, "tests", "golden", "models", name + ".bnm"))


def reads_past_its_input(model):
    """whether a Ternary layer has a non-zero trit at a column past the bytes dll.c defines for it: the image's img_bytes for
    the first FC layer of an FC model, the previous FC layer's n_out for every later one"""
    from bitnetmcu_b200 import model as M, pack as P
    width = model.img_bytes if model.model_class == M.MODEL_FCMNIST else None
    for l in model.fc_layers:
        if l.bitperweight == M.ENC_TERNARY and width is not None and width < l.n_in:
            trits = P.unpack_ternary(l.weights[: l.n_out * (l.n_in // 10)], l.n_out, l.n_in)
            if trits[:, width:].any():
                return True
        width = l.n_out
    return False


def dll_models():
    """the fixtures dll.c is built for: every listed model but those whose Ternary pad trits it would read undefined"""
    return [n for n in FC_MODELS + CNN_MODELS if not reads_past_its_input(load(n))]


def main(argv):
    if argv[1:] == ["--list"]:
        print(" ".join(dll_models()))
        return 0
    if len(argv) != 3 or argv[1] not in dll_models():
        print(__doc__, file=sys.stderr)
        return 2
    from bitnetmcu_b200.pack import write_header
    os.makedirs(os.path.dirname(os.path.abspath(argv[2])), exist_ok=True)
    write_header(load(argv[1]), argv[2])
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
