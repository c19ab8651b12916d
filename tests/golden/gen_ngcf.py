"""Golden vectors for NGCF propagation from the UNMODIFIED reference module
(libreco/algorithms/torch_modules/ngcf_module.py) on CPU.

    python tests/golden/gen_ngcf.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402

load_reference()
import torch  # noqa: E402
from libreco.algorithms.torch_modules.ngcf_module import NGCFModel  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def case(seed, n_users, n_items, d, layers, mean_deg, name, head_users=0):
    """``head_users > 0``: those users also consume item 0 and nobody consumes item n_items - 1, so
    the graph has a row above the SpMM's long-row threshold and an item with only its self loop."""
    rng = np.random.default_rng(seed)
    consumed = {}
    w = 1.0 / np.arange(1, n_items + 1)
    w /= w.sum()
    for u in range(n_users):
        c = max(1, int(min(rng.poisson(mean_deg), n_items)))
        items = rng.choice(n_items, size=c, replace=False, p=w).tolist()
        if c > 3:
            items.append(items[0])
        if head_users:
            items = [i for i in items if i != n_items - 1]
            if u < head_users:
                items.append(0)
        consumed[u] = items
    consumed[n_users - 1] = []               # isolated user: only its self loop
    torch.manual_seed(seed)
    m = NGCFModel(n_users, n_items, d, list(layers), 0.0, 0.0, consumed, torch.device("cpu"))
    with torch.no_grad():
        for k in range(len(layers)):         # non-zero biases so that they are exercised
            m.weight_dict[f"b_self_{k}"].normal_(0, 0.05)
            m.weight_dict[f"b_pair_{k}"].normal_(0, 0.05)
        ue, ie = m.embedding_propagation(use_dropout=False)
    lap = m.laplacian_matrix.coalesce()
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    for u in range(n_users):
        indptr[u + 1] = indptr[u] + len(consumed[u])
    idx = np.concatenate([np.asarray(consumed[u], dtype=np.int32) for u in range(n_users)])
    data = dict(n_users=n_users, n_items=n_items, indptr=indptr, idx=idx,
                user_embed=m.embedding_dict["user_embed"].detach().numpy(),
                item_embed=m.embedding_dict["item_embed"].detach().numpy(),
                user_out=ue.numpy(), item_out=ie.numpy(), lap_row=lap.indices()[0].numpy(),
                lap_col=lap.indices()[1].numpy(), lap_val=lap.values().numpy())
    for k, v in m.weight_dict.items():
        data[k] = v.detach().numpy()
    np.savez_compressed(os.path.join(OUT, f"ngcf_{name}.npz"), **data)
    print(name, ue.shape, ie.shape, lap._nnz())


CASES = {
    "d16": lambda: case(41, 120, 90, 16, (16, 16, 16), 7, "d16"),
    "d64": lambda: case(42, 80, 150, 64, (64, 32), 12, "d64"),
    # layer-input widths 10 / 24 / 36 / 132 cover the scalar (lpr 16), vec4 (LPR 8, 16) and scalar T = 5
    # SpMM paths; the head item's row (over 1 024 users + self loop) takes the long-row chunk kernels
    "d10": lambda: case(43, 1200, 150, 10, (24, 7), 4, "d10", head_users=1100),
    "d36": lambda: case(44, 1060, 60, 36, (132, 20), 4, "d36", head_users=1040),
}

if __name__ == "__main__":
    for key in sys.argv[1:] or CASES:
        CASES[key]()
