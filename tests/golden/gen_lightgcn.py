"""Golden vectors for LightGCN propagation from the UNMODIFIED reference module
(libreco/algorithms/torch_modules/lightgcn_module.py) on CPU.

    python tests/golden/gen_lightgcn.py              # every case
    python tests/golden/gen_lightgcn.py drop_d16     # only the named cases

``lightgcn_drop_*.npz`` run ``forward(use_dropout=True)`` (edge dropout, :90-96) and its backward:
they store the reference's own ``torch.rand`` draw as the mask, the Laplacian COO in the order the
mask indexes it, both outputs, a fixed upstream weight ``W`` and the init-embedding gradients of
``(cat(user_out, item_out) * W).sum()``.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402

load_reference()
import torch  # noqa: E402
from libreco.algorithms.torch_modules.lightgcn_module import LightGCNModel  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def case(seed, n_users, n_items, d, n_layers, mean_deg, name):
    rng = np.random.default_rng(seed)
    consumed = {}
    w = 1.0 / np.arange(1, n_items + 1)
    w /= w.sum()
    for u in range(n_users):
        c = max(1, int(min(rng.poisson(mean_deg), n_items)))
        items = rng.choice(n_items, size=c, replace=False, p=w).tolist()
        if c > 3:
            items.append(items[0])           # duplicates collapse to one edge
        consumed[u] = items
    consumed[n_users - 1] = []               # isolated user -> zero row
    torch.manual_seed(seed)
    m = LightGCNModel(n_users, n_items, d, n_layers, 0.0, consumed, torch.device("cpu"))
    with torch.no_grad():
        ue, ie = m.embedding_propagation(use_dropout=False)
    lap = m.laplacian_matrix.coalesce()
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    for u in range(n_users):
        indptr[u + 1] = indptr[u] + len(consumed[u])
    idx = np.concatenate([np.asarray(consumed[u], dtype=np.int32) for u in range(n_users)])
    np.savez_compressed(
        os.path.join(OUT, f"lightgcn_{name}.npz"), n_users=n_users, n_items=n_items, n_layers=n_layers,
        indptr=indptr, idx=idx,
        user_init=m.user_init_embeds.weight.detach().numpy(), item_init=m.item_init_embeds.weight.detach().numpy(),
        user_out=ue.numpy(), item_out=ie.numpy(),
        lap_row=lap.indices()[0].numpy(), lap_col=lap.indices()[1].numpy(), lap_val=lap.values().numpy())
    print(name, ue.shape, ie.shape, lap._nnz())


def drop_case(seed, n_users, n_items, d, n_layers, dropout, mean_deg, name):
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, n_items + 1) ** 1.2        # Zipf popularity: the head item's row is long
    w /= w.sum()
    consumed = {}
    for u in range(n_users):
        c = max(1, int(min(rng.poisson(mean_deg), n_items - 1)))
        consumed[u] = rng.choice(n_items - 1, size=c, replace=False, p=w[:-1] / w[:-1].sum()).tolist()
    consumed[n_users - 1] = []               # isolated user; item n_items - 1 is never consumed
    head = sum(0 in v for v in consumed.values())
    assert head > 1024, head                 # the head item's Laplacian row takes the chunked path
    torch.manual_seed(seed)
    m = LightGCNModel(n_users, n_items, d, n_layers, dropout, consumed, torch.device("cpu"))
    lap = m.laplacian_matrix                 # uncoalesced: the order sparse_dropout's mask indexes
    draws = []
    rand = torch.rand

    def recording_rand(*a, **k):
        r = rand(*a, **k)
        draws.append(r.clone())
        return r

    torch.rand = recording_rand
    try:
        torch.manual_seed(seed)
        ue, ie = m.forward(use_dropout=True)
    finally:
        torch.rand = rand
    assert len(draws) == 1 and draws[0].numel() == lap._nnz()
    mask = torch.floor(draws[0] + (1 - dropout)).bool()
    W = torch.from_numpy(np.random.default_rng(seed + 1).standard_normal((n_users + n_items, d)).astype(np.float32))
    (torch.cat([ue, ie]) * W).sum().backward()
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    for u in range(n_users):
        indptr[u + 1] = indptr[u] + len(consumed[u])
    idx = np.concatenate([np.asarray(consumed[u], dtype=np.int32) for u in range(n_users)])
    np.savez_compressed(
        os.path.join(OUT, f"lightgcn_{name}.npz"), n_users=n_users, n_items=n_items, n_layers=n_layers,
        dropout=dropout, seed=seed, nnz=lap._nnz(), indptr=indptr, idx=idx,
        user_init=m.user_init_embeds.weight.detach().numpy(), item_init=m.item_init_embeds.weight.detach().numpy(),
        user_out=ue.detach().numpy(), item_out=ie.detach().numpy(),
        lap_row=lap._indices()[0].numpy(), lap_col=lap._indices()[1].numpy(), lap_val=lap._values().numpy(),
        mask=mask.numpy(), W=W.numpy(),
        user_grad=m.user_init_embeds.weight.grad.numpy(), item_grad=m.item_init_embeds.weight.grad.numpy())
    print(name, ue.shape, ie.shape, lap._nnz(), "head degree", head, "kept", int(mask.sum()))


CASES = {
    "d16": lambda: case(31, 200, 120, 16, 3, 8, "d16"),
    "d64": lambda: case(32, 150, 400, 64, 2, 15, "d64"),
    "d10": lambda: case(33, 60, 50, 10, 4, 5, "d10"),
    "drop_d16": lambda: drop_case(34, 1300, 400, 16, 3, 0.3, 12, "drop_d16"),
    "drop_d10": lambda: drop_case(35, 1300, 300, 10, 2, 0.5, 10, "drop_d10"),
}

if __name__ == "__main__":
    for key in sys.argv[1:] or CASES:
        CASES[key]()
