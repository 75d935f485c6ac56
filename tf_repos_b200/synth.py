"""Synthetic Criteo-39-field batches in the id layout `get_criteo_feature.py:116-167` produces:
one global id space; fields 0..12 are the continuous features with id = f+1 and a min-max scaled
value; fields 13..38 are categoricals with val = 1 and id = offset_f + index, the 26 sub-vocabularies
partitioning [14, N).  (SURVEY.md 8d; also reproduces the row-13 collision quirk Q7 when
`collide=True`: C1's <unk> shares id 13 with I13.)"""
from __future__ import annotations

import numpy as np
import torch

N_CONT, N_CAT = 13, 26


def field_offsets(N: int, n_fields: int = N_CONT + N_CAT):
    n_cat = n_fields - N_CONT
    lo = N_CONT + 1
    edges = np.linspace(lo, N, n_cat + 1).astype(np.int64)
    return edges[:-1], np.maximum(edges[1:] - edges[:-1], 1)


def criteo_batch(B: int, N: int, F: int = 39, seed: int = 0, device="cpu", zipf: float = 0.0):
    """returns ids int32 [B,F], vals f32 [B,F], labels f32 [B]"""
    assert F > N_CONT, "layout needs the 13 continuous fields"
    g = torch.Generator(device="cpu").manual_seed(seed)
    off, size = field_offsets(N, F)
    ids = torch.empty(B, F, dtype=torch.int64)
    vals = torch.ones(B, F, dtype=torch.float32)
    ids[:, :N_CONT] = torch.arange(1, N_CONT + 1)
    vals[:, :N_CONT] = torch.round(torch.rand(B, N_CONT, generator=g) * 1e6) / 1e6
    u = torch.rand(B, F - N_CONT, generator=g, dtype=torch.float64)
    if zipf > 0.0:  # heavy-tailed index inside each sub-vocabulary
        u = u ** (1.0 + 4.0 * zipf)
    idx = (u * torch.from_numpy(size).to(torch.float64)).floor().to(torch.int64)
    idx = torch.minimum(idx, torch.from_numpy(size - 1))
    ids[:, N_CONT:] = torch.from_numpy(off) + idx
    ids.clamp_(0, N - 1)
    labels = (torch.rand(B, generator=g) < 0.25).to(torch.float32)
    return ids.to(torch.int32).to(device), vals.to(device), labels.to(device)


def write_libsvm(path: str, ids, vals, labels):
    """`<label> <id>:<val> ...` with single spaces (DeepFM.py:62,69-75)."""
    ids, vals, labels = ids.cpu().numpy(), vals.cpu().numpy(), labels.cpu().numpy()
    with open(path, "w") as fo:
        for b in range(ids.shape[0]):
            toks = ["%d" % int(labels[b])]
            toks += ["%d:%s" % (int(i), ("%.6f" % v).rstrip("0").rstrip(".") if v != 1.0 else "1")
                     for i, v in zip(ids[b], vals[b])]
            fo.write(" ".join(toks) + "\n")


def din_batch(B: int, N: int, Fp: int = 11, P: int = 100, max_a_int: int = 8, seed: int = 0, device="cpu",
              fixed_len: bool = False):
    """Synthetic DIN batch with the feature names/shapes of DIN.py:60-77 (Ali-CCP layout): ids uniform in
    [1, N) (0 = padding sentinel), behaviour lengths ~ U{1..P} (or all P), weights ~ U(0,3), a_int bags of
    1..max_a_int ids; label ~ Bernoulli(0.25).  (SURVEY.md 8d)"""
    g = torch.Generator().manual_seed(seed)
    ri = lambda *shape: torch.randint(1, N, shape, generator=g, dtype=torch.int64).to(torch.int32)
    feat_ids = ri(B, Fp)
    a_ids = ri(3, B)
    lens_a = torch.randint(1, max_a_int + 1, (B,), generator=g)
    a_off = torch.zeros(B + 1, dtype=torch.int32)
    a_off[1:] = torch.cumsum(lens_a, 0).to(torch.int32)
    a_int_ids = ri(int(a_off[-1]))
    u_ids = ri(4, B, P)
    u_wgt = torch.rand(4, B, P, generator=g) * 3.0
    if not fixed_len:
        lens = torch.randint(1, P + 1, (4, B), generator=g)
        pad = torch.arange(P).view(1, 1, P) >= lens.unsqueeze(-1)
        u_ids[pad] = 0
        u_wgt[pad] = 0.0
    labels = (torch.rand(B, generator=g) < 0.25).float()
    batch = {"feat_ids": feat_ids, "a_ids": a_ids, "a_int_ids": a_int_ids, "a_int_off": a_off,
             "u_ids": u_ids, "u_wgt": u_wgt}
    return {k: v.to(device) for k, v in batch.items()}, labels.to(device)


def esmm_batch(B: int, N: int, Fp: int = 11, max_lens=(49, 499, 49, 49, 8), min_len: int = 1, seed: int = 0,
               device="cpu"):
    """Synthetic ESMM batch (DeepCvrMTL.py:66-83, Ali-CCP layout) in the CSR form of tf_repos_b200.esmm: ids uniform in
    [0, N) (id 0 is an ordinary id), bag j of each sample ~ U{min_len..max_lens[j]} ids (j = u_cat, u_shop, u_brand,
    u_int, a_int), weights ~ U(0,3); y ~ Bernoulli(0.25), z = y * Bernoulli(0.3) (a conversion follows a click).
    Returns (batch, (y, z))."""
    g = torch.Generator().manual_seed(seed)
    ri = lambda *shape: torch.randint(0, N, shape, generator=g, dtype=torch.int64).to(torch.int32)
    feat_ids = ri(B, Fp)
    a_ids = ri(3, B)
    lens = torch.stack([torch.randint(min_len, m + 1, (B,), generator=g) for m in max_lens])     # [5, B]
    off = torch.zeros(5 * B + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(lens.reshape(-1), 0).to(torch.int32)
    nnz = int(off[-1])
    bag_ids = ri(nnz)
    bag_wgt = torch.rand(nnz, generator=g) * 3.0
    y = (torch.rand(B, generator=g) < 0.25).float()
    z = y * (torch.rand(B, generator=g) < 0.3).float()
    batch = {"feat_ids": feat_ids, "a_ids": a_ids, "bag_ids": bag_ids, "bag_wgt": bag_wgt, "bag_off": off}
    return {k: v.to(device) for k, v in batch.items()}, (y.to(device), z.to(device))
