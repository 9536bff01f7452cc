"""The reference's few-shot occupancy evaluation (datasets/metrics.py:180-472 of NVlabs/EmerNeRF@8c051d7), restated
op for op as its formulation runs on the GPU -- TEST INFRASTRUCTURE ONLY, the baseline of tools/bench_occupancy.py.

Per frame: a density pass, the ``density > 0.2`` filter by boolean indexing, a second pass with the feature head over
the kept voxels; centroids as per-class means of the concatenated kept features of every train frame; classification
by the cosine kNN with k = 1 (fp32 normalisation, a similarity matrix, ``topk``, the temperature-weighted one-hot
scores and their ``argsort``) and per-class counts read back with ``.item()``.  The progress bars are left out.
"""
from __future__ import annotations

import torch


def _forward(model, coords, t, features):
    with torch.no_grad():
        return model.forward(positions=coords, data_dict={"normed_timestamps": t}, combine_static_dynamic=True,
                             query_feature_head=features, query_pe_head=False)


def _kept(dataset, index, model, device):
    coords, labels, t = (x.to(device) for x in dataset.get_occ(index))
    keep = (_forward(model, coords, t, False)["density"] > 0.2).squeeze()
    return coords, labels, t, keep


def collect_centroids(train_indices, dataset, model, device):
    feats, labels_all = [], []
    for i in train_indices:
        coords, labels, t, keep = _kept(dataset, i, model, device)
        labels, coords, t = labels[keep], coords[keep], t[keep]
        feats.append(_forward(model, coords, t, True)["dino_feat"])
        labels_all.append(labels)
    feats, labels_all = torch.cat(feats, 0), torch.cat(labels_all, 0)
    means = {int(c): feats[labels_all == c].mean(dim=0, keepdim=True) for c in torch.unique(labels_all)}
    k = len(dataset.label_mapping)
    bank = torch.cat([means.get(j, torch.zeros(1, 64, device=device)) for j in range(k)], 0)
    return bank, torch.tensor(list(range(k))).to(device)


def knn_top1(queries, centroids, labels, n_classes, temperature=0.1):
    """The reference's knn_predict(..., knn_k=1, similarity="cosine")[..., 0]."""
    bank = centroids / (centroids.norm(dim=-1, keepdim=True) + 1e-7)
    sim = torch.mm(queries / (queries.norm(dim=-1, keepdim=True) + 1e-7), bank.T)
    w, idx = sim.topk(k=1, dim=-1)
    picked = torch.gather(labels.expand(queries.size(0), -1), dim=-1, index=idx)
    one_hot = torch.zeros(queries.size(0), n_classes, device=picked.device).scatter(-1, picked.view(-1, 1), 1.0)
    scores = (one_hot.view(queries.size(0), -1, n_classes) * (w / temperature).exp().unsqueeze(-1)).sum(1)
    return scores.argsort(dim=-1, descending=True)[..., 0]


def eval_few_shot_occ(test_indices, dataset, model, device, centroids_bank, label_bank):
    mapping = dataset.label_mapping
    correct_all = total_all = measured = total_points = 0
    correct_per = {c: 0 for c in mapping}
    total_per = {c: 0 for c in mapping}
    accs = non_zero = 0
    for i in test_indices:
        coords, labels, t, keep = _kept(dataset, i, model, device)
        total_points += len(labels)
        if keep.sum() == 0:
            continue
        coords, labels, t = coords[keep], labels[keep], t[keep]
        measured += len(labels)
        pred = knn_top1(_forward(model, coords, t, True)["dino_feat"], centroids_bank, label_bank, len(mapping))
        correct = pred == labels
        present, counts = torch.unique(labels, return_counts=True)
        total_per.update({c.item(): total_per[c.item()] + n.item() for c, n in zip(present, counts)})
        per_class = torch.bincount(labels[correct].long())
        correct_per.update({c.item(): correct_per[c.item()] + per_class[c.long()].item()
                            for c in present if c < len(per_class)})
        correct_all += correct.sum().item()
        total_all += len(labels)
        accs = non_zero = 0
        for c in mapping:
            if total_per[c]:
                accs += correct_per[c] / total_per[c]
                non_zero += 1
    return {
        "micro_accuracy": correct_all / total_all,
        "macro_accuracy": accs / non_zero,
        "per_class_accuracy": {name: correct_per[c] / (total_per[c] + 1e-10) for c, name in mapping.items()},
        "cover_rate": measured / total_points,
        "num_measured_points": measured,
        "num_total_points": total_points,
    }
