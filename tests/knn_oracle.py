"""float64 numpy restatement of the k-NN selection order and vote of csrc/knn.cu (the GPU tests compare against it).

Selection: entries rank by similarity descending, then bank index ascending (a total order), so the k best of a row
are the first k entries of that sort.  Vote: neighbour weight w = exp(s / T) with the quotient s / T rounded to fp32
as the kernel computes it; a class's score is the sum of its neighbours' weights; classes rank by score descending,
then class index ascending."""
import numpy as np


def topk(sim, k, n0=0):
    """Per row of sim [Q, N] (similarity of bank row n0 + j in column j): (values [Q, m], indices [Q, m]) of the
    m = min(k, N) best entries, best first."""
    sim = np.asarray(sim)
    q, n = sim.shape
    m = min(k, n)
    cols = np.arange(n)
    vals = np.empty((q, m), dtype=sim.dtype)
    idx = np.empty((q, m), dtype=np.int64)
    for r in range(q):
        order = np.lexsort((cols, -sim[r].astype(np.float64)))[:m]   # last key is primary
        vals[r] = sim[r, order]
        idx[r] = order + n0
    return vals, idx


def weights(vals, temperature):
    """exp(s / T) in float64 of the fp32 quotient s / T."""
    q32 = np.asarray(vals, dtype=np.float32) / np.float32(temperature)
    return np.exp(q32.astype(np.float64))


def class_scores(vals, idx, bank_labels, num_classes, temperature):
    """float64 [Q, num_classes]: per class the sum of its neighbours' weights, in rank order (index -1: empty)."""
    vals, idx = np.asarray(vals), np.asarray(idx)
    labels = np.asarray(bank_labels)
    w = weights(vals, temperature)
    scores = np.zeros((vals.shape[0], num_classes), dtype=np.float64)
    for r in range(vals.shape[0]):
        for j in range(vals.shape[1]):
            if idx[r, j] >= 0:
                scores[r, labels[idx[r, j]]] += w[r, j]
    return scores


def rank_classes(scores, top=5):
    """int [Q, min(top, C)]: classes by score descending, then class index ascending."""
    scores = np.asarray(scores, dtype=np.float64)
    q, c = scores.shape
    classes = np.arange(c)
    return np.stack([np.lexsort((classes, -scores[r]))[:min(top, c)] for r in range(q)])


def classify(sim, bank_labels, num_classes, k, temperature):
    """Top-5 classes of each row of the full similarity matrix (the whole k-NN classifier in float64)."""
    vals, idx = topk(sim, k)
    return rank_classes(class_scores(vals, idx, bank_labels, num_classes, temperature))
