"""TEST INFRASTRUCTURE ONLY -- numpy restatement of the random-forest regressor RandomForestEIChooser fits and queries
(RF = chooser/RandomForestEIChooser.py): scikit-learn 1.9's DepthFirstTreeBuilder + BestSplitter + MSE criterion on
one bootstrap-weighted tree, and the per-tree predict, mean and ddof=1 variance of RF:16-26.

No sklearn import, so GPU tests and ``smoke()`` can check the device forest against it.  The builder is written for
clarity; every floating-point value is formed by the same sequence of double operations as sklearn's, which decides
ties between candidate splits (tests/test_rf_oracle.py compares the trees with sklearn's own ``tree_`` arrays):

  * X is float32, y and the sample weights (bootstrap counts) float64; only samples of non-zero weight take part.
  * node order: depth-first, pop a node, push the right then the left child; one rand_r state per tree is consumed in
    that order by the Fisher-Yates feature draw over the ``features`` / ``constant_features`` arrays, which persist
    across nodes.
  * a feature is constant in a node when max <= min + 1e-7 in float32; split positions between values within 1e-7
    (float32) are skipped; the threshold is x[p-1]/2 + x[p]/2 in double.
  * sum_total / sq_sum_total accumulate over samples[start:end] in array order; sum_left accumulates in sorted order,
    from whichever end (pos or end) is nearer, as RegressionCriterion.update does.
  * the best split is the first strictly greater proxy sl^2/wl + sr^2/wr in draw order, then position order.
  * samples[start:end] is left sorted by the last feature that was sorted (a constant one included), then swap-
    partitioned; the children inherit that order.  Equal keys are ordered by sample index (sklearn's introsort leaves
    them in an unspecified order; inputs on distinct coordinates have none).
"""
import numpy as np
import scipy.stats as sps

EPSILON = np.finfo(np.float64).eps
FEATURE_THRESHOLD = np.float32(1e-7)
RAND_R_MAX = 0x7FFFFFFF
TREE_LEAF, TREE_UNDEFINED = -1, -2


def _seqsum(a):
    """Left-to-right double sum (np.sum is pairwise)."""
    return float(np.add.accumulate(a)[-1]) if len(a) else 0.0


class _RandR(object):
    def __init__(self, state):
        self.s = np.uint32(state)

    def rand_int(self, low, high):
        s = int(self.s) or 1
        s ^= (s << 13) & 0xFFFFFFFF
        s ^= s >> 17
        s ^= (s << 5) & 0xFFFFFFFF
        self.s = np.uint32(s)
        return low + (s % (RAND_R_MAX + 1)) % (high - low)


class Tree(object):
    """Node arrays in sklearn's layout (tree_.feature, .threshold, .children_left, .children_right,
    .n_node_samples, .value[:, 0, 0])."""

    def __init__(self):
        self.feature, self.threshold, self.children_left, self.children_right = [], [], [], []
        self.n_node_samples, self.value = [], []

    def _add(self, parent, is_left, is_leaf, feature, threshold, n, value):
        nid = len(self.feature)
        if parent != TREE_UNDEFINED:
            if is_left:
                self.children_left[parent] = nid
            else:
                self.children_right[parent] = nid
        self.feature.append(TREE_UNDEFINED if is_leaf else feature)
        self.threshold.append(float(TREE_UNDEFINED) if is_leaf else threshold)
        self.children_left.append(TREE_LEAF)
        self.children_right.append(TREE_LEAF)
        self.n_node_samples.append(n)
        self.value.append(value)
        return nid

    def finish(self):
        for k, dt in (("feature", np.int64), ("threshold", np.float64), ("children_left", np.int64),
                      ("children_right", np.int64), ("n_node_samples", np.int64), ("value", np.float64)):
            setattr(self, k, np.asarray(getattr(self, k), dtype=dt))
        return self

    def apply(self, X):
        X = np.asarray(X, dtype=np.float32)
        node = np.zeros(X.shape[0], dtype=np.int64)
        active = self.children_left[node] != TREE_LEAF
        while np.any(active):
            a = np.nonzero(active)[0]
            nd = node[a]
            go_left = X[a, self.feature[nd]].astype(np.float64) <= self.threshold[nd]
            node[a] = np.where(go_left, self.children_left[nd], self.children_right[nd])
            active[a] = self.children_left[node[a]] != TREE_LEAF
        return node

    def predict(self, X):
        return self.value[self.apply(X)]


def _sums(wy, w, start, pos, end, sum_total, wn):
    """(sum_left, weighted_n_left) after RegressionCriterion.reset(); update(pos): from start forwards or from end
    backwards, whichever is shorter."""
    if pos - start <= end - pos:
        return _seqsum(wy[start:pos]), _seqsum(w[start:pos])
    sl, wl = sum_total, wn
    for q in range(end - 1, pos - 1, -1):
        sl -= wy[q]
        wl -= w[q]
    return sl, wl


def _scan(xs, wy, w, sum_total, wn):
    """Best split of one feature over a node whose samples are sorted by it (xs float32, ascending):
    (proxy, pos, threshold) of the first maximum, or None when no position is valid (relative positions)."""
    n = xs.shape[0]
    valid = np.nonzero(xs[1:] > xs[:-1] + FEATURE_THRESHOLD)[0] + 1       # next_p: positions not inside a tie
    if valid.shape[0] == 0:
        return None
    prev = np.concatenate(([0], valid[:-1]))
    if np.all(valid - prev <= n - valid):                                 # every update runs forwards
        csl, cwl = np.add.accumulate(wy), np.add.accumulate(w)
        sl, wl = csl[valid - 1], cwl[valid - 1]
    else:
        sl, wl = np.empty(valid.shape[0]), np.empty(valid.shape[0])
        s, ww, pos = 0.0, 0.0, 0
        for k, p in enumerate(valid):
            if p - pos <= n - p:
                for q in range(pos, p):
                    s += wy[q]
                    ww += w[q]
            else:
                s, ww = sum_total, wn
                for q in range(n - 1, p - 1, -1):
                    s -= wy[q]
                    ww -= w[q]
            sl[k], wl[k], pos = s, ww, p
    sr, wr = sum_total - sl, wn - wl
    proxy = sl * sl / wl + sr * sr / wr
    k = int(np.argmax(proxy))
    p = int(valid[k])
    thr = float(np.float64(xs[p - 1]) / 2.0 + np.float64(xs[p]) / 2.0)
    return float(proxy[k]), p, thr


def build_tree(X, y, weight, rand_r_state, max_features, max_depth=None, min_samples_split=2):
    """One regression tree as sklearn 1.9 grows it with the given sample weights and splitter rand_r state."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    y = np.asarray(y, dtype=np.float64)
    weight = np.asarray(weight, dtype=np.float64)
    N, D = X.shape
    max_depth = np.iinfo(np.int32).max if max_depth is None else int(max_depth)
    rng = _RandR(rand_r_state)
    samples = np.nonzero(weight != 0.0)[0]
    weighted_n_samples = _seqsum(weight)
    features = np.arange(D)
    constant_features = np.empty(D, dtype=np.int64)
    tree = Tree()
    stack = [(0, samples.shape[0], 0, TREE_UNDEFINED, False, np.inf, 0)]
    first = True
    while stack:
        start, end, depth, parent, is_left, impurity, n_known = stack.pop()
        n_node = end - start
        seg = samples[start:end]
        wy_seg, w_seg = weight[seg] * y[seg], weight[seg]
        sum_total, wn = _seqsum(wy_seg), _seqsum(w_seg)
        sq_sum_total = _seqsum(wy_seg * y[seg])
        is_leaf = depth >= max_depth or n_node < min_samples_split or n_node < 2
        if first:
            impurity = sq_sum_total / wn - (sum_total / wn) ** 2
            first = False
        is_leaf = is_leaf or impurity <= EPSILON
        split = None
        n_total = n_known
        if not is_leaf:
            best = None                                       # (proxy, feature, pos, threshold)
            last_order = None
            f_i, n_found, n_drawn, n_visited = D, 0, 0, 0
            n_total = n_known
            while f_i > n_total and (n_visited < max_features or n_visited <= n_found + n_drawn):
                n_visited += 1
                f_j = rng.rand_int(n_drawn, f_i - n_found)
                if f_j < n_known:
                    features[n_drawn], features[f_j] = features[f_j], features[n_drawn]
                    n_drawn += 1
                    continue
                f_j += n_found
                f = features[f_j]
                xv = X[seg, f]
                order = np.lexsort((seg, xv))
                last_order = order
                xs = xv[order]
                if xs[-1] <= xs[0] + FEATURE_THRESHOLD:
                    features[f_j], features[n_total] = features[n_total], features[f_j]
                    n_found += 1
                    n_total += 1
                    continue
                f_i -= 1
                features[f_i], features[f_j] = features[f_j], features[f_i]
                r = _scan(xs, wy_seg[order], w_seg[order], sum_total, wn)
                if r is not None and (best is None or r[0] > best[0]):
                    best = (r[0], f, start + r[1], r[2])
            if last_order is not None:                         # the splitter sorts samples in place
                samples[start:end] = seg[last_order]
            if best is not None and best[2] < end:
                _, f, pos, thr = best
                ps, pe = start, end                            # partition_samples_final: swap partition
                while ps < pe:
                    if np.float64(X[samples[ps], f]) <= thr:
                        ps += 1
                    else:
                        pe -= 1
                        samples[ps], samples[pe] = samples[pe], samples[ps]
                seg = samples[start:end]
                wy_p, w_p = weight[seg] * y[seg], weight[seg]
                sl, wl = _sums(wy_p, w_p, 0, pos - start, n_node, sum_total, wn)
                sq_l = _seqsum(wy_p[:pos - start] * y[seg[:pos - start]])
                sr, wr = sum_total - sl, wn - wl
                imp_l = sq_l / wl - (sl / wl) ** 2
                imp_r = (sq_sum_total - sq_l) / wr - (sr / wr) ** 2
                improvement = (wn / weighted_n_samples) * (impurity - wr / wn * imp_r - wl / wn * imp_l)
                split = (f, thr, pos, imp_l, imp_r)
                is_leaf = improvement + EPSILON < 0.0
            else:
                is_leaf = True
            features[:n_known] = constant_features[:n_known]
            constant_features[n_known:n_known + n_found] = features[n_known:n_known + n_found]
        nid = tree._add(parent, is_left, is_leaf, split[0] if split else 0, split[1] if split else 0.0, n_node,
                        sum_total / wn)
        if not is_leaf:
            f, thr, pos, imp_l, imp_r = split
            stack.append((pos, end, depth + 1, nid, False, imp_r, n_total))
            stack.append((start, pos, depth + 1, nid, True, imp_l, n_total))
    return tree.finish()


def fit(X, y, weights, rand_r_states, max_features, max_depth=None, min_samples_split=2):
    return [build_tree(X, y, w, s, max_features, max_depth, min_samples_split) for w, s in zip(weights, rand_r_states)]


def predict(forest, X):
    """(mean, var) of RF:16-26: mean = sum(all)/T in tree order, var = np.var(all, axis=0, ddof=1)."""
    allp = np.array([t.predict(X) for t in forest])
    T = allp.shape[0]
    mean = np.add.accumulate(allp, axis=0)[-1] / T
    with np.errstate(invalid="ignore", divide="ignore"):
        var = np.add.accumulate((allp - mean) ** 2, axis=0)[-1] / (T - 1) if T > 1 else np.full(allp.shape[1], np.nan)
    return mean, var


def ei(mean, var, best):
    """RF:80-85."""
    with np.errstate(invalid="ignore"):
        s = np.sqrt(var) + 0.0001
        u = (best - mean) / s
        return s * (u * sps.norm.cdf(u) + sps.norm.pdf(u))


class OracleBackend(object):
    """The forest part of DeviceBackend's interface, on this oracle.  ``fits`` records every fit's arguments and
    ``forest`` / ``best`` the last fit and EI reference value, so tests can look inside a next() call."""
    name = "rf-oracle"

    def __init__(self):
        self.fits, self.forest, self.best = [], None, None

    def forest_fit(self, X, y, weights, rand_r_states, max_features, max_depth=None, min_samples_split=2):
        self.fits.append(dict(X=np.array(X), y=np.array(y), weights=weights, rand_r_states=rand_r_states,
                              max_features=max_features, max_depth=max_depth, min_samples_split=min_samples_split))
        self.forest = fit(X, y, weights, rand_r_states, max_features, max_depth, min_samples_split)
        return self.forest

    def forest_predict(self, forest, X):
        return predict(forest, X)

    def forest_argmax_ei(self, forest, cand, best):
        self.best = best
        m, v = predict(forest, cand)
        return int(np.argmax(ei(m, v, best)))
