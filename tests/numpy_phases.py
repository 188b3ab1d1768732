"""A numpy restatement of the split-phase normalise/select calls (fl_norm_* / fl_select_*), used
only to test the sharding PROTOCOL of filtlong_b200/sharding.py on CPU (gloo, world size 2) and to
cross-check the weighted radix-select formulation against the oracle's sort + prefix walk."""
import math
import types

import numpy as np


def score_keys(final):
    """Ascending key == descending score; NaN -> best key (fl_select.cu: score_key)."""
    x = np.asarray(final, dtype=np.float64) + 0.0
    b = x.view(np.uint64)
    neg = (b >> np.uint64(63)).astype(bool)
    u = np.where(neg, ~b, b | np.uint64(1 << 63))
    k = ~u
    k[np.isnan(x)] = 0
    return k


def target_and_status(p, total, passed_bases):
    """main.cpp:229-244: the signed target and the status (0 no target, 1 not enough reads, 2 already
    below the target, 3 cut). The target is 0 when neither option is set, as fl_summary reports it."""
    if not (p.target_bases_set or p.keep_percent_set):
        return 0, 0
    target = p.target_bases if p.target_bases_set else (1 << 63) - 1
    if p.keep_percent_set:
        target = min(target, int((p.keep_percent / 100.0) * total))
    return target, (1 if target >= total else (2 if target >= passed_bases else 3))


class NumpyPhases:
    def __init__(self, mean, window, length, passed, params):
        self.mean = np.asarray(mean, dtype=np.float64)
        self.window = np.asarray(window, dtype=np.float64)
        self.length = np.asarray(length, dtype=np.int64)
        self.passed = np.asarray(passed, dtype=bool)
        self.p = params
        self.state = types.SimpleNamespace()

    def norm_partial1(self, sums, mn, mx):
        m = self.mean
        s = sums.numpy()
        s[0], s[1] = len(m), m.sum() if len(m) else 0.0
        s[2], s[3] = self.length[self.passed].sum(), self.length.sum()
        lo, hi = 100.0, 0.0
        for x in m:
            if x > hi: hi = x
            if x < lo: lo = x
        mn.numpy()[0], mx.numpy()[0] = lo, hi

    def norm_partial2(self, sums, mn, mx, sq):
        mean = sums.numpy()[1] / sums.numpy()[0]
        sq.numpy()[0] = ((self.mean - mean) ** 2).sum() if len(self.mean) else 0.0

    def norm_apply(self, sums, mn, mx, sq):
        n = sums.numpy()[0]
        mean = sums.numpy()[1] / n
        sd = math.sqrt(sq.numpy()[0] / n)
        if sd > 0.0:
            minz, maxz = (mn.numpy()[0] - mean) / sd, (mx.numpy()[0] - mean) / sd
        else:
            minz = maxz = 1.0
        with np.errstate(all="ignore"):
            ratio = self.window / self.mean
            ratio = np.where(ratio > 1.0, 1.0, ratio)
            z = (self.mean - mean) / sd
            nm = 100.0 * (z - minz) / (maxz - minz)
            nw = nm * ratio
            ls = 100.0 * (1.0 + (-5000.0 / (self.length + 5000.0)))
            lw, mw, ww = self.p.length_weight, self.p.mean_q_weight, self.p.window_q_weight
            fs = np.power(np.power(ls, lw) * np.power(nm, mw), 1.0 / (lw + mw))
            r = nw / nm
            sf = np.where(nm > 0.0, np.where(1.0 < r, 1.0, r), 1.0)
            wf = ww / (lw + mw + ww)
            self.final = fs * ((1.0 - wf) + sf * wf)
        self.key = score_keys(self.final)
        self.pfinal = self.passed.copy()

    def select_begin(self, total, sums):
        st = self.state
        p = self.p
        st.passed_bases, st.total = int(sums.numpy()[2]), total
        st.target, st.status = target_and_status(p, total, st.passed_bases)
        st.active = st.status == 3 and st.target > 0          # a target <= 0 keeps nothing
        st.prefix, st.cum = 0, 0

    def select_hist(self, level, hist):
        h = hist.numpy()
        h[:] = 0
        st = self.state
        if not st.active:
            return
        shift = 56 - 8 * level
        for k, l, ok in zip(self.key, self.length, self.passed):
            k = int(k)
            if not ok or (level > 0 and (k >> (shift + 8)) != st.prefix):
                continue
            h[(k >> shift) & 0xFF] += int(l)

    def select_pick(self, level, hist):
        st = self.state
        if not st.active:
            return
        cum = st.cum
        for d, c in enumerate(hist.numpy()):
            c = int(c)
            if c and cum + c >= st.target:
                st.prefix, st.cum = (st.prefix << 8) | d, cum
                return
            cum += c
        raise AssertionError("no digit reaches the target although status == 3")

    def select_tie_local(self, tie, rank, world):
        st = self.state
        t = tie.numpy()
        t[:] = 0
        if st.active:
            self.tie_mask = self.passed & (self.key == np.uint64(st.prefix))
            t[rank] = int(self.length[self.tie_mask].sum())

    def select_apply(self, tie, rank, keeping):
        st = self.state
        keeping.numpy()[0] = 0
        if st.status == 3 and not st.active:
            self.pfinal = np.zeros_like(self.passed)
        if not st.active:
            return
        before = int(tie.numpy()[:rank].sum())
        room = st.target - st.cum
        keep = self.passed & (self.key < np.uint64(st.prefix))
        run = before
        for i in np.nonzero(self.tie_mask)[0]:
            if run < room:
                keep[i] = True
            run += int(self.length[i])
        self.pfinal = keep
        keeping.numpy()[0] = int(self.length[keep].sum())

    def select_summary(self, sums, mn, mx, sq, keeping, total):
        st = self.state
        return types.SimpleNamespace(status=st.status, target=st.target, passed_bases=st.passed_bases,
                                     keeping=int(keeping.numpy()[0]) if st.status == 3 else 0, total_bases=total)
