"""The film accumulator of rayn_b200_accum_round / accum_resolve (include/rayn_b200.h, at RaynAdaptiveDesc) restated in
numpy.  Float32 arrays with float32 scalars throughout, np.fmax (NaN-ignoring, like fmaxf), and the tile sum is the
sequential np.cumsum in float64, never the pairwise np.sum."""
import numpy as np

F = np.float32
TINY = F(2.0 ** -10)
NC = {"color": 3, "alpha": 1, "background": 3, "normal": 3}


def tile_grid(w, h, tw, th):
    return (w + w % tw) // tw, (h + h % th) // th  # film.rs:399-404


def tile_error(sc, sb, hh, k, kh):
    """E of one tile from its S.color, S.background and H rows ([count, 3] float32, ascending pixel index)."""
    i = (sc + sb) / F(k)
    a = hh / F(kh)
    dd = np.abs(i - a)
    d = (dd[:, 0] + dd[:, 1]) + dd[:, 2]
    s = (i[:, 0] + i[:, 1]) + i[:, 2]
    e = d / np.sqrt(np.fmax(s, TINY))
    e = np.where(np.isnan(e), F(np.inf), e).astype(np.float32)
    return float(np.cumsum(e.astype(np.float64))[-1]) / float(len(e))


class AccumMirror:
    def __init__(self, w, h, tw, th):
        self.w, self.h, self.tw, self.th = w, h, tw, th
        self.ntx, self.nty = tile_grid(w, h, tw, th)
        self.n_tiles = self.ntx * self.nty
        npx = w * h
        self.S = {k: np.zeros(npx * c, np.float32) for k, c in NC.items()}
        self.H = np.zeros(3 * npx, np.float32)
        self.K = np.zeros(self.n_tiles, np.int64)
        self.Kh = np.zeros(self.n_tiles, np.int64)
        self.rounds = np.zeros(self.n_tiles, np.int32)
        self.E = np.full(self.n_tiles, np.inf)

    def tile_pixels(self, t):
        """in-image pixel indices x + y*w of tile t, ascending"""
        tx, ty = divmod(t, self.nty)
        x0, y0 = tx * self.tw, ty * self.th
        xs, ys = np.arange(x0, min(x0 + self.tw, self.w)), np.arange(y0, min(y0 + self.th, self.h))
        return (ys[:, None] * self.w + xs[None, :]).ravel()

    def active(self, min_rounds, max_rounds, threshold):
        thr = float(F(threshold))
        return [t for t in range(self.n_tiles)
                if self.rounds[t] < max_rounds and (self.rounds[t] < min_rounds or not (self.E[t] <= thr))]

    def fold(self, planes, tiles, samples):
        """One round: `planes` (flat float32, already / spp) rendered over `tiles` at 4*samples spp."""
        n = F(4 * samples)
        for t in tiles:
            p = self.tile_pixels(t)
            for k, c in NC.items():
                idx = (p[:, None] * c + np.arange(c)).ravel()
                self.S[k][idx] = self.S[k][idx] + planes[k][idx] * n
            idx3 = (p[:, None] * 3 + np.arange(3)).ravel()
            upd_h = self.rounds[t] % 2 == 0
            if upd_h:
                self.H[idx3] = self.H[idx3] + (planes["color"][idx3] + planes["background"][idx3]) * n
                self.Kh[t] += 4 * samples
            self.K[t] += 4 * samples
            self.rounds[t] += 1
            if self.rounds[t] >= 2:
                self.E[t] = tile_error(self.S["color"][idx3].reshape(-1, 3), self.S["background"][idx3].reshape(-1, 3),
                                       self.H[idx3].reshape(-1, 3), self.K[t], self.Kh[t])
            else:
                self.E[t] = np.inf

    def resolve(self):
        npx = self.w * self.h
        x, y = np.arange(npx) % self.w, np.arange(npx) // self.w
        tx, ty = x // self.tw, y // self.th
        covered = (tx < self.ntx) & (ty < self.nty)
        k = np.where(covered, self.K[np.where(covered, tx * self.nty + ty, 0)], 1).astype(np.float32)
        out = {}
        for ch, c in NC.items():
            v = self.S[ch].reshape(npx, c) / k[:, None]
            out[ch] = np.where(covered[:, None], v, F(0)).astype(np.float32).ravel()
        return out
