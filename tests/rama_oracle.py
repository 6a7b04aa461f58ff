"""numpy restatement of VIAMD's Ramachandran density task (src/components/ramachandran/ramachandran.cpp:1277-1370). TEST INFRASTRUCTURE ONLY.

Scatter of (phi, psi) into a 512 x 512 map per residue class, the float saturation of the reference's `+= 1.0f`, and the running-sum recurrence
of its box passes (blur_density_gaussian), vectorised over lines x channels. Pinned against tests/golden/rama.npz by tests/test_rama_density.py.
"""
from __future__ import annotations

import numpy as np

RAMA_DIM = 512


def rama_box_radii(sigma):
    """boxes_for_gauss(., 3, sigma) (:333-344), float32 for float32"""
    f = np.float32; s = f(sigma)
    lo = int(np.sqrt(f(12) * s * s / f(3) + f(1)))
    if lo % 2 == 0: lo -= 1
    n_lo = int((f(12) * s * s - f(3 * lo * lo) - f(12 * lo) - f(9)) / f(-4 * lo - 4) + f(0.5))
    return [lo if i < n_lo else lo + 2 for i in range(3)]


def rama_texel(a):
    """texture coordinate of an angle: ((uint32_t)((a * (float)(1 / 2pi) + 0.5f) * 512.0f)) & 511, truncation toward zero"""
    w = ((np.asarray(a, np.float32) * np.float32(1.0 / (2.0 * 3.1415926535897932))) + np.float32(0.5)) * np.float32(RAMA_DIM)
    return np.where(w > 0, np.minimum(w, np.float32(4294967040.0)), np.float32(0)).astype(np.int64) & (RAMA_DIM - 1)   # w <= 0 and NaN -> 0


def _rama_box_pass(src, k):
    """blur_rows_acc along axis 0 of src [512, lines], all lines at once, in the reference's order of operations"""
    scl = np.float32(1) / np.float32(2 * k + 1)
    acc = np.zeros(src.shape[1:], np.float32)
    for x in range(-(k + 1), k): acc = acc + src[x & (RAMA_DIM - 1)]
    out = np.empty_like(src)
    for x in range(RAMA_DIM):
        acc = np.maximum(np.float32(0), (acc - src[(x - k - 1) & (RAMA_DIM - 1)]) + src[(x + k) & (RAMA_DIM - 1)])
        out[x] = acc * scl
    return out


def rama_blur(m, sigma):
    """blur_density_gaussian (:368-387) of m [4, 512 (y), 512 (x)] float32 -> [512 (y), 512 (x), 4]: three passes along x, three along y"""
    box = rama_box_radii(sigma)
    a = np.ascontiguousarray(np.asarray(m, np.float32).transpose(2, 0, 1)).reshape(RAMA_DIM, -1)    # [x][(c, y)]
    for k in box: a = _rama_box_pass(a, k)
    b = np.ascontiguousarray(a.reshape(RAMA_DIM, 4, RAMA_DIM).transpose(2, 1, 0)).reshape(RAMA_DIM, -1)   # [y][(c, x)]
    for k in box: b = _rama_box_pass(b, k)
    return np.ascontiguousarray(b.reshape(RAMA_DIM, 4, RAMA_DIM).transpose(0, 2, 1))


def rama_counts(angles, seg, class_off, frames):
    """samples per texel [4, 512 (y), 512 (x)] (int64) and per class of angles [F, nseg, 2] over the frame indices `frames`"""
    a = np.asarray(angles, np.float32)[np.asarray(frames, np.int64)]
    counts = np.zeros((4, RAMA_DIM * RAMA_DIM), np.int64); n = np.zeros(4, np.int64)
    for c in range(4):
        p = a[:, np.asarray(seg[class_off[c]:class_off[c + 1]], np.int64)].reshape(-1, 2)
        p = p[~((p[:, 0] == 0) & (p[:, 1] == 0))]   # segments without angles
        counts[c] = np.bincount(rama_texel(p[:, 1]) * RAMA_DIM + rama_texel(p[:, 0]), minlength=RAMA_DIM * RAMA_DIM); n[c] = len(p)
    return counts.reshape(4, RAMA_DIM, RAMA_DIM), n


def rama_density(angles, seg, class_off, frames, sigma):
    """-> (tex [512, 512, 4] float32 in VIAMD's density_tex layout, sums [4] float32): texel values saturate at 2^24 as `+= 1.0f` does"""
    counts, n = rama_counts(angles, seg, class_off, frames)
    return rama_blur(np.minimum(counts, 1 << 24).astype(np.float32), sigma), np.array([np.float32(float(v)) for v in n], np.float32)
