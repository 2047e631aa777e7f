"""Models, float64 references, bounds and edge-case generators for the kernels ahead of the head: the device preprocess,
the greedy NMS shared by frcnn_proposals / frcnn_nms_sorted_dev / frcnn_nms_host, the score sort, the SIMT convolutions and
max pool (`test_front_edges_gpu.py`; their teeth are shown on the CPU by `test_front_ref64.py`).  No GPU here."""
from fractions import Fraction

import numpy as np
import torch

from stage_ref64 import TINY, U, gamma

F = np.float32

# ---- preprocess ---------------------------------------------------------------------------------------------------------
# preprocess_kernel<HFLIP> per output pixel (dx, dy), per axis:
#   c  = (d + 0.5) * inv - 0.5      float64, inv = RN(1 / f); nvcc contracts it into one DFMA, so c is rounded ONCE
#   s  = floor(c), fr = float32(c - s)  (the subtraction is exact)
#   s < 0 -> (s, fr) = (0, 0);  s >= n - 1 -> (s, fr) = (n - 1, 0);  s1 = min(s + 1, n - 1)
# then v = float32(pixel - mean) (float64 difference, rounded once), a0 = fl(1 - fr_x), b0 = fl(1 - fr_y), and
#   out = fl(fl(t0 * b0) + fl(t1 * b1)),  t_r = fl(fl(v[r, x0] * a0) + fl(v[r, x1] * a1))     (__f*_rn: no FMA)
# HFLIP reads column n - 1 - s of the image for source column s.


def axis_model(n_out, n_in, f, frac32=False, right_keeps_frac=False):
    """Source indices (s0, s1) and float32 fractions of one axis.  frac32 / right_keeps_frac are the mutants of
    test_front_ref64.py: the fraction of the float32 coordinate, and a right-border clamp that leaves the fraction."""
    inv = Fraction(1.0 / f)
    c = np.array([float((d + Fraction(1, 2)) * inv - Fraction(1, 2)) for d in range(n_out)])   # one rounding
    s = np.floor(c)
    fr = ((c.astype(F) - np.floor(c.astype(F))) if frac32 else (c - s)).astype(F)
    s = s.astype(np.int64)
    lo, hi = s < 0, s >= n_in - 1
    fr[lo] = 0
    s[lo] = 0
    if not right_keeps_frac:
        fr[hi] = 0
    s[hi] = n_in - 1
    return s, np.minimum(s + 1, n_in - 1), fr


def preprocess_model(img, means, fx, fy, H, W, hflip=False, frac32=False, fma=False, right_keeps_frac=False, flip_off=0):
    """preprocess_kernel in numpy -> float32 [H, W, 3].  fma / flip_off are mutants (FMA-contracted lerps, HFLIP off by one)."""
    h0, w0 = img.shape[:2]
    v = (img.astype(np.float64) - np.asarray(means, np.float64)).astype(F)
    sx0, sx1, ax = axis_model(W, w0, fx, frac32, right_keeps_frac)
    sy0, sy1, ay = axis_model(H, h0, fy, frac32, right_keeps_frac)
    if hflip:
        sx0, sx1 = np.clip(w0 - 1 - sx0 + flip_off, 0, w0 - 1), np.clip(w0 - 1 - sx1 + flip_off, 0, w0 - 1)
    a0, a1 = (F(1) - ax)[None, :, None], ax[None, :, None]
    b0, b1 = (F(1) - ay)[:, None, None], ay[:, None, None]

    def lerp(p, wp, q, wq):
        if fma:          # fl(p * wp + fl(q * wq)) with one rounding for the first product: a contracted FFMA
            return (p.astype(np.float64) * wp + (q * wq).astype(np.float64)).astype(F)
        return (p * wp + q * wq).astype(F)

    t0 = lerp(v[sy0][:, sx0], a0, v[sy0][:, sx1], a1)
    t1 = lerp(v[sy1][:, sx0], a0, v[sy1][:, sx1], a1)
    return lerp(t0, b0, t1, b1)


def _axis_truth(n_out, n_in, f):
    """Exact coordinate clamped into [0, n_in - 1] -> up to 4 (index, weight) slots: the two interpolation taps and their
    outer neighbours (weight 0), and the allowance E per slot for the kernel's weight error."""
    inv64 = 1.0 / f
    c = np.array([float((d + Fraction(1, 2)) / Fraction(f) - Fraction(1, 2)) for d in range(n_out)])
    c = np.clip(c, 0.0, n_in - 1)
    t = np.floor(c).astype(np.int64)
    fr = c - t
    idx = np.clip(np.stack([t - 1, t, t + 1, t + 2], axis=1), 0, n_in - 1)
    w = np.stack([np.zeros_like(fr), 1 - fr, fr, np.zeros_like(fr)], axis=1)
    for j in range(1, 4):                       # a clipped tap that repeats an earlier index carries no weight of its own
        for i in range(j):
            dup = idx[:, j] == idx[:, i]
            w[dup, i] += w[dup, j]
            w[dup, j] = 0
            idx[dup, j] = -1
    # kernel weight error: the coordinate (inv = RN(1/f): 2^-53 relative; the DFMA: 2^-53 |c|) moves the fraction by dc;
    # rounding it to fp32 adds u |fr|, and fl(1 - fr) another u.  When the exact coordinate lies within dc of an integer
    # the kernel's taps may be the neighbours', with a weight <= dc + u on them: hence the outer slots.
    dc = 2.0 ** -52 * ((np.arange(n_out) + 0.5) * inv64 + 1.0)
    E = dc + 2 * U
    return idx, w, E


def preprocess_truth(img, means, fx, fy, H, W, hflip=False):
    """(float64 bilinear value of pixel - mean at the exact, border-clamped source coordinate, per-element bound).

    Bound.  Per axis the kernel's weights differ from the exact ones by at most E (above) on each of the 4 slots; v differs
    from V = pixel - mean by u |V|; each output is 2 products + 1 sum per pass, two passes, so (v, 4 operations on the
    longest path) the arithmetic adds gamma_5 * sum |Wy Wx V| over the taps, computed with the weights inflated by E:
        |out - out64| <= sum_{p,q} |V_pq| ((|Wy_p| + Ey)(|Wx_q| + Ex) - |Wy_p||Wx_q|) (1 + gamma_5) + gamma_5 sum |Wy Wx V|."""
    h0, w0 = img.shape[:2]
    V = img.astype(np.float64) - np.asarray(means, np.float64)
    if hflip:
        V = V[:, ::-1]
    iy, wy, ey = _axis_truth(H, h0, fy)
    ix, wx, ex = _axis_truth(W, w0, fx)
    val = np.zeros((H, W, 3))
    s_abs = np.zeros((H, W, 3))
    s_coef = np.zeros((H, W, 3))
    for p in range(4):
        for q in range(4):
            vy, vx = iy[:, p] >= 0, ix[:, q] >= 0
            Vpq = V[np.maximum(iy[:, p], 0)][:, np.maximum(ix[:, q], 0)] * (vy[:, None] & vx[None, :])[..., None]
            Wp, Wq = wy[:, p][:, None, None], wx[:, q][None, :, None]
            val += Wp * Wq * Vpq
            s_abs += np.abs(Wp * Wq * Vpq)
            s_coef += np.abs(Vpq) * ((np.abs(Wp) + ey[:, None, None]) * (np.abs(Wq) + ex[None, :, None]) - np.abs(Wp * Wq))
    g5 = gamma(5)
    return val, (s_coef * (1 + g5) + g5 * s_abs) * (1 + 8 * U) + TINY


def blob_size(h0, w0, f):
    """cv2.resize's dsize for fx = fy = f: round half to even of the scaled size (model/test.py::blob_geometry)."""
    return int(np.rint(h0 * f)), int(np.rint(w0 * f))


# image geometries: (name, h0, w0, fx, fy, H, W); fx / fy are what the C ABI takes, H / W the blob
def preprocess_geometries():
    g = []
    for name, h0, w0, f in (("x0.5", 240, 322, 0.5), ("x1", 97, 131, 1.0), ("x2", 61, 83, 2.0)):
        g.append((name, h0, w0, f, f) + blob_size(h0, w0, f))
    g += [("1xN", 1, 517, 1.6, 1.6, 2, 827), ("Nx1", 389, 1, 1.6, 1.6, 622, 2),
          ("1x1", 1, 1, 600.0, 600.0, 600, 600), ("2x2", 2, 2, 300.0, 300.0, 600, 600), ("3x1", 3, 1, 200.0, 200.0, 600, 200),
          ("fx!=fy", 375, 500, 1.6, 1.2, 450, 800),
          ("aspect", 30, 1400, 1000 / 1400, 1000 / 1400) + blob_size(30, 1400, 1000 / 1400)]
    return g


def tta_geometries(h0=375, w0=500, scales=((600, 1000), (480, 2000), (720, 2000))):
    """The blob of each TEST.SCALES / BBOX_AUG.SCALES short side (model/test.py::_scale_factor)."""
    out = []
    for target, max_size in scales:
        f = float(target) / min(h0, w0)
        if np.round(f * max(h0, w0)) > max_size:
            f = float(max_size) / max(h0, w0)
        out.append(("scale%d" % target, h0, w0, f, f) + blob_size(h0, w0, f))
    return out


def edge_image(rng, h0, w0):
    """uint8 BGR image with the extremes present: 0 and 255 in the corners, the rest uniform."""
    im = rng.integers(0, 256, (h0, w0, 3), dtype=np.uint8)
    im.reshape(-1, 3)[0] = 0
    im.reshape(-1, 3)[-1] = 255
    return im


# ---- greedy NMS (block_greedy_nms, nms.cu) ------------------------------------------------------------------------------
PLUS_ONE, INCLUSIVE, SKIP_DEGENERATE = 1, 2, 4      # FRCNN_NMS_* flags
WIDE, CHUNK = 1024, 256


def canon(b, flags):
    if flags & PLUS_ONE:
        return b.astype(F)
    return np.stack([np.minimum(b[:, 0], b[:, 2]), np.minimum(b[:, 1], b[:, 3]),
                     np.maximum(b[:, 0], b[:, 2]), np.maximum(b[:, 1], b[:, 3])], axis=1).astype(F)


def box_area(b, flags):
    if flags & PLUS_ONE:
        return ((b[:, 2] - b[:, 0] + F(1)) * (b[:, 3] - b[:, 1] + F(1))).astype(F)
    return ((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])).astype(F)


def suppresses(a, aa, b, ab, thr, flags):
    """Matrix [len(a), len(b)]: does a suppress b (the kernel's `suppresses`, fp32 op by op)."""
    a, b = a[:, None, :], b[None, :, :]
    aa, ab = aa[:, None], ab[None, :]
    one = F(1) if flags & PLUS_ONE else F(0)
    w = np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]) + one
    h = np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]) + one
    inter = (np.maximum(w, F(0)) * np.maximum(h, F(0))).astype(F)
    with np.errstate(divide="ignore", invalid="ignore"):
        ovr = (inter / ((aa + ab) - inter)).astype(F)
    s = (ovr >= F(thr)) if flags & INCLUSIVE else (ovr > F(thr))
    if not flags & PLUS_ONE and flags & SKIP_DEGENERATE:
        s &= (aa > 0) & (ab > 0)
    return s


def greedy_nms_model(boxes, thr, flags, max_out, mutant=None):
    """block_greedy_nms over `boxes` given in priority order -> (kept positions, path counters).
    Counters: rounds, tpc4 (rounds with 4 threads per candidate), cuts (windows cut after the 256th survivor), cut_rounds,
    maxout_mid_chunk (max_out reached with unresolved survivors left in the chunk), window_ends (base after each round).
    mutant: 'resolve_suppressed' (every row's mask is applied, a suppressed one's too), 'cut_skip' / 'cut_repeat' (the
    window cut one candidate after the 257th survivor / at the 256th survivor)."""
    b = canon(np.asarray(boxes, F).reshape(-1, 4), flags)
    ar = box_area(b, flags)
    m = b.shape[0]
    kept = []
    st = dict(rounds=0, tpc4=0, tpc1=0, cuts=0, cut_rounds=[], maxout_mid_chunk=False, window_ends=[])
    tot_alive, last_wn, base = WIDE, WIDE, 0
    while base < m and len(kept) < max_out:
        tpc = 4 if tot_alive * 3 >= last_wn else 1
        wn = min(WIDE // tpc, m - base)
        win = np.arange(base, base + wn)
        dead = np.zeros(wn, bool)
        if thr >= 0 and kept:
            k = np.asarray(kept)
            dead = suppresses(b[k], ar[k], b[win], ar[win], thr, flags).any(axis=0)
        alive = win[~dead]
        tot_alive, last_wn = alive.shape[0], wn
        st["rounds"] += 1
        st["tpc4" if tpc == 4 else "tpc1"] += 1
        consumed = wn
        if alive.shape[0] > CHUNK:
            st["cuts"] += 1
            st["cut_rounds"].append(st["rounds"] - 1)
            consumed = int(alive[CHUNK]) - base
            if mutant == "cut_skip":
                consumed += 1
            elif mutant == "cut_repeat":
                consumed = int(alive[CHUNK - 1]) - base
        chunk = alive[:CHUNK]
        removed = np.zeros(chunk.shape[0], bool)
        mask = suppresses(b[chunk], ar[chunk], b[chunk], ar[chunk], thr, flags) if thr >= 0 else None
        for i in range(chunk.shape[0]):
            if removed[i] and mutant != "resolve_suppressed":
                continue
            if not removed[i]:
                if len(kept) >= max_out:
                    st["maxout_mid_chunk"] = True
                    break
                kept.append(int(chunk[i]))
            if mask is not None:
                removed[i + 1:] |= mask[i, i + 1:]
        base += consumed
        st["window_ends"].append(base)
    return np.asarray(kept, np.int64), st


def oracle_keep(boxes, scores, thr, flags, max_out):
    """The oracle's survivors (positions in priority order) of boxes already in priority order, for the flag set."""
    from oracle import nms as ONMS
    boxes = np.ascontiguousarray(boxes, F)
    scores = np.ascontiguousarray(scores, F)
    if flags & PLUS_ONE:
        dets = np.hstack([boxes, scores[:, None]]).astype(F)
        return ONMS.nms_plus1_c(dets, float(thr), bool(flags & INCLUSIVE))[:max_out].astype(np.int64)
    return ONMS.nms_tf_c(boxes, scores, max_out, float(thr)).astype(np.int64)


MODES = {"tf": SKIP_DEGENERATE, "gpu_nms": PLUS_ONE, "cpu_nms": PLUS_ONE | INCLUSIVE}


def grid_boxes(n, size=20.0, pitch=30.0, cols=64, x0=0.0, y0=0.0):
    """n disjoint size x size boxes on a pitch grid: every candidate survives in every mode."""
    i = np.arange(n)
    x, y = x0 + (i % cols) * pitch, y0 + (i // cols) * pitch
    return np.stack([x, y, x + size - 1, y + size - 1], axis=1).astype(F)


def identical_boxes(n, box=(100.0, 100.0, 180.0, 160.0)):
    return np.tile(np.asarray(box, F), (n, 1))


CHAIN_THR = 0.3


def chain(x0, y0):
    """A -> B -> C, each shifted 50 px: IoU(A, B) = IoU(B, C) = 1/3 (+1 areas) or 49/149 (TF), IoU(A, C) = 0, so at
    CHAIN_THR C survives only because B died."""
    a = [x0, y0, x0 + 99, y0 + 99]
    b = [x0 + 50, y0, x0 + 149, y0 + 99]
    c = [x0 + 100, y0, x0 + 199, y0 + 99]
    return np.asarray([a, b, c], F)


def warm_prefix(box=(5000.0, 5000.0, 5099.0, 5099.0)):
    """512 copies of one box: round 1 (4 threads per candidate) keeps it, round 2 kills the other 256, so the next round is a
    1024-candidate window (1 thread per candidate)."""
    return identical_boxes(2 * CHUNK, box)


def nms_cases():
    """(name, boxes in priority order, thr, max_out, expected path) -- path keys checked against the model's counters."""
    cases = []
    g = grid_boxes(1500)
    cases.append(("grid1500", g, 0.5, 1500, dict(cuts=0, tpc1=0)))
    cases.append(("identical700", identical_boxes(700), 0.5, 300, dict(cuts=0, kept=1)))
    # the window cut: 1024 survivors in a 1-thread window, the 257th starts the next round
    cut = np.vstack([warm_prefix(), grid_boxes(1024)])
    cases.append(("cut", cut, 0.5, 1024, dict(cuts=1, min_tpc1=1)))
    # chain across the cut, A = 256th survivor, B = 257th, C after it
    ch = grid_boxes(1024, y0=3000)
    ch[100:103] = chain(-1000, -500)                 # and a chain inside the chunk (resolved by the bitmask)
    ch[255:258] = chain(-500, -500)
    cases.append(("chain_cut_256", np.vstack([warm_prefix(), ch]), CHAIN_THR, 1024, dict(cuts=1, chain_at=512 + 255)))
    # chain with A = 255th, B = 256th (dies in the chunk's resolve), C = 257th (re-examined next round)
    ch = grid_boxes(1024, y0=3000)
    ch[100:103] = chain(-1000, -500)
    ch[254:257] = chain(-500, -500)
    cases.append(("chain_cut_255", np.vstack([warm_prefix(), ch]), CHAIN_THR, 1024, dict(cuts=1, chain_at=512 + 254)))
    # chain across the 1024-candidate window boundary: A last of a 1-thread window, B / C first of the next
    w = identical_boxes(WIDE, (5000.0, 5000.0, 5099.0, 5099.0))
    w[-1] = chain(-500, -500)[0]
    tail = np.vstack([chain(-500, -500)[1:], grid_boxes(40, y0=3000)])
    cases.append(("chain_window", np.vstack([warm_prefix(), w, tail]), CHAIN_THR, 300, dict(window_end=512 + WIDE, chain_at=512 + WIDE - 1)))
    # max_out reached in the middle of a chunk
    cases.append(("maxout_mid", grid_boxes(600), 0.5, 300, dict(maxout_mid_chunk=True)))
    return cases


def point_cut_case():
    """The cut case with the 256th survivor a zero-area box: under the TF rule it never suppresses (not even itself), so a
    window that re-examines it keeps it twice."""
    g = grid_boxes(1024)
    g[255, 2:] = g[255, :2]
    return np.vstack([warm_prefix(), g])


def exact_threshold_cases():
    """(boxes, thr, survivors per mode) with the overlap exactly at thr: fl(50 / 150) under both area rules.
    gpu_nms (>) and TF (>) keep B, cpu_nms (>=) suppresses it."""
    thr = float(F(50) / F(150))
    plus1 = np.asarray([[0, 0, 9, 9], [0, 5, 9, 14]], F)          # +1 areas 100, 100; inter 10 * 5
    tf = np.asarray([[0, 0, 10, 10], [0, 5, 10, 15]], F)          # areas 100, 100; inter 10 * 5
    return thr, {"gpu_nms": (plus1, [0, 1]), "cpu_nms": (plus1, [0]), "tf": (tf, [0, 1])}


def check_path(st, kept, expect, what=""):
    """The counters of greedy_nms_model confirm the path a case claims to force."""
    for k, v in expect.items():
        if k == "min_tpc1":
            assert st["tpc1"] >= v, "%s: %d 1-thread rounds" % (what, st["tpc1"])
        elif k == "kept":
            assert kept.shape[0] == v, "%s: kept %d" % (what, kept.shape[0])
        elif k == "chain_at":
            assert v in kept and v + 1 not in kept and v + 2 in kept, "%s: chain not A, C" % what
        elif k == "window_end":
            assert v in st["window_ends"], "%s: no round ends at %d (%s)" % (what, v, st["window_ends"])
        else:
            assert st[k] == v, "%s: %s = %r, want %r" % (what, k, st[k], v)


# ---- score sort (sort.cu) -----------------------------------------------------------------------------------------------
def desc_bits(keys):
    """sort.cu's desc_bits: the order-preserving float -> uint map, complemented (ascending key == descending float)."""
    u = np.ascontiguousarray(keys, F).view(np.uint32)
    return ~np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def sort_ref(keys):
    """The device order: stable ascending argsort of desc_bits -- +NaN before +Inf, -NaN after -Inf, +0 before -0, ties by
    index.  Returns (order, sorted keys)."""
    o = np.argsort(desc_bits(keys), kind="stable")
    return o.astype(np.int32), np.ascontiguousarray(keys, F)[o]


def radix_model(keys, mutant=None):
    """cluster_sort_desc_kernel as 4 stable LSD passes of 8-bit digits.  mutant: 'ties_reversed' (pass 2 puts equal digits
    in reverse order), 'shift' (pass 3 reads the digit at bit 16 again)."""
    k = desc_bits(keys)
    idx = np.arange(k.shape[0])
    for p in range(4):
        shift = 16 if (mutant == "shift" and p == 3) else 8 * p
        d = (k[idx] >> np.uint32(shift)) & np.uint32(255)
        if mutant == "ties_reversed" and p == 2:
            idx = idx[::-1][np.argsort(d[::-1], kind="stable")]
        else:
            idx = idx[np.argsort(d, kind="stable")]
    return idx.astype(np.int32)


def from_bits(k):
    """Inverse of desc_bits: uint32 sort keys -> fp32 values."""
    u = ~np.asarray(k, np.uint32)
    return np.where(u & np.uint32(0x80000000), u & np.uint32(0x7fffffff), ~u).astype(np.uint32).view(F)


def one_byte_keys(rng, n, byte):
    """n keys whose sort keys share 3 of their 4 radix bytes: only byte `byte` varies (few distinct values: ties too)."""
    base = np.uint32(rng.integers(0, 2 ** 32, dtype=np.uint64))
    k = np.full(n, base, np.uint32) & ~np.uint32(0xff << (8 * byte))
    k |= (rng.integers(0, 256, n).astype(np.uint32) << np.uint32(8 * byte))
    return from_bits(k)


def special_keys(rng, n):
    """n keys with ±Inf, both NaN signs, ±0, ± subnormals and ties among random values."""
    keys = rng.standard_normal(n).astype(F)
    sp = np.array([np.inf, -np.inf, np.nan, -np.nan, 0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 3e38, -3e38], F)
    sp_bits = sp.view(np.uint32).copy()
    sp_bits[3] = 0xffc00000                         # -NaN
    sp = sp_bits.view(F)
    pos = rng.integers(0, n, max(n // 4, len(sp)))
    keys[pos] = sp[np.arange(pos.shape[0]) % len(sp)]
    return keys


# ---- SIMT convolutions and max pool -------------------------------------------------------------------------------------
def conv64_nhwc(x, w_oihw, stride, pt, pl, ho, wo, groups=1):
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    kh, kw = w_oihw.shape[2:]
    pb = max((ho - 1) * stride + kh - x.shape[1] - pt, 0)
    pr = max((wo - 1) * stride + kw - x.shape[2] - pl, 0)
    xt = torch.nn.functional.pad(xt, (pl, pr, pt, pb))
    y = torch.nn.functional.conv2d(xt, torch.from_numpy(w_oihw.astype(np.float64)), None, stride=stride, groups=groups)
    return y.permute(0, 2, 3, 1).numpy()[:, :ho, :wo]


def fma_chain_ref(x, w_oihw, stride, pt, pl, ho, wo, K, scale, shift, act, groups=1):
    """(float64 output, bound) of a SIMT conv: each output one fixed-order chain of K fmaf from 0, then v*scale and + shift
    rounded once each, then the activation (0 none, 1 ReLU, 2 ReLU6; 1-Lipschitz):
        |got - y64| <= (|scale| gamma_K S + u (|v scale| + |v scale + shift|)) (1 + 4 K u) + 1e-37,  S = sum |x||w|."""
    v = conv64_nhwc(x, w_oihw, stride, pt, pl, ho, wo, groups)
    S = conv64_nhwc(np.abs(x), np.abs(w_oihw), stride, pt, pl, ho, wo, groups)
    sc = np.ones(v.shape[-1]) if scale is None else scale.astype(np.float64)
    a = v * sc
    b = a if shift is None else a + shift.astype(np.float64)
    y = b if act == 0 else np.maximum(b, 0) if act == 1 else np.minimum(np.maximum(b, 0), 6)
    bound = (np.abs(sc) * gamma(K) * S + U * (np.abs(a) + np.abs(b))) * (1 + 4 * K * U) + 1e-37
    return y, bound


def max_pool_model(x, k, stride, pt, pl, ho, wo, pad_neg_inf, zeros_as_ninf=False):
    """max_pool_kernel in numpy: fmaxf from -Inf over the window (a NaN input is dropped, as fmaxf drops it); outside the
    map a cell is skipped (pad_neg_inf) or a 0 (ZEROPAD1).  zeros_as_ninf: the mutant that skips the ZEROPAD1 zeros."""
    n, h, w, c = x.shape
    out = np.full((n, ho, wo, c), -np.inf, F)
    for r in range(k):
        for s in range(k):
            iy = np.arange(ho) * stride - pt + r
            ix = np.arange(wo) * stride - pl + s
            vy, vx = (iy >= 0) & (iy < h), (ix >= 0) & (ix < w)
            v = x[:, np.clip(iy, 0, h - 1)][:, :, np.clip(ix, 0, w - 1)]
            inside = (vy[:, None] & vx[None, :])[None, :, :, None]
            if pad_neg_inf or zeros_as_ninf:
                v = np.where(inside, v, F(-np.inf))
            else:
                v = np.where(inside, v, F(0))
            out = np.fmax(out, v)
    return out


POOL_MODES = ("SAME", "ZEROPAD1", "VALID")


def pool_geometry(h, w, k, stride, mode):
    """engine.py's max_pool arguments for a mode -> (ho, wo, pt, pl, pad_neg_inf)."""
    if mode == "SAME":
        pt = max((-(-h // stride) - 1) * stride + k - h, 0) // 2
        pl = max((-(-w // stride) - 1) * stride + k - w, 0) // 2
        return -(-h // stride), -(-w // stride), pt, pl, True
    if mode == "ZEROPAD1":
        return (h + 2 - k) // stride + 1, (w + 2 - k) // stride + 1, 1, 1, False
    return (h - k) // stride + 1, (w - k) // stride + 1, 0, 0, True


def pool_oracle(x, k, stride, mode):
    from oracle import layers as L
    if mode == "ZEROPAD1":
        return L.max_pool(np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0))), k, stride, "VALID")
    return L.max_pool(x, k, stride, mode)
