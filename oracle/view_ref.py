"""ORACLE — test infrastructure, never the product path.

A numpy statement of the agent's debug view: LAVAgent.visualize (team_code_v2/lav_agent_fast.py:459-518, lidar_to_bev at
:567-581), the frame run_step keeps every tick (:354-358) and flush_data sends to wandb as a 20 fps video (:160-167).  It is
the contract lavb_agent_view (include/lav_b200.h) is tested against.  ``frame`` is steps 1-4 of visualize (the LiDAR BEV,
the drawing on it, the predicted BEV, the two resizes); ``annotate`` is step 5, the reference's four cv2.putText calls.

The OpenCV primitives visualize calls are restated here and checked against cv2 (4.13) by tests/test_agent_view_cpu.py:
  * cv2.resize, INTER_LINEAR on 8-bit images (``resize``): per output column / row the source index and the weight
    f = float32((d + 0.5) / (dst / src) - 0.5) - floor, the 11-bit coefficients rint((1 - f) * 2048) and rint(f * 2048)
    taken separately, columns clamped to the image, a horizontal pass in int32 and the vertical pass
    (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2 over rows clamped to the image;
  * cv2.circle, filled, LINE_8 (``circle``): radius 1 is a plus, radius 2 a 13-pixel diamond, clipped to the image;
  * cv2.drawContours with thickness 2 (``thick_polyline``): per segment, the end points are clipped to the image grown by the
    thickness (clipLine on the rectangle (-2, -2, W + 4, H + 4)); the segment is a 16.16 fixed-point quad filled by
    FillConvexPoly (its outline drawn by the fixed-point line walker, then the scanlines) and capped by a radius-1 circle at
    its end point.

Where this statement departs from the reference (the GPU view does the same):
  * a plan or forecast point, or a target, that is NaN or whose pixel falls outside int32 is not drawn (visualize raises
    there: cv2 cannot parse the centre); likewise a vehicle box whose corners are not finite or fall outside int32;
  * the target and the text are built from the values the port holds: its targets and controls are fp32 where the reference
    holds fp64;
  * the predicted BEV's sigmoid is taken on the fp32 logits (16-bit logits are widened first), as torch.sigmoid takes it on the
    device; a NaN mean gives 0.
"""
import numpy as np

H = W = 320                                   # the LiDAR view: (max_x - min_x) * pixels_per_meter
EGO = (160, 280)                              # visualize's ego pixel (x, y)
XBINS = np.linspace(-10, 71, 321)             # lidar_to_bev's edges: max_x + 1 and max_y + 1 as the reference writes them
YBINS = np.linspace(-40, 41, 321)
HIST_MAX = 10
CAM_W, TEL_W = 853, 800                       # int(768 / 288 * 320), int(480 / 192 * 320)
CANVAS_W = CAM_W + TEL_W + W + W              # 2293
OUT_H, OUT_W = 160, 1146                      # the canvas halved, int() of each side
PLAN_COLOR, BOX_COLOR, TARGET_COLOR = (255, 0, 0), (255, 0, 0), (0, 255, 0)
CMD_NAMES = {0: 'left', 1: 'right', 2: 'straight', 3: 'follow', 4: 'change left', 5: 'change right'}
XY_SHIFT, XY_ONE = 16, 1 << 16
INT32 = (-2 ** 31, 2 ** 31 - 1)

# matplotlib's _jet_data (x, y0, y1 per segment)
_JET = {
    "red": ((0., 0, 0), (0.35, 0, 0), (0.66, 1, 1), (0.89, 1, 1), (1, 0.5, 0.5)),
    "green": ((0., 0, 0), (0.125, 0, 0), (0.375, 1, 1), (0.64, 1, 1), (0.91, 0, 0), (1, 0, 0)),
    "blue": ((0., 0.5, 0.5), (0.11, 1, 1), (0.34, 1, 1), (0.65, 0, 0), (1, 0, 0)),
}
JET_N = 256


def _lookup_table(n, data):
    """matplotlib.colors._create_lookup_table(n, data, gamma=1)."""
    a = np.array(data, dtype=np.float64)
    x, y0, y1 = a[:, 0] * (n - 1), a[:, 1], a[:, 2]
    xind = (n - 1) * np.linspace(0, 1, n) ** 1.0
    ind = np.searchsorted(x, xind)[1:-1]
    distance = (xind[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    lut = np.concatenate([[y1[0]], distance * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]])
    return np.clip(lut, 0.0, 1.0)


def jet_rgba():
    """matplotlib's jet as LinearSegmentedColormap('jet', _jet_data, 256)._lut after _init: 256 colours, then the under, over
    and bad (NaN) entries (the first colour, the last colour, transparent black)."""
    lut = np.ones((JET_N + 3, 4))
    for j, ch in enumerate(("red", "green", "blue")):
        lut[:-3, j] = _lookup_table(JET_N, _JET[ch])
    lut[JET_N] = lut[0]
    lut[JET_N + 1] = lut[JET_N - 1]
    lut[JET_N + 2] = 0.0
    return lut


def jet_index(score):
    """the row of jet_rgba() Colormap.__call__ reads for an fp32 score: x * N in fp32, N -> N - 1, under / over / bad rows,
    then truncation."""
    xa = np.array(score, dtype=np.float32, copy=True)
    xa *= np.float32(JET_N)
    xa[xa == JET_N] = JET_N - 1
    under, over, bad = xa < 0, xa >= JET_N, np.isnan(xa)
    with np.errstate(invalid="ignore"):
        idx = xa.astype(np.int64)
    idx[under], idx[over], idx[bad] = JET_N, JET_N + 1, JET_N + 2
    return idx


def jet_bytes():
    """(259, 3) uint8: visualize's (int(r * 255), int(g * 255), int(b * 255)) of every row of jet_rgba()."""
    return (jet_rgba()[:, :3] * 255).astype(np.int64).astype(np.uint8)


# ---- step 1: the LiDAR BEV ------------------------------------------------------------------------------------------------
def hist_bins(v, edges):
    """np.histogramdd's bin of each value along one axis: searchsorted(side='right') on the fp64 edges, the last edge moved
    into the last bin; -1 for NaN, +-inf and anything outside the edges."""
    v = np.asarray(v, dtype=np.float64)
    n = np.searchsorted(edges, v, side="right")
    n[v == edges[-1]] -= 1
    b = n - 1
    b[(n < 1) | (n > len(edges) - 1) | np.isnan(v)] = -1
    return b


def lidar_counts(points):
    """(320, 320) int64 histogram of the points' (x, y), rows x bins, columns y bins (not yet flipped)."""
    pts = np.asarray(points, dtype=np.float32).reshape(-1, np.asarray(points).shape[-1])
    bx, by = hist_bins(pts[:, 0], XBINS), hist_bins(pts[:, 1], YBINS)
    ok = (bx >= 0) & (by >= 0)
    c = np.zeros((H, W), np.int64)
    np.add.at(c, (bx[ok], by[ok]), 1)
    return c


def grey_of_count():
    """the grey of a bin holding c points, c = 0 .. 10: min(c, 10) / 10 * 255 in fp64, truncated."""
    return (np.arange(HIST_MAX + 1, dtype=np.float64) / HIST_MAX * 255.).astype(np.uint8)


def lidar_bev(points):
    """lidar_to_bev(...).astype(uint8) as a (320, 320) grey image, rows flipped."""
    c = np.minimum(lidar_counts(points), HIST_MAX)
    return grey_of_count()[c][::-1, :]


# ---- step 2: the drawing --------------------------------------------------------------------------------------------------
_STENCIL = {1: [(0, 0), (-1, 0), (1, 0), (0, -1), (0, 1)],
            2: [(dx, dy) for dy in range(-2, 3) for dx in range(-2, 3) if abs(dx) + abs(dy) <= 2]}


def circle(img, cx, cy, r, color):
    """cv2.circle(img, (cx, cy), r, color, -1) for r = 1, 2."""
    h, w = img.shape[:2]
    for dx, dy in _STENCIL[r]:
        x, y = cx + dx, cy + dy
        if 0 <= x < w and 0 <= y < h:
            img[y, x] = color


def _cdiv(a, b):
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def clip_line(w, h, x1, y1, x2, y2):
    """OpenCV's clipLine on the int64 rectangle (0, 0, w, h): (inside, x1, y1, x2, y2)."""
    right, bottom = w - 1, h - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1, c1 = a, 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2, c2 = a, 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def _line_fixed(px, w, h, p1, p2):
    """the 16.16 fixed-point line walker FillConvexPoly outlines with (8-connected); pixels into the set px, not yet clipped to
    the image."""
    ok, x1, y1, x2, y2 = clip_line(w << XY_SHIFT, h << XY_SHIFT, *p1, *p2)
    if not ok:
        return
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:
            x1, x2, y1, y2, dy = x2, x1, y2, y1, -dy
        step = _cdiv(dy << XY_SHIFT, ax | 1)
        n = (x2 - x1) >> XY_SHIFT
    else:
        if dy < 0:
            x1, x2, y1, y2, dx = x2, x1, y2, y1, -dx
        step = _cdiv(dx << XY_SHIFT, ay | 1)
        n = (y2 - y1) >> XY_SHIFT
    px.add(((x2 + (XY_ONE >> 1)) >> XY_SHIFT, (y2 + (XY_ONE >> 1)) >> XY_SHIFT))
    x1 += XY_ONE >> 1
    y1 += XY_ONE >> 1
    if ax > ay:
        x1 >>= XY_SHIFT
        for _ in range(n + 1):
            px.add((x1, y1 >> XY_SHIFT))
            x1, y1 = x1 + 1, y1 + step
    else:
        y1 >>= XY_SHIFT
        for _ in range(n + 1):
            px.add((x1 >> XY_SHIFT, y1))
            x1, y1 = x1 + step, y1 + 1


def _fill_convex(px, w, h, v):
    """FillConvexPoly of the 16.16 fixed-point polygon v (LINE_8): outline, then the scanlines between its two edges."""
    n, delta = len(v), XY_ONE >> 1
    xs_, ys_ = [p[0] for p in v], [p[1] for p in v]
    imin = int(np.argmin(ys_))
    for i in range(n):
        _line_fixed(px, w, h, v[i - 1], v[i])
    xmin, xmax = (min(xs_) + delta) >> XY_SHIFT, (max(xs_) + delta) >> XY_SHIFT
    ymin, ymax = (min(ys_) + delta) >> XY_SHIFT, (max(ys_) + delta) >> XY_SHIFT
    if n < 3 or xmax < 0 or ymin >= h or xmin >= w:
        return
    ymax = min(ymax, h - 1)
    edges = n
    e = [[imin, 1, -XY_ONE, 0, ymin], [imin, n - 1, -XY_ONE, 0, ymin]]   # idx, di, x, dx, ye
    y = ymin
    while True:
        for ed in e:
            if y >= ed[4]:
                idx0 = ed[0]
                idx = (idx0 + ed[1]) % n
                while True:
                    edges -= 1
                    if edges < 0:
                        break
                    ty = (v[idx][1] + delta) >> XY_SHIFT
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        ed[4] = ty
                        ed[3] = _cdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        ed[2] = xs
                        ed[0] = idx
                        break
                    idx0, idx = idx, (idx + ed[1]) % n
        if edges < 0:
            break
        if y >= 0:
            l, r = (e[1], e[0]) if e[0][2] > e[1][2] else (e[0], e[1])
            x1, x2 = (l[2] + delta) >> XY_SHIFT, (r[2] + delta) >> XY_SHIFT
            if x2 >= 0 and x1 < w:
                px.update((x, y) for x in range(max(x1, 0), min(x2, w - 1) + 1))
        e[0][2] += e[0][3]
        e[1][2] += e[1][3]
        y += 1
        if y > ymax:
            break


def thick_segment_pixels(w, h, p0, p1):
    """the pixels ThickLine (thickness 2, LINE_8) writes for one contour segment p0 -> p1, with the cap at p1 only."""
    px = set()
    ok, x1, y1, x2, y2 = clip_line(w + 4, h + 4, p0[0] + 2, p0[1] + 2, p1[0] + 2, p1[1] + 2)
    if not ok:
        return px
    a = ((x1 - 2) << XY_SHIFT, (y1 - 2) << XY_SHIFT)
    b = ((x2 - 2) << XY_SHIFT, (y2 - 2) << XY_SHIFT)
    dx, dy = (a[0] - b[0]) * (1.0 / XY_ONE), (b[1] - a[1]) * (1.0 / XY_ONE)
    rr = dx * dx + dy * dy
    if abs(rr) > np.finfo(np.float64).eps:
        r = XY_ONE / np.sqrt(rr)
        ex, ey = int(np.rint(dy * r)), int(np.rint(dx * r))
        _fill_convex(px, w, h, [(a[0] + ex, a[1] + ey), (a[0] - ex, a[1] - ey), (b[0] - ex, b[1] - ey), (b[0] + ex, b[1] + ey)])
    px.update((x2 - 2 + ox, y2 - 2 + oy) for ox, oy in _STENCIL[1])
    return {(x, y) for x, y in px if 0 <= x < w and 0 <= y < h}


def thick_polyline(img, pts, color):
    """cv2.drawContours(img, np.array([pts]), 0, color, 2) for one closed contour of int points."""
    h, w = img.shape[:2]
    for j in range(len(pts)):
        for x, y in thick_segment_pixels(w, h, pts[j - 1], pts[j]):
            img[y, x] = color


def point_pixel(loc, ppm):
    """(ego + loc * ppm).astype(int): loc * ppm in fp32, the sum in fp64, truncated; None when NaN or outside int32."""
    v = np.asarray(loc, dtype=np.float32) * np.float32(ppm)
    p = np.array(EGO, dtype=np.int64) + v.astype(np.float64)
    if not np.isfinite(p).all() or (p <= INT32[0] - 1).any() or (p >= INT32[1] + 1).any():
        return None
    return int(p[0]), int(p[1])


def box_corners(box):
    """visualize's four corners of a vehicle box (x, y, w, h, cos, sin), fp64, truncated; None when not finite or outside
    int32."""
    x, y, ww, hh, cos, sin = (float(v) for v in box)
    m = ((-sin, cos), (-cos, -sin))
    out = []
    for sw, sh in ((-ww, -hh), (-ww, hh), (ww, hh), (ww, -hh)):
        cx = x + (sw * m[0][0] + sh * m[1][0])
        cy = y + (sw * m[0][1] + sh * m[1][1])
        if not (np.isfinite(cx) and np.isfinite(cy)) or not all(INT32[0] - 1 < c < INT32[1] + 1 for c in (cx, cy)):
            return None
        out.append((int(cx), int(cy)))
    return out


def target_pixel(tgt, ppm):
    """np.clip(ego + tgt * ppm, 0, 255).astype(int) in fp64; None when NaN."""
    p = np.clip(np.array(EGO, dtype=np.int64) + np.asarray(tgt, dtype=np.float64) * ppm, 0, 255)
    if np.isnan(p).any():
        return None
    return int(p[0]), int(p[1])


def draw(img, plan, cast_locs, cast_cmds, boxes, tgt, ppm, cmd_thresh):
    """step 2 on the (320, 320, 3) LiDAR image, in place, in visualize's order."""
    for loc in plan:
        p = point_pixel(loc, ppm)
        if p is not None:
            circle(img, *p, 1, PLAN_COLOR)
    jet = jet_bytes()
    for trajs, cmds in zip(cast_locs, cast_cmds):
        for traj, score in zip(trajs, np.asarray(cmds, dtype=np.float32)):
            if score < cmd_thresh:
                continue
            color = tuple(int(c) for c in jet[int(jet_index(score))])
            for loc in traj:
                p = point_pixel(loc, ppm)
                if p is not None:
                    circle(img, *p, 1, color)
    for box in boxes:
        pts = box_corners(box)
        if pts is not None:
            thick_polyline(img, pts, BOX_COLOR)
    p = target_pixel(tgt, ppm)
    if p is not None:
        circle(img, *p, 2, TARGET_COLOR)
    return img


# ---- steps 3-4: the predicted BEV and the canvas --------------------------------------------------------------------------
def bev_mean(sig):
    """(255 * p.mean(axis=0)).astype(uint8) of the fp32 sigmoid p (C, 320, 320): channels summed in order, divided by C, all
    fp32; NaN gives 0."""
    p = np.asarray(sig, dtype=np.float32)
    s = p[0].copy()
    for c in range(1, p.shape[0]):
        s = s + p[c]
    v = np.float32(255) * (s / np.float32(p.shape[0]))
    v = np.where(np.isnan(v), np.float32(0), v)
    return v.astype(np.uint8)


def _axis(src, dst, clamp):
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * (1.0 / (dst / src)) - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        lo, hi = s < 0, s >= src - 1
        f[lo | hi] = 0
        s[lo], s[hi] = 0, src - 1
    c0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    c1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return s, c0, c1


def resize(img, w, h):
    """cv2.resize(img, (w, h)) for an 8-bit (H, W, C) image, INTER_LINEAR."""
    sh, sw = img.shape[:2]
    sx, a0, a1 = _axis(sw, w, True)
    sy, b0, b1 = _axis(sh, h, False)
    im = img.astype(np.int64)
    rows = im[:, sx] * a0[None, :, None] + im[:, np.minimum(sx + 1, sw - 1)] * a1[None, :, None]
    s0, s1 = rows[np.clip(sy, 0, sh - 1)], rows[np.clip(sy + 1, 0, sh - 1)]
    v = (((b0[:, None, None] * (s0 >> 4)) >> 16) + ((b1[:, None, None] * (s1 >> 4)) >> 16) + 2) >> 2
    return v.astype(np.uint8)


def frame(rgb, tel, points, sig_bev, plan, cast_locs, cast_cmds, boxes, tgt, ppm=4, cmd_thresh=0.2):
    """visualize's canvas before the text: (160, 1146, 3) uint8.
    rgb (288, 768, 3) the three cameras side by side; tel (192, 480, 3); points (n, >=2) fp32, NaN rows allowed; sig_bev
    (C, 320, 320) fp32 sigmoid of pred_bev; plan (T, 2) fp32 (the plan after the 4/5 swap); cast_locs (K, M, T, 2) /
    cast_cmds (K, M) fp32; boxes [(x, y, w, h, cos, sin)]; tgt (2,) the target [-wx, -wy]."""
    lidar = np.repeat(lidar_bev(points)[..., None], 3, axis=2)
    draw(lidar, plan, cast_locs, cast_cmds, boxes, tgt, ppm, cmd_thresh)
    bev = np.repeat(bev_mean(sig_bev)[..., None], 3, axis=2)
    canvas = np.concatenate([resize(rgb, CAM_W, H), resize(tel, TEL_W, H), lidar, bev], axis=1)
    return resize(canvas, OUT_W, OUT_H)


def annotate(canvas, spd, cmd, steer, throt, brake, pred_bra):
    """step 5 in place: visualize's four cv2.putText lines, from the values as given."""
    import cv2
    args = (cv2.FONT_HERSHEY_SIMPLEX, 0.3, (255, 255, 255), 1)
    cv2.putText(canvas, f'speed: {spd:.3f}m/s', (4, 10), *args)
    cv2.putText(canvas, 'cmd: {}'.format(CMD_NAMES.get(cmd)), (4, 30), *args)
    cv2.putText(canvas, f'steer: {steer:.3f} throttle: {throt:.3f} brake: {brake:.3f}', (4, 20), *args)
    cv2.putText(canvas, f'predicted brake: {pred_bra:.3f}', (4, 40), *args)
    return canvas


# ---- seeded cases (oracle/pin_view.py, tests) ------------------------------------------------------------------------------
def _smooth_image(rng, h, w):
    """a camera-like uint8 RGB image that compresses well in the golden: a flat background and a few flat blocks, whose edges
    the resizes interpolate."""
    img = np.empty((h, w, 3), np.uint8)
    img[:] = rng.integers(0, 256, 3)
    for _ in range(12):
        y0, x0 = rng.integers(0, h - 8), rng.integers(0, w - 8)
        img[y0:y0 + rng.integers(4, 80), x0:x0 + rng.integers(4, 80)] = rng.integers(0, 256, 3)
    return img


def view_case(seed, kind, num_cmds=6, steps=20, channels=4):
    """one seeded input of visualize (the values as the port holds them): kind names what the case exercises."""
    rng = np.random.default_rng([seed, len(kind), sum(map(ord, kind))])
    n = 3000 if kind != "saturated" else 20000
    pts = np.concatenate([rng.uniform([-12, -42, -3, 0], [73, 43, 2, 1], (n, 4)),
                          rng.normal([15, 0, 0, 0.5], [6, 4, 1, 0.2], (n // 2, 4))]).astype(np.float32)
    if kind == "saturated":
        pts[:n // 2, :2] = rng.normal([20, 0], [0.3, 0.3], (n // 2, 2))
    if kind == "edges":          # exactly on bin edges (fp32 of the fp64 edge), one ulp either side, and on the last edge
        e = np.concatenate([XBINS.astype(np.float32)[:, None], YBINS.astype(np.float32)[:, None]], 1)
        on = np.concatenate([e, np.nextafter(e, np.float32(np.inf)), np.nextafter(e, -np.float32(np.inf)),
                             np.float32([[71, 41], [71, 0], [0, 41], [-10, -40]])])
        pts = np.concatenate([pts, np.concatenate([on, np.zeros((len(on), 2), np.float32)], 1)])
    sig = np.stack([(np.sin(np.mgrid[0:H, 0:W][0] / rng.uniform(5, 40) + rng.uniform(0, 6)) + 1) / 2
                    * rng.uniform(0.5, 1) for _ in range(channels)]).astype(np.float32)
    plan = np.cumsum(rng.normal([0, -1.2], [0.3, 0.4], (steps, 2)), 0).astype(np.float32)
    if kind == "plan_off":
        plan *= np.float32(40)
    k = {"empty": 0, "full": 15}.get(kind, int(rng.integers(1, 6)))
    boxes = []
    for _ in range(k):
        x, y = (int(v) for v in rng.integers(-10, 330, 2)) if kind == "boxes_off" else (int(v) for v in rng.integers(20, 300, 2))
        a = rng.uniform(0, 2 * np.pi)
        boxes.append((x, y, float(np.float32(rng.uniform(1, 12))), float(np.float32(rng.uniform(1, 12))),
                      float(np.float32(np.cos(a))), float(np.float32(np.sin(a)))))
    starts = np.array([[b[0] - EGO[0], b[1] - EGO[1]] for b in boxes], np.float32).reshape(k, 1, 1, 2) / np.float32(4)
    cast = (starts + np.cumsum(rng.normal(0, 0.6, (k, num_cmds, steps, 2)), 2)).astype(np.float32)
    cmds = rng.uniform(0, 1, (k, num_cmds)).astype(np.float32)
    if kind == "thresh" and k:
        t = np.float32(0.2)
        cmds[:, :3] = [np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1))]
    if kind == "scores_top" and k:
        cmds[:, :3] = [1.0, np.nextafter(np.float32(1), np.float32(0)), 1.5]
    tgt = rng.normal(0, 8, 2).astype(np.float32)
    if kind == "target_far":
        tgt = np.float32([30.0, -75.0])
    cmd = {"cmd4": 4, "cmd5": 5}.get(kind, int(rng.integers(0, 4)))
    return dict(rgb=_smooth_image(rng, 288, 768), tel=_smooth_image(rng, 192, 480), points=pts, sig_bev=sig, plan=plan,
                cast_locs=cast, cast_cmds=cmds, boxes=boxes, tgt=tgt, cmd=cmd, spd=float(np.float32(rng.uniform(0, 9))),
                steer=float(np.float32(rng.uniform(-1, 1))), throt=float(np.float32(rng.uniform(0, 0.75))),
                brake=float(np.float32(rng.integers(0, 2))), pred_bra=float(np.float32(rng.uniform(0, 1))))


VIEW_KINDS = ("empty", "full", "thresh", "boxes_off", "target_far", "edges", "cmd4", "cmd5", "scores_top", "saturated",
              "plan_off", "plain")


def case_frame(c, ppm=4, cmd_thresh=0.2):
    """frame() + annotate() of a view_case."""
    f = frame(c["rgb"], c["tel"], c["points"], c["sig_bev"], c["plan"], c["cast_locs"], c["cast_cmds"], c["boxes"], c["tgt"],
              ppm, cmd_thresh)
    return annotate(f, c["spd"], c["cmd"], c["steer"], c["throt"], c["brake"], c["pred_bra"])
