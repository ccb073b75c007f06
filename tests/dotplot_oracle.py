"""CPU oracle of `autocycler dotplot` (the reference's dotplot.rs), in two forms:

* literal: the reference's own steps -- get_all_kmer_positions (dotplot.rs:433-450) as dicts of k-mer positions, and the loops of
  create_dotplot (:202-215) and draw_dots (:394-423) in their order, each dot overwriting the pixel it lands on;
* vectorised: every window's forward bytes and reverse-complement bytes numbered with np.unique, the dots of each number formed as
  whole arrays, and each pixel's colour taken from the largest key (a * n + b, j, forward) among its dots, which is the dot the
  literal loops write last.

Both share the layout (get_sizes, between_seq_gap, get_positions, :224-283), the boxes (:286-305), the two passes of create_dotplot
(:184-200) and the labels (reduce_scale, draw_labels, draw_vertical_text, :308-391).  The labels restate the published rules of the
crates the reference draws them with: a TrueType subset (head, hhea, maxp, cmap format 4, hmtx, loca, simple glyf outlines with
implied on-curve midpoints; a composite glyph advances but draws no ink), ab_glyph's advances (advance * px / (ascender - descender),
no kerning), ab_glyph_rasterizer's signed-area coverage with quadratic flattening, and imageproc's draw_text_mut blend -- all in f32.
Without a font no label is drawn and reduce_scale keeps the largest size.  A test checks that the two forms agree.
"""
import math
import struct

import numpy as np

BACKGROUND = (255, 255, 255)
SELF_VS_SELF = (211, 211, 211)
SELF_VS_OTHER = (245, 245, 245)
OUTLINE = (0, 0, 0)
FORWARD = (0, 0, 205)
REVERSE = (178, 34, 34)
U32 = 0xFFFFFFFF


def complement_base(b):                     # misc.rs:324-333
    return {65: 84, 84: 65, 71: 67, 67: 71, 46: 46}.get(b, 78)


def reverse_complement(seq):
    return bytes(complement_base(b) for b in reversed(seq))


def rust_round(x):                          # f64::round: half away from zero (x >= 0 here)
    f = math.floor(x)
    return f + 1.0 if x - f >= 0.5 else f


def as_u32(x):                              # Rust's saturating `as u32` (NaN to 0)
    if x != x or x <= 0:
        return 0
    return U32 if x >= 4294967295.0 else int(x)


def f32(x):
    return float(np.float32(x))


def between_seq_gap(gap, max_total_gap, seq_count):   # :236-246
    if seq_count <= 1:
        return gap
    if (seq_count - 1) * gap > max_total_gap:
        return max_total_gap / (seq_count - 1)
    return gap


def get_sizes(res, seq_count):              # :224-233
    r = float(res)
    return (as_u32(rust_round(0.1 * r)), max(as_u32(rust_round(0.015 * r)), 2),
            max(as_u32(rust_round(between_seq_gap(0.01, 0.1, seq_count) * r)), 2),
            max(as_u32(rust_round(0.0025 * r)), 1), max(as_u32(rust_round(0.025 * r)), 1))


def get_positions(seqs, res, kmer, top_left_gap, bottom_right_gap, between):   # :249-283, u32 arithmetic wrapping
    n = len(seqs)
    lens = [min(max(len(s) - kmer, 0) + 1, U32) for _, _, s in seqs]
    all_gaps = (top_left_gap + bottom_right_gap + between * (n - 1)) & U32
    pixels = max(res - all_gaps, 0)
    if all_gaps > pixels and n > 1:
        between = ((((res // 2) - top_left_gap - bottom_right_gap) & U32) // (n - 1))
        all_gaps = (top_left_gap + bottom_right_gap + between * (n - 1)) & U32
        pixels = max(res - all_gaps, 0)
    total = sum(lens) & U32
    bpp = total / pixels if pixels else (math.inf if total else math.nan)
    starts, ends, cur = [], [], top_left_gap
    for ln in lens:
        starts.append(cur)
        cur = (cur + as_u32(rust_round(ln / bpp) if bpp == bpp else math.nan)) & U32
        ends.append(cur)
        cur = (cur + between) & U32
    return starts, ends, bpp


F = np.float32


class Font:
    """The TrueType subset the labels need, from the file's bytes"""

    def __init__(self, data):
        self.d = data
        n = self.u16(4)
        self.tables = {data[12 + 16 * i:16 + 16 * i].decode("latin-1"): self.u32(12 + 16 * i + 8) for i in range(n)}
        head, hhea, maxp, self.glyf, self.loca, self.hmtx = (self.tables[t] for t in ("head", "hhea", "maxp", "glyf", "loca", "hmtx"))
        self.long_loca = self.s16(head + 50) != 0
        self.n_glyphs = self.u16(maxp + 4)
        self.n_hmetrics = self.u16(hhea + 34)
        if self.n_hmetrics == 0:
            raise ValueError("the font has no horizontal metrics")
        self.ascent, self.descent = F(self.s16(hhea + 4)), F(self.s16(hhea + 6))
        os2 = self.tables.get("OS/2")
        if os2 is not None and self.u16(os2) >= 4 and self.u16(os2 + 62) & 0x80:     # USE_TYPO_METRICS
            self.ascent, self.descent = F(self.s16(os2 + 68)), F(self.s16(os2 + 70))
        cmap = self.tables["cmap"]
        self.cmap4, best = None, 0
        for i in range(self.u16(cmap + 2)):
            pid, eid, off = self.u16(cmap + 4 + 8 * i), self.u16(cmap + 6 + 8 * i), cmap + self.u32(cmap + 8 + 8 * i)
            rank = 2 if (pid, eid) == (3, 1) else 1 if pid == 0 else 0
            if self.u16(off) == 4 and rank > best:
                self.cmap4, best = off, rank

    def u16(self, o):
        return struct.unpack_from(">H", self.d, o)[0]

    def s16(self, o):
        return struct.unpack_from(">h", self.d, o)[0]

    def u32(self, o):
        return struct.unpack_from(">I", self.d, o)[0]

    def glyph_id(self, ch):
        c = ord(ch)
        if self.cmap4 is None or c > 0xFFFF:
            return 0
        b = self.cmap4
        segx2 = self.u16(b + 6)
        ends, starts = b + 14, b + 16 + segx2
        deltas, ranges = starts + segx2, starts + 2 * segx2
        for s in range(0, segx2, 2):
            if c > self.u16(ends + s):
                continue
            start = self.u16(starts + s)
            if c < start:
                return 0
            delta, ro = self.u16(deltas + s), self.u16(ranges + s)
            if ro == 0:
                return (c + delta) & 0xFFFF
            g = self.u16(ranges + s + ro + 2 * (c - start))
            return 0 if g == 0 else (g + delta) & 0xFFFF
        return 0

    def advance(self, g):
        return F(self.u16(self.hmtx + 4 * min(g, self.n_hmetrics - 1)))

    def height(self):
        return F(self.ascent - self.descent)

    def outline(self, g):
        """-> None (no ink) or (x_min, y_min, x_max, y_max, curves); a curve is (p0, control or None, p2), points (x, y) in f32"""
        if g >= self.n_glyphs:
            return None
        a, b = ((self.u32(self.loca + 4 * g), self.u32(self.loca + 4 * g + 4)) if self.long_loca
                else (2 * self.u16(self.loca + 2 * g), 2 * self.u16(self.loca + 2 * g + 2)))
        if b <= a:
            return None
        at = self.glyf + a
        nc = self.s16(at)
        if nc <= 0:
            return None                     # composite: no ink
        bbox = [F(self.s16(at + 2 + 2 * i)) for i in range(4)]
        end_pts = [self.u16(at + 10 + 2 * i) for i in range(nc)]
        n = end_pts[-1] + 1
        p = at + 10 + 2 * nc
        p += 2 + self.u16(p)
        flags = []
        while len(flags) < n:
            f = self.d[p]
            p += 1
            flags.append(f)
            if f & 8:
                r = self.d[p]
                p += 1
                while r and len(flags) < n:
                    flags.append(f)
                    r -= 1
        coords = []
        for short_bit, same_bit in ((2, 16), (4, 32)):
            v, vals = 0, []
            for f in flags:
                if f & short_bit:
                    dv = self.d[p]
                    p += 1
                    v += dv if f & same_bit else -dv
                elif not f & same_bit:
                    v += self.s16(p)
                    p += 2
                vals.append(F(((v + 0x8000) & 0xFFFF) - 0x8000))
            coords.append(vals)
        xs, ys = coords
        curves = []
        state = {"last": None, "move": None}

        def lerp(a, b, t):
            return (F(a[0] + F(t) * F(b[0] - a[0])), F(a[1] + F(t) * F(b[1] - a[1])))

        def move_to(q):
            state["last"] = state["move"] = q

        def line_to(q):
            curves.append((state["last"], None, q))
            state["last"] = q

        def quad_to(c, q):
            curves.append((state["last"], c, q))
            state["last"] = q

        first = 0
        for c in range(nc):
            first_on = first_off = last_off = None
            for i in range(first, end_pts[c] + 1):
                q, on = (xs[i], ys[i]), flags[i] & 1
                if first_on is None:
                    if on:
                        first_on = q
                        move_to(q)
                    elif first_off is not None:
                        mid = lerp(first_off, q, 0.5)
                        first_on, last_off = mid, q
                        move_to(mid)
                    else:
                        first_off = q
                elif last_off is not None and on:
                    quad_to(last_off, q)
                    last_off = None
                elif last_off is not None:
                    prev, last_off = last_off, q
                    quad_to(prev, lerp(prev, q, 0.5))
                elif on:
                    line_to(q)
                else:
                    last_off = q
            if first_off is not None and last_off is not None:
                quad_to(last_off, lerp(last_off, first_off, 0.5))
                last_off = None
            if first_on is not None and first_off is not None:
                quad_to(first_off, first_on)
            elif first_on is not None and last_off is not None:
                quad_to(last_off, first_on)
            elif first_on is not None:
                line_to(first_on)
            if first_on is not None and state["last"] != state["move"]:
                line_to(state["move"])
            first = end_pts[c] + 1
        return (bbox[0], bbox[1], bbox[2], bbox[3], curves) if curves else None


class Raster:
    """ab_glyph_rasterizer: signed-area accumulation, coverage = min(|running sum|, 1) over the buffer in row-major order"""

    def __init__(self, w, h):
        self.w, self.h = w, h
        self.a = [F(0)] * (w * h + 4)

    def add(self, i, v):
        if 0 <= i < len(self.a):
            self.a[i] = F(self.a[i] + v)

    def line(self, p0, p1):
        if abs(F(p0[1] - p1[1])) <= F(1.1920929e-7):
            return
        if p0[1] < p1[1]:
            d = F(1)
        else:
            d, p0, p1 = F(-1), p1, p0
        dxdy = F(F(p1[0] - p0[0]) / F(p1[1] - p0[1]))
        x = p0[0]
        y0 = int(p0[1]) if p0[1] > 0 else 0
        if p0[1] < 0:
            x = F(x - F(p0[1] * dxdy))
        c1 = np.ceil(p1[1])
        yend = min(self.h, int(c1) if c1 > 0 else 0)
        for y in range(y0, yend):
            ls = y * self.w
            dy = F(min(F(y + 1), p1[1]) - max(F(y), p0[1]))
            xnext = F(x + F(dxdy * dy))
            dd = F(dy * d)
            x0, x1 = (x, xnext) if x < xnext else (xnext, x)
            x0floor = np.floor(x0)
            x0i = int(x0floor)
            x1ceil = np.ceil(x1)
            x1i = int(x1ceil)
            if ls + x0i < 0:
                x = xnext
                continue
            if x1i <= x0i + 1:
                xmf = F(F(F(0.5) * F(x + xnext)) - x0floor)
                self.add(ls + x0i, F(dd - F(dd * xmf)))
                self.add(ls + x0i + 1, F(dd * xmf))
            else:
                s = F(F(1) / F(x1 - x0))
                x0f = F(x0 - x0floor)
                a0 = F(F(F(F(0.5) * s) * F(F(1) - x0f)) * F(F(1) - x0f))
                x1f = F(F(x1 - x1ceil) + F(1))
                am = F(F(F(F(0.5) * s) * x1f) * x1f)
                self.add(ls + x0i, F(dd * a0))
                if x1i == x0i + 2:
                    self.add(ls + x0i + 1, F(dd * F(F(F(1) - a0) - am)))
                else:
                    a1 = F(s * F(F(1.5) - x0f))
                    self.add(ls + x0i + 1, F(dd * F(a1 - a0)))
                    for xi in range(x0i + 2, x1i - 1):
                        self.add(ls + xi, F(dd * s))
                    a2 = F(a1 + F(F(x1i - x0i - 3) * s))
                    self.add(ls + x1i - 1, F(dd * F(F(F(1) - a2) - am)))
                self.add(ls + x1i, F(dd * am))
            x = xnext

    def quad(self, p0, p1, p2):
        devx = F(F(p0[0] - F(F(2) * p1[0])) + p2[0])
        devy = F(F(p0[1] - F(F(2) * p1[1])) + p2[1])
        devsq = F(F(devx * devx) + F(devy * devy))
        if devsq < F(0.333):
            self.line(p0, p2)
            return
        n = 1 + int(np.floor(np.sqrt(np.sqrt(F(F(3) * devsq)))))
        p, nrecip, t = p0, F(F(1) / F(n)), F(0)

        def lerp(t, a, b):
            return (F(a[0] + F(t * F(b[0] - a[0]))), F(a[1] + F(t * F(b[1] - a[1]))))
        for _ in range(n - 1):
            t = F(t + nrecip)
            pn = lerp(t, lerp(t, p0, p1), lerp(t, p1, p2))
            self.line(p, pn)
            p = pn
        self.line(p, p2)


def text_width(text, scale, font):          # calculate_text_width (:361-367)
    hf = F(F(scale) / font.height())
    w = F(0)
    for ch in text:
        w = F(w + F(hf * font.advance(font.glyph_id(ch))))
    return w


def draw_text(img, x, y, scale, font, text):
    """imageproc draw_text_mut, black: each glyph's coverage gv blends pixel * (1 - gv) + 0 * gv, truncated to u8"""
    h_img, w_img = img.shape[0], img.shape[1]
    hf = vf = F(F(scale) / font.height())
    ascent = F(vf * font.ascent)
    caret = F(0)
    for ch in text:
        g = font.glyph_id(ch)
        pos = (caret, ascent)
        caret = F(caret + F(hf * font.advance(g)))
        o = font.outline(g)
        if o is None:
            continue
        x_min, y_min, x_max, y_max, curves = o
        minx, miny = np.floor(F(F(x_min * hf) + pos[0])), np.floor(F(F(y_max * -vf) + pos[1]))
        maxx, maxy = np.ceil(F(F(x_max * hf) + pos[0])), np.ceil(F(F(y_min * -vf) + pos[1]))
        bw, bh = F(maxx - minx), F(maxy - miny)
        w, h = (int(bw) if bw > 0 else 0), (int(bh) if bh > 0 else 0)
        off = (F(pos[0] - minx), F(pos[1] - miny))

        def up(q):
            return (F(F(q[0] * hf) + off[0]), F(F(q[1] * -vf) + off[1]))
        r = Raster(w, h)
        for p0, c, p2 in curves:
            if c is None:
                r.line(up(p0), up(p2))
            else:
                r.quad(up(p0), up(c), up(p2))
        xs, ys = x + int(minx), y + int(miny)
        acc = F(0)
        for idx in range(w * h):
            acc = F(acc + r.a[idx])
            gv = min(abs(acc), F(1))
            ix, iy = idx % w + xs, idx // w + ys
            if 0 <= ix < w_img and 0 <= iy < h_img:
                for k in range(3):
                    v = F(F(F(int(img[iy, ix, k])) * F(F(1) - gv)) + F(F(0) * gv))
                    img[iy, ix, k] = 0 if v < 0 else 255 if v > 255 else int(v)


def reduce_scale(seqs, starts, ends, font, max_font_size):   # :308-327 -> (text_height, the LAST sequence's available width)
    text_height = scale = F(max_font_size)
    available = F(1)
    for i, (filename, name, _) in enumerate(seqs):
        available = F((ends[i] - starts[i]) & U32)
        if font is None:
            continue
        tw = max(text_width(filename, scale, font), text_width(name, scale, font))
        if tw > available:
            text_height = F(text_height * F(available / tw))
            scale = text_height
    return text_height, available


def draw_labels(img, seqs, starts, ends, text_gap, font, max_font_size):   # :336-391
    res = img.shape[0]
    min_pos = min(starts)
    text_height, available = reduce_scale(seqs, starts, ends, font, max_font_size)
    dim_w, dim_h = as_u32(float(np.ceil(available))), as_u32(float(text_height))

    def vertical(text, x, y):
        tmp = np.full((dim_h, dim_w, 3), 255, dtype=np.uint8)
        draw_text(tmp, 0, 0, text_height, font, text)
        for i in range(dim_w):
            new_y = (y - i) & U32
            if new_y >= res:
                continue
            for j in range(dim_h):
                new_x = (x + j) & U32
                if new_x < res and tuple(tmp[j, i]) != BACKGROUND:
                    img[new_y, new_x] = tmp[j, i]
    for i, (filename, name, _) in enumerate(seqs):
        pos_1 = (min_pos - text_gap - dim_h) & U32
        pos_2 = (pos_1 - dim_h) & U32
        s32 = lambda v: v - (1 << 32) if v >= 1 << 31 else v
        draw_text(img, starts[i], s32(pos_1), text_height, font, name)
        draw_text(img, starts[i], s32(pos_2), text_height, font, filename)
        vertical(name, pos_1, ends[i])
        vertical(filename, pos_2, ends[i])


def load_font(font):
    if font is None or isinstance(font, Font):
        return font
    return Font(open(font, "rb").read() if isinstance(font, str) else bytes(font))


def layout(seqs, res, kmer, font=None):
    """create_dotplot's two passes (:184-198) -> (starts, ends, bp_per_pixel, text_height)"""
    tlg, border, between, _, max_font = get_sizes(res, len(seqs))
    starts, ends, _ = get_positions(seqs, res, kmer, tlg, border, between)
    text_height, _ = reduce_scale(seqs, starts, ends, font, max_font)
    top_left_gap = as_u32(float(F(F(2) * text_height))) + border
    starts, ends, bpp = get_positions(seqs, res, kmer, top_left_gap, border, between)
    return starts, ends, bpp, float(text_height)


def base_image(seqs, res, kmer, font):
    """background, filled boxes and labels (:189, :199-200) -> (image, starts, ends, bp_per_pixel)"""
    font = load_font(font)
    starts, ends, bpp, _ = layout(seqs, res, kmer, font)
    img = np.full((res, res, 3), 255, dtype=np.uint8)
    draw_boxes(img, starts, ends, True)
    if font is not None:
        draw_labels(img, seqs, starts, ends, get_sizes(res, len(seqs))[3], font, get_sizes(res, len(seqs))[4])
    return img, starts, ends, bpp


def draw_boxes(img, starts, ends, fill):    # :286-305
    res = img.shape[0]
    for a in range(len(starts)):
        l, r = starts[a] - 1, ends[a] + 1
        for b in range(len(starts)):
            t, bo = starts[b] - 1, ends[b] + 1
            if fill:
                img[max(t, 0):min(bo, res - 1) + 1, max(l, 0):min(r, res - 1) + 1] = SELF_VS_SELF if a == b else SELF_VS_OTHER
            for y in (t, bo):
                if 0 <= y < res:
                    img[y, max(l, 0):min(r, res - 1) + 1] = OUTLINE
            for x in (l, r):
                if 0 <= x < res:
                    img[max(t, 0):min(bo, res - 1) + 1, x] = OUTLINE


def pixel(start, pos, bpp):                 # :401, :405
    return (as_u32(rust_round(pos / bpp)) + start) & U32


def get_all_kmer_positions(kmer, seq, rev_comp_seq):   # :433-450
    forward, reverse = {}, {}
    if len(seq) < kmer:
        return forward, reverse
    seq_len = len(seq) - kmer + 1
    for i in range(seq_len):
        forward.setdefault(seq[i:i + kmer], []).append(i)
        reverse.setdefault(rev_comp_seq[i:i + kmer], []).append(seq_len - i - 1)
    return forward, reverse


def _prepare(seqs):
    return [(f, n, bytes(s).upper() if not isinstance(s, str) else s.upper().encode()) for f, n, s in seqs]


def dotplot_literal(seqs, res, kmer, font=None):
    """seqs: [(filename, name, bytes)] -> (res, res, 3) uint8, by the reference's loops.  font: a TrueType file's path or bytes"""
    seqs = _prepare(seqs)
    img, starts, ends, bpp = base_image(seqs, res, kmer, font)
    for ai, (_, _, seq_a) in enumerate(seqs):
        forward, reverse = get_all_kmer_positions(kmer, seq_a, reverse_complement(seq_a))
        for bi, (_, _, seq_b) in enumerate(seqs):
            if len(seq_a) < kmer or len(seq_b) < kmer:
                continue
            for j in range(len(seq_b) - kmer + 1):
                j_pixel = pixel(starts[bi], j, bpp)
                k = seq_b[j:j + kmer]
                for positions, colour in ((reverse.get(k), REVERSE), (forward.get(k), FORWARD)):
                    for i in positions or ():
                        i_pixel = pixel(starts[ai], i, bpp)
                        if i_pixel < res and j_pixel < res:
                            img[j_pixel, i_pixel] = colour
    draw_boxes(img, starts, ends, False)
    return img


def _np_pixels(start, n_windows, bpp):
    pos = np.arange(n_windows, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        v = pos / bpp
    f = np.floor(v)
    r = np.where(v - f >= 0.5, f + 1.0, f)
    r = np.where(np.isnan(r) | (r <= 0), 0.0, np.minimum(r, 4294967295.0))
    return (r.astype(np.uint64) + np.uint64(start)) & np.uint64(U32)


def max_keys(seqs, res, kmer, starts, bpp, chunk=1 << 22):
    """-> a (res * res) uint64 array: each pixel's largest dot key (0: no dot), and the number of dots"""
    n = len(seqs)
    win_f, px, tag = [], [], []
    for s, (_, _, q) in enumerate(seqs):
        nw = len(q) - kmer + 1
        if nw <= 0:
            continue
        a = np.frombuffer(q, dtype=np.uint8)
        w = np.lib.stride_tricks.sliding_window_view(a, kmer)
        win_f.append(w)
        px.append(_np_pixels(starts[s], nw, bpp))
        tag.append((np.uint64(s) << np.uint64(34)) | (np.arange(nw, dtype=np.uint64) << np.uint64(2)) | np.uint64(1))
    best = np.zeros(res * res, dtype=np.uint64)
    if not win_f:
        return best, 0
    F = np.ascontiguousarray(np.concatenate(win_f))
    comp = np.full(256, 78, dtype=np.uint8)
    for x, y in ((65, 84), (84, 65), (71, 67), (67, 71), (46, 46)):
        comp[x] = y
    R = np.ascontiguousarray(comp[F[:, ::-1]])
    px, tag = np.concatenate(px), np.concatenate(tag)
    N = len(F)
    _, ids = np.unique(np.concatenate([F, R]).view(np.dtype((np.void, kmer))).ravel(), return_inverse=True)
    fid, rid = ids[:N].ravel(), ids[N:].ravel()
    seq_of = tag >> np.uint64(34)
    dots = 0
    # forward dots: (u, v) with F[u] == F[v]; reverse dots: (u, v) with R[u] == F[v].  u: row (sequence a, x), v: column (b, j, y)
    order_v = np.argsort(fid, kind="stable")
    fid_sorted = fid[order_v]
    for forward, uid in ((1, fid), (0, rid)):
        order_u = np.argsort(uid, kind="stable")
        uid_sorted = uid[order_u]
        lo = np.searchsorted(fid_sorted, uid_sorted, side="left")
        hi = np.searchsorted(fid_sorted, uid_sorted, side="right")
        cnt = (hi - lo).astype(np.int64)
        keep = cnt > 0
        us, lo, cnt = order_u[keep], lo[keep], cnt[keep]
        total = int(cnt.sum())
        dots += total
        if total == 0:
            continue
        # expand in chunks of rows
        cum = np.cumsum(cnt)
        start_row = 0
        while start_row < len(us):
            base = cum[start_row - 1] if start_row else 0
            end_row = int(np.searchsorted(cum, base + chunk, side="right"))
            end_row = max(end_row, start_row + 1)
            c = cnt[start_row:end_row]
            rows = np.repeat(np.arange(start_row, end_row), c)
            offs = np.arange(int(c.sum())) - np.repeat(np.cumsum(c) - c, c)
            u = us[rows]
            v = order_v[lo[rows] + offs]
            x, y = px[u], px[v]
            ok = (x < res) & (y < res)
            u, v, x, y = u[ok], v[ok], x[ok], y[ok]
            pair = seq_of[u] * np.uint64(n) + seq_of[v]
            key = (pair << np.uint64(34)) | (tag[v] & np.uint64(0x3FFFFFFFD)) | np.uint64(forward << 1)
            np.maximum.at(best, (y * np.uint64(res) + x).astype(np.int64), key)
            start_row = end_row
    return best, dots


def dotplot_vectorised(seqs, res, kmer, font=None):
    """The same image from the per-pixel maximum of the dot keys"""
    seqs = _prepare(seqs)
    img, starts, ends, bpp = base_image(seqs, res, kmer, font)
    best, _ = max_keys(seqs, res, kmer, starts, bpp)
    best = best.reshape(res, res)
    hit = best != 0
    fwd = (best & np.uint64(2)) != 0
    img[hit & fwd] = FORWARD
    img[hit & ~fwd] = REVERSE
    draw_boxes(img, starts, ends, False)
    return img
