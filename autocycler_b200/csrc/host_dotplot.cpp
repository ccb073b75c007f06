// `autocycler dotplot` on the host (see host_dotplot.h).  Citations are file:line in the reference's src/.
#include "host_dotplot.h"

#include <sys/stat.h>
#include <zlib.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <set>
#include <unordered_map>

#include "host_graph.h"
#include "host_io.h"

static void fail(const std::string& m) { throw InputError{m}; }

void dotplot_check_settings(uint32_t res, uint32_t kmer) {       // dotplot.rs:55-60
    if (res < 500) fail("--res cannot be less than 500");
    if (res > 10000) fail("--res cannot be greater than 10000");
    if (kmer < 10) fail("--kmer cannot be less than 10");
    if (kmer > 100) fail("--kmer cannot be greater than 100");
}

// The whole file, gunzipped when it is gzipped (zlib reads a plain file as it is).
static bool read_any(const std::string& path, std::string& out) {
    gzFile g = gzopen(path.c_str(), "rb");
    if (!g) return false;
    std::vector<char> buf(1 << 20);
    int n;
    out.clear();
    while ((n = gzread(g, buf.data(), (unsigned)buf.size())) > 0) out.append(buf.data(), (size_t)n);
    gzclose(g);
    return n >= 0;
}

// first_char_in_file (misc.rs:474-506): the first character of the first non-empty line; 0 when there is none
static char first_char(const std::string& text) {
    size_t pos = 0;
    while (pos < text.size()) {
        size_t eol = text.find('\n', pos);
        if (eol == std::string::npos) eol = text.size();
        size_t end = eol;
        if (end > pos && text[end - 1] == '\r') --end;
        if (end > pos) return text[pos];
        pos = eol + 1;
    }
    return 0;
}

static std::string upper(std::string s) { for (char& c : s) if (c >= 'a' && c <= 'z') c = (char)(c - 32); return s; }
static std::string base_name(const std::string& path) { const size_t s = path.find_last_of('/'); return s == std::string::npos ? path : path.substr(s + 1); }
static char complement(char b) { return b == 'A' ? 'T' : b == 'T' ? 'A' : b == 'G' ? 'C' : b == 'C' ? 'G' : b == '.' ? '.' : 'N'; }   // misc.rs:324-333

std::vector<DotplotInput> dotplot_load(const std::string& input, bool verbose) {
    std::vector<DotplotInput> seqs;
    struct stat st;
    const bool exists = stat(input.c_str(), &st) == 0;
    if (exists && S_ISDIR(st.st_mode)) {                                      // load_from_directory (:161-176)
        if (verbose) fprintf(stderr, "\nLoading sequences\n    Sequences are now loaded from FASTA files in the provided directory.\n\n");
        for (const std::string& path : find_all_assemblies(input)) {
            const std::string filename = base_name(path);
            for (FastaRecord& r : load_fasta(path)) {
                if (verbose) fprintf(stderr, "%s %s (%zu bp)\n", filename.c_str(), r.name.c_str(), r.seq.size());
                seqs.push_back(DotplotInput{filename, r.name, std::move(r.seq)});
            }
        }
    } else {
        if (!exists || !S_ISREG(st.st_mode)) fail("--input is neither a file nor a directory");   // :66-71
        std::string text;
        if (!read_any(input, text)) fail("unable to load " + input);
        const char c = first_char(text);
        if (c == '>') {                                                       // load_from_fasta (:147-158)
            if (verbose) fprintf(stderr, "\nLoading sequences\n    Sequences are now loaded from the provided FASTA file.\n\n");
            for (FastaRecord& r : load_fasta(input)) {
                if (verbose) fprintf(stderr, "%s (%zu bp)\n", r.name.c_str(), r.seq.size());
                seqs.push_back(DotplotInput{std::string(), r.name, std::move(r.seq)});
            }
        } else if (c == 'H' || c == 'S') {                                    // load_from_graph + reconstruct_original_sequences_u8 (:135-144)
            if (verbose) fprintf(stderr, "\nLoading sequences\n    Sequences are now loaded from the provided unitig graph.\n\n");
            HostGraph g; std::vector<HostSeq> hs;
            try { g.load_gfa(text.data(), text.size(), hs); }
            catch (const std::runtime_error& e) { fail(e.what()); }
            for (size_t i = 0; i < hs.size(); ++i) {
                std::string s;
                for (uint64_t x = g.path_off[i]; x < g.path_off[i + 1]; ++x) {   // get_sequence_from_path (unitig_graph.rs:390-400)
                    const UStrand u = g.path[x]; const uint32_t n = g.rec[us_index(u)].len; const char* src = g.seq_ptr(us_index(u));
                    if (!us_reverse(u)) s.append(src, n);
                    else for (uint32_t j = 0; j < n; ++j) s.push_back(complement(src[n - 1 - j]));
                }
                if (s.size() != hs[i].length) fail("reconstructed sequence does not have expected length");
                const std::string& h = hs[i].contig_header;                   // contig_name(): up to the first space (sequence.rs:77-79)
                const size_t sp = h.find(' ');
                if (verbose) fprintf(stderr, "%u: %s %s (%llu bp)\n", (unsigned)hs[i].id, hs[i].filename.c_str(), h.c_str(), (unsigned long long)hs[i].length);
                seqs.push_back(DotplotInput{hs[i].filename, sp == std::string::npos ? h : h.substr(0, sp), std::move(s)});
            }
            for (DotplotInput& d : seqs) d.seq = upper(std::move(d.seq));
            std::sort(seqs.begin(), seqs.end(), [](const DotplotInput& a, const DotplotInput& b) {
                if (a.filename != b.filename) return a.filename < b.filename;
                if (a.name != b.name) return a.name < b.name;
                return a.seq < b.seq;
            });
        } else {
            fail("--input is neither GFA or FASTA");
        }
    }
    if (seqs.empty()) fail("no sequences were loaded");                     // :128-130
    if (verbose) fprintf(stderr, "\n");
    for (DotplotInput& d : seqs) d.seq = upper(std::move(d.seq));
    std::set<std::pair<std::string, std::string>> seen;
    for (const DotplotInput& d : seqs)       // the reference keys its boxes by (filename, name): two such sequences would share one box
        if (!seen.insert({d.filename, d.name}).second) fail("two sequences are named " + (d.filename.empty() ? d.name : d.filename + " " + d.name));
    return seqs;
}

// ---- layout (dotplot.rs:224-283) --------------------------------------------------------------------------------------------------
static uint32_t sat_u32(double v) { return !(v > 0.0) ? 0u : v >= 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)v; }   // Rust's `as u32`
static uint32_t sat_u32f(float v) { return !(v > 0.0f) ? 0u : v >= 4294967295.0f ? 0xFFFFFFFFu : (uint32_t)v; }

static double between_seq_gap(double gap, double max_total_gap, size_t seq_count) {   // :236-246
    if (seq_count <= 1) return gap;
    if ((double)(seq_count - 1) * gap > max_total_gap) return max_total_gap / (double)(seq_count - 1);
    return gap;
}

struct Sizes { uint32_t top_left_gap, border_gap, between_seq_gap, text_gap, max_font_size; };
static Sizes get_sizes(uint32_t res_u, size_t seq_count) {                     // :224-233
    const double res = res_u;
    Sizes s;
    s.top_left_gap = sat_u32(std::round(0.1 * res));
    s.border_gap = std::max(sat_u32(std::round(0.015 * res)), 2u);
    s.between_seq_gap = std::max(sat_u32(std::round(between_seq_gap(0.01, 0.1, seq_count) * res)), 2u);
    s.text_gap = std::max(sat_u32(std::round(0.0025 * res)), 1u);
    s.max_font_size = std::max(sat_u32(std::round(0.025 * res)), 1u);
    return s;
}

struct Positions { std::vector<uint32_t> start, end; double bpp; };
// :249-283, u32 arithmetic wrapping as in the reference's release build
static Positions get_positions(const std::vector<DotplotInput>& seqs, uint32_t res, uint32_t kmer, uint32_t top_left_gap, uint32_t bottom_right_gap,
                               uint32_t between) {
    const uint32_t n = (uint32_t)seqs.size();
    std::vector<uint32_t> len(n);
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t l = (uint32_t)seqs[i].seq.size(), d = l > kmer ? l - kmer : 0u;
        len[i] = d == 0xFFFFFFFFu ? d : d + 1;
    }
    uint32_t all_gaps = top_left_gap + bottom_right_gap + between * (n - 1);
    uint32_t pixels = res > all_gaps ? res - all_gaps : 0u;
    if (all_gaps > pixels && n > 1) {                                          // not enough room: shrink the gaps (boxes may touch)
        between = ((res / 2) - top_left_gap - bottom_right_gap) / (n - 1);
        all_gaps = top_left_gap + bottom_right_gap + between * (n - 1);
        pixels = res > all_gaps ? res - all_gaps : 0u;
    }
    uint32_t total = 0;
    for (uint32_t l : len) total += l;
    Positions p;
    p.bpp = (double)total / (double)pixels;
    uint32_t cur = top_left_gap;
    for (uint32_t i = 0; i < n; ++i) {
        p.start.push_back(cur);
        cur += sat_u32(std::round((double)len[i] / p.bpp));
        p.end.push_back(cur);
        cur += between;
    }
    return p;
}

// ---- drawing (imageproc draw_filled_rect_mut / draw_hollow_rect_mut, clipped to the image) ----------------------------------------
static void put(std::vector<uint8_t>& img, uint32_t res, int64_t x, int64_t y, const uint8_t c[3]) {
    if (x < 0 || y < 0 || x >= res || y >= res) return;
    uint8_t* p = &img[((uint64_t)y * res + (uint64_t)x) * 3];
    p[0] = c[0]; p[1] = c[1]; p[2] = c[2];
}
static const uint8_t OUTLINE[3] = {0, 0, 0}, SELF_VS_SELF[3] = {211, 211, 211}, SELF_VS_OTHER[3] = {245, 245, 245};   // :35-41

// draw_sequence_boxes (:286-305): box (a, b) spans [start - 1, end + 2) on both axes; outline = its edge pixels
static void draw_boxes(std::vector<uint8_t>& img, uint32_t res, const Positions& p, bool fill) {
    const size_t n = p.start.size();
    for (size_t a = 0; a < n; ++a) {
        const int64_t l = (int64_t)p.start[a] - 1, r = (int64_t)p.end[a] + 1;
        for (size_t b = 0; b < n; ++b) {
            const int64_t t = (int64_t)p.start[b] - 1, bo = (int64_t)p.end[b] + 1;
            if (fill) {
                const uint8_t* c = a == b ? SELF_VS_SELF : SELF_VS_OTHER;
                for (int64_t y = std::max<int64_t>(t, 0); y <= std::min<int64_t>(bo, (int64_t)res - 1); ++y)
                    for (int64_t x = std::max<int64_t>(l, 0); x <= std::min<int64_t>(r, (int64_t)res - 1); ++x) put(img, res, x, y, c);
            }
            for (int64_t x = l; x <= r; ++x) { put(img, res, x, t, OUTLINE); put(img, res, x, bo, OUTLINE); }
            for (int64_t y = t; y <= bo; ++y) { put(img, res, l, y, OUTLINE); put(img, res, r, y, OUTLINE); }
        }
    }
}

// ---- labels: a TrueType subset, ab_glyph's metrics and ab_glyph_rasterizer's coverage, imageproc's draw_text_mut -----------------
// The rules below restate the published algorithms of those crates (not checked against the crates themselves).  Tables read: head,
// hhea, maxp, cmap format 4, hmtx, loca, glyf with simple glyphs (implied on-curve midpoints); OS/2 only for its USE_TYPO_METRICS bit.
// A composite glyph advances but draws no ink.  No kerning.  All label arithmetic is f32, as in the crates.
namespace {
struct FPoint { float x, y; };
struct Curve { bool quad; FPoint p0, p1, p2; };                    // a line p0-p2, or a quadratic p0-p1-p2
struct GlyphOutline { bool ink = false; float x_min = 0, y_min = 0, x_max = 0, y_max = 0; std::vector<Curve> curves; };

uint16_t be16(const std::string& d, size_t o) { if (o + 2 > d.size()) throw InputError{"the font file is truncated"}; return (uint16_t)(((uint8_t)d[o] << 8) | (uint8_t)d[o + 1]); }
int16_t bes16(const std::string& d, size_t o) { return (int16_t)be16(d, o); }
uint32_t be32r(const std::string& d, size_t o) { return ((uint32_t)be16(d, o) << 16) | be16(d, o + 2); }

FPoint lerp(FPoint a, FPoint b, float t) { return FPoint{a.x + t * (b.x - a.x), a.y + t * (b.y - a.y)}; }   // ttf-parser Point::lerp
}  // namespace

struct DotplotFont {
    std::string d;
    size_t glyf = 0, loca = 0, hmtx = 0, cmap4 = 0;
    bool has_cmap = false, long_loca = false;
    uint16_t n_glyphs = 0, n_hmetrics = 0;
    float ascent = 0, descent = 0;                                   // font units
    size_t table(const char* tag, bool need) const {
        const uint16_t n = be16(d, 4);
        for (uint16_t i = 0; i < n; ++i) if (d.compare(12 + 16 * i, 4, tag) == 0) {
            const uint32_t off = be32r(d, 12 + 16 * i + 8), len = be32r(d, 12 + 16 * i + 12);
            if ((uint64_t)off + len > d.size()) throw InputError{std::string("the font's ") + tag + " table lies outside the file"};
            return off;
        }
        if (need) throw InputError{std::string("the font has no ") + tag + " table"};
        return 0;
    }
    void parse() {
        if (d.size() < 12) throw InputError{"the font file is truncated"};
        const size_t head = table("head", true), hhea = table("hhea", true), maxp = table("maxp", true), os2 = table("OS/2", false);
        glyf = table("glyf", true); loca = table("loca", true); hmtx = table("hmtx", true);
        long_loca = bes16(d, head + 50) != 0;
        n_glyphs = be16(d, maxp + 4);
        n_hmetrics = be16(d, hhea + 34);
        if (n_hmetrics == 0) throw InputError{"the font has no horizontal metrics"};
        ascent = bes16(d, hhea + 4); descent = bes16(d, hhea + 6);
        if (os2 && be16(d, os2) >= 4 && (be16(d, os2 + 62) & 0x80)) { ascent = bes16(d, os2 + 68); descent = bes16(d, os2 + 70); }   // USE_TYPO_METRICS
        const size_t cmap = table("cmap", true);
        const uint16_t nsub = be16(d, cmap + 2);
        int best = -1;
        for (uint16_t i = 0; i < nsub; ++i) {                        // a Unicode BMP subtable in format 4: (3, 1) first, then (0, *)
            const uint16_t pid = be16(d, cmap + 4 + 8 * i), eid = be16(d, cmap + 6 + 8 * i);
            const size_t off = cmap + be32r(d, cmap + 8 + 8 * i);
            if (be16(d, off) != 4) continue;
            const int rank = pid == 3 && eid == 1 ? 2 : pid == 0 ? 1 : 0;
            if (rank > best) { best = rank; cmap4 = off; }
        }
        has_cmap = best > 0;
    }
    uint16_t glyph_id(uint32_t c) const {                            // cmap format 4; anything else is glyph 0
        if (!has_cmap || c > 0xFFFF) return 0;
        const uint16_t segx2 = be16(d, cmap4 + 6);
        const size_t ends = cmap4 + 14, starts = ends + segx2 + 2, deltas = starts + segx2, ranges = deltas + segx2;
        for (uint16_t s = 0; s < segx2; s += 2) {
            if (c > be16(d, ends + s)) continue;
            const uint16_t start = be16(d, starts + s);
            if (c < start) return 0;
            const uint16_t delta = be16(d, deltas + s), ro = be16(d, ranges + s);
            if (ro == 0) return (uint16_t)(c + delta);
            const uint16_t g = be16(d, ranges + s + ro + 2 * (c - start));
            return g == 0 ? 0 : (uint16_t)(g + delta);
        }
        return 0;
    }
    float advance_units(uint16_t g) const { return (float)be16(d, hmtx + 4 * (g < n_hmetrics ? g : n_hmetrics - 1)); }
    float height_units() const { return ascent - descent; }
    GlyphOutline outline(uint16_t g) const;
};

GlyphOutline DotplotFont::outline(uint16_t g) const {
    GlyphOutline o;
    if (g >= n_glyphs) return o;
    const uint32_t a = long_loca ? be32r(d, loca + 4 * g) : 2u * be16(d, loca + 2 * g);
    const uint32_t b = long_loca ? be32r(d, loca + 4 * g + 4) : 2u * be16(d, loca + 2 * g + 2);
    if (b <= a) return o;                                            // no outline (a space)
    const size_t at = glyf + a;
    const int16_t n_contours = bes16(d, at);
    if (n_contours <= 0) return o;                                   // composite glyphs draw no ink
    o.x_min = bes16(d, at + 2); o.y_min = bes16(d, at + 4); o.x_max = bes16(d, at + 6); o.y_max = bes16(d, at + 8);
    std::vector<uint16_t> end_pts(n_contours);
    for (int i = 0; i < n_contours; ++i) end_pts[i] = be16(d, at + 10 + 2 * i);
    const uint32_t n_pts = (uint32_t)end_pts.back() + 1;
    size_t p = at + 10 + 2 * n_contours;
    p += 2 + be16(d, p);                                             // instructions
    std::vector<uint8_t> flags;
    while (flags.size() < n_pts) {
        if (p >= d.size()) throw InputError{"the font file is truncated"};
        const uint8_t f = (uint8_t)d[p++];
        flags.push_back(f);
        if (f & 8) { if (p >= d.size()) throw InputError{"the font file is truncated"}; for (uint8_t r = (uint8_t)d[p++]; r && flags.size() < n_pts; --r) flags.push_back(f); }
    }
    std::vector<float> xs(n_pts), ys(n_pts);
    for (int axis = 0; axis < 2; ++axis) {
        const uint8_t short_bit = axis ? 4 : 2, same_bit = axis ? 32 : 16;
        int32_t v = 0;
        for (uint32_t i = 0; i < n_pts; ++i) {
            if (flags[i] & short_bit) { if (p >= d.size()) throw InputError{"the font file is truncated"}; const int32_t dv = (uint8_t)d[p++]; v += (flags[i] & same_bit) ? dv : -dv; }
            else if (!(flags[i] & same_bit)) { v += bes16(d, p); p += 2; }
            (axis ? ys : xs)[i] = (float)(int16_t)v;
        }
    }
    // ttf-parser's contour builder (implied on-curve midpoints, a contour may start off the curve), into ab_glyph's curve list
    FPoint last{0, 0}, move{0, 0};
    auto move_to = [&](FPoint q) { last = move = q; };
    auto line_to = [&](FPoint q) { o.curves.push_back(Curve{false, last, q, q}); last = q; };
    auto quad_to = [&](FPoint c, FPoint q) { o.curves.push_back(Curve{true, last, c, q}); last = q; };
    uint32_t first = 0;
    for (int c = 0; c < n_contours; ++c) {
        bool have_first_on = false, have_first_off = false, have_last_off = false;
        FPoint first_on{0, 0}, first_off{0, 0}, last_off{0, 0};
        for (uint32_t i = first; i <= end_pts[c] && i < n_pts; ++i) {
            const FPoint q{xs[i], ys[i]};
            const bool on = flags[i] & 1;
            if (!have_first_on) {
                if (on) { have_first_on = true; first_on = q; move_to(q); }
                else if (have_first_off) { const FPoint mid = lerp(first_off, q, 0.5f); have_first_on = true; first_on = mid; have_last_off = true; last_off = q; move_to(mid); }
                else { have_first_off = true; first_off = q; }
            } else if (have_last_off && on) { have_last_off = false; quad_to(last_off, q); }
            else if (have_last_off) { const FPoint prev = last_off; last_off = q; quad_to(prev, lerp(prev, q, 0.5f)); }
            else if (on) line_to(q);
            else { have_last_off = true; last_off = q; }
        }
        if (have_first_off && have_last_off) { have_last_off = false; quad_to(last_off, lerp(last_off, first_off, 0.5f)); }
        if (have_first_on && have_first_off) quad_to(first_off, first_on);
        else if (have_first_on && have_last_off) quad_to(last_off, first_on);
        else if (have_first_on) line_to(first_on);
        if (have_first_on && (last.x != move.x || last.y != move.y)) line_to(move);   // ab_glyph closes an open contour
        first = end_pts[c] + 1u;
    }
    o.ink = !o.curves.empty();
    return o;
}

namespace {
// ab_glyph_rasterizer: signed-area accumulation per cell; coverage = |running sum| capped at 1, row-major over the whole buffer
struct Raster {
    size_t w, h; std::vector<float> a;
    Raster(size_t w_, size_t h_) : w(w_), h(h_), a(w_ * h_ + 4, 0.0f) {}
    void line(FPoint p0, FPoint p1) {
        if (std::fabs(p0.y - p1.y) <= 1.1920929e-7f) return;
        float dir;
        if (p0.y < p1.y) dir = 1.0f; else { dir = -1.0f; std::swap(p0, p1); }
        const float dxdy = (p1.x - p0.x) / (p1.y - p0.y);
        float x = p0.x;
        const size_t y0 = p0.y > 0.0f ? (size_t)p0.y : 0;
        if (p0.y < 0.0f) x -= p0.y * dxdy;
        const float ceil1 = std::ceil(p1.y);
        const size_t yend = std::min(h, ceil1 > 0.0f ? (size_t)ceil1 : (size_t)0);
        for (size_t y = y0; y < yend; ++y) {
            const size_t linestart = y * w;
            const float dy = std::min((float)(y + 1), p1.y) - std::max((float)y, p0.y);
            const float xnext = x + dxdy * dy;
            const float dd = dy * dir;
            const float x0 = x < xnext ? x : xnext, x1 = x < xnext ? xnext : x;
            const float x0floor = std::floor(x0);
            const int32_t x0i = (int32_t)x0floor;
            const float x1ceil = std::ceil(x1);
            const int32_t x1i = (int32_t)x1ceil;
            const int64_t ls0 = (int64_t)linestart + x0i;
            if (ls0 < 0) { x = xnext; continue; }
            if (x1i <= x0i + 1) {
                const float xmf = 0.5f * (x + xnext) - x0floor;
                at(ls0) += dd - dd * xmf;
                at(ls0 + 1) += dd * xmf;
            } else {
                const float s = 1.0f / (x1 - x0);
                const float x0f = x0 - x0floor;
                const float a0 = 0.5f * s * (1.0f - x0f) * (1.0f - x0f);
                const float x1f = x1 - x1ceil + 1.0f;
                const float am = 0.5f * s * x1f * x1f;
                at(ls0) += dd * a0;
                if (x1i == x0i + 2) at(ls0 + 1) += dd * (1.0f - a0 - am);
                else {
                    const float a1 = s * (1.5f - x0f);
                    at(ls0 + 1) += dd * (a1 - a0);
                    for (int32_t xi = x0i + 2; xi < x1i - 1; ++xi) at((int64_t)linestart + xi) += dd * s;
                    const float a2 = a1 + (float)(x1i - x0i - 3) * s;
                    at((int64_t)linestart + x1i - 1) += dd * (1.0f - a2 - am);
                }
                at((int64_t)linestart + x1i) += dd * am;
            }
            x = xnext;
        }
    }
    float& at(int64_t i) { static float sink; return i >= 0 && (size_t)i < a.size() ? a[(size_t)i] : (sink = 0.0f); }   // the crate panics past its buffer; a label never gets there
    void quad(FPoint p0, FPoint p1, FPoint p2) {
        const float devx = p0.x - 2.0f * p1.x + p2.x, devy = p0.y - 2.0f * p1.y + p2.y;
        const float devsq = devx * devx + devy * devy;
        if (devsq < 0.333f) { line(p0, p2); return; }
        const float tol = 3.0f;
        const size_t n = 1 + (size_t)std::floor(std::sqrt(std::sqrt(tol * devsq)));
        FPoint p = p0;
        const float nrecip = 1.0f / (float)n;
        float t = 0.0f;
        for (size_t i = 0; i + 1 < n; ++i) {
            t += nrecip;
            const FPoint pn = lerp(lerp(p0, p1, t), lerp(p1, p2, t), t);
            line(p, pn);
            p = pn;
        }
        line(p, p2);
    }
};

struct Canvas { std::vector<uint8_t>& px; uint32_t w, h; };

// imageproc draw_text_mut (black text): glyphs laid out from caret 0 at baseline `ascent`, each blended as
// pixel * (1 - coverage) + 0 * coverage, truncated to u8
void draw_text(Canvas c, int32_t x, int32_t y, float scale, const DotplotFont& font, const std::string& text);
}  // namespace

static std::vector<uint32_t> utf8_chars(const std::string& s) {
    std::vector<uint32_t> out;
    for (size_t i = 0; i < s.size();) {
        const uint8_t b = (uint8_t)s[i];
        const int n = b < 0x80 ? 1 : (b >> 5) == 6 ? 2 : (b >> 4) == 14 ? 3 : (b >> 3) == 30 ? 4 : 1;
        uint32_t c = n == 1 ? b : n == 2 ? (b & 0x1F) : n == 3 ? (b & 0x0F) : (b & 0x07);
        for (int k = 1; k < n && i + k < s.size(); ++k) c = (c << 6) | ((uint8_t)s[i + k] & 0x3F);
        out.push_back(n == 1 && b >= 0x80 ? 0xFFFD : c);
        i += n;
    }
    return out;
}

static float text_width(const std::string& text, float scale, const DotplotFont& font) {          // calculate_text_width (:361-367)
    const float hf = scale / font.height_units();
    float w = 0.0f;
    for (uint32_t c : utf8_chars(text)) w += hf * font.advance_units(font.glyph_id(c));
    return w;
}

namespace {
void draw_text(Canvas cv, int32_t x, int32_t y, float scale, const DotplotFont& font, const std::string& text) {
    const float hf = scale / font.height_units(), vf = scale / font.height_units();
    const float ascent = vf * font.ascent;
    float caret = 0.0f;
    for (uint32_t ch : utf8_chars(text)) {
        const uint16_t g = font.glyph_id(ch);
        const FPoint pos{caret, ascent};
        caret += hf * font.advance_units(g);
        const GlyphOutline o = font.outline(g);
        if (!o.ink) continue;
        // OutlinedGlyph::px_bounds: bounds (x_min, y_max)-(x_max, y_min) scaled, y flipped, floored / ceiled
        const float minx = std::floor(o.x_min * hf + pos.x), miny = std::floor(o.y_max * -vf + pos.y);
        const float maxx = std::ceil(o.x_max * hf + pos.x), maxy = std::ceil(o.y_min * -vf + pos.y);
        const float bw = maxx - minx, bh = maxy - miny;
        const size_t w = bw > 0.0f ? (size_t)bw : 0, h = bh > 0.0f ? (size_t)bh : 0;
        const FPoint off{pos.x - minx, pos.y - miny};
        auto up = [&](FPoint q) { return FPoint{q.x * hf + off.x, q.y * -vf + off.y}; };
        Raster r(w, h);
        for (const Curve& c : o.curves) { if (c.quad) r.quad(up(c.p0), up(c.p1), up(c.p2)); else r.line(up(c.p0), up(c.p2)); }
        const int32_t xs = x + (int32_t)minx, ys = y + (int32_t)miny;
        float acc = 0.0f;
        for (size_t idx = 0; idx < w * h; ++idx) {
            acc += r.a[idx];
            const float gv = std::min(std::fabs(acc), 1.0f);
            const int64_t ix = (int64_t)(idx % w) + xs, iy = (int64_t)(idx / w) + ys;
            if (ix < 0 || iy < 0 || ix >= cv.w || iy >= cv.h) continue;
            uint8_t* p = &cv.px[((uint64_t)iy * cv.w + (uint64_t)ix) * 3];
            for (int k = 0; k < 3; ++k) {
                const float v = (float)p[k] * (1.0f - gv) + 0.0f * gv;
                p[k] = v < 0.0f ? 0 : v > 255.0f ? 255 : (uint8_t)v;
            }
        }
    }
}
}  // namespace

std::shared_ptr<DotplotFont> dotplot_font_load(const std::string& path) {
    std::string data;
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) fail("cannot read the font file " + path);
    char buf[1 << 16]; size_t n;
    while ((n = fread(buf, 1, sizeof buf, f)) > 0) data.append(buf, n);
    fclose(f);
    auto font = std::make_shared<DotplotFont>();
    font->d = std::move(data);
    font->parse();
    if (!(font->height_units() > 0.0f)) fail("the font's ascender and descender give no line height: " + path);
    return font;
}

std::shared_ptr<DotplotFont> dotplot_font_default(std::string* found) {
    static const char* const paths[] = {"/usr/share/fonts/truetype/dejavu/DejaVuSans.ttf", "/usr/share/fonts/TTF/DejaVuSans.ttf",
                                        "/usr/share/fonts/dejavu/DejaVuSans.ttf", "/usr/share/fonts/dejavu-sans-fonts/DejaVuSans.ttf",
                                        "/usr/share/fonts/truetype/DejaVuSans.ttf", "/usr/local/share/fonts/DejaVuSans.ttf"};
    for (const char* p : paths) {
        struct stat st;
        if (stat(p, &st) == 0 && S_ISREG(st.st_mode)) { if (found) *found = p; return dotplot_font_load(p); }
    }
    return nullptr;
}

// reduce_scale (:308-327): the font size shrinks until every label fits its box, in sequence order; also returns the LAST sequence's
// available width, which draw_labels uses for every vertical label
static float reduce_scale(const std::vector<DotplotInput>& seqs, const Positions& p, const DotplotFont* font, float max_font_size, float* available) {
    float text_height = max_font_size, scale = text_height, available_width = 1.0f;
    for (size_t i = 0; i < seqs.size(); ++i) {
        available_width = (float)(p.end[i] - p.start[i]);
        if (!font) continue;                                          // no labels: nothing is wider than its box
        const float tw = std::max(text_width(seqs[i].filename, scale, *font), text_width(seqs[i].name, scale, *font));
        if (tw > available_width) { text_height *= available_width / tw; scale = text_height; }
    }
    if (available) *available = available_width;
    return text_height;
}

// draw_labels (:336-358) and draw_vertical_text (:370-391)
static void draw_labels(std::vector<uint8_t>& img, uint32_t res, const std::vector<DotplotInput>& seqs, const Positions& p, uint32_t text_gap,
                        const DotplotFont& font, float max_font_size) {
    const uint32_t min_pos = *std::min_element(p.start.begin(), p.start.end());
    float available = 0.0f;
    const float text_height = reduce_scale(seqs, p, &font, max_font_size, &available);
    const uint32_t dim_w = sat_u32f(std::ceil(available)), dim_h = sat_u32f(text_height);
    auto vertical = [&](const std::string& text, uint32_t x, uint32_t y) {
        std::vector<uint8_t> tmp((size_t)dim_w * dim_h * 3, 255);
        draw_text(Canvas{tmp, dim_w, dim_h}, 0, 0, text_height, font, text);
        for (uint32_t i = 0; i < dim_w; ++i) {
            const uint32_t new_y = y - i;                             // u32: wraps below 0 and is then skipped
            if (new_y >= res) continue;
            for (uint32_t j = 0; j < dim_h; ++j) {
                const uint32_t new_x = x + j;
                if (new_x >= res) continue;
                const uint8_t* q = &tmp[((size_t)j * dim_w + i) * 3];
                if (q[0] == 255 && q[1] == 255 && q[2] == 255) continue;
                uint8_t* d = &img[((uint64_t)new_y * res + new_x) * 3];
                d[0] = q[0]; d[1] = q[1]; d[2] = q[2];
            }
        }
    };
    for (size_t i = 0; i < seqs.size(); ++i) {
        const uint32_t pos_1 = min_pos - text_gap - dim_h, pos_2 = pos_1 - dim_h;
        draw_text(Canvas{img, res, res}, (int32_t)p.start[i], (int32_t)pos_1, text_height, font, seqs[i].name);
        draw_text(Canvas{img, res, res}, (int32_t)p.start[i], (int32_t)pos_2, text_height, font, seqs[i].filename);
        vertical(seqs[i].name, pos_1, p.end[i]);
        vertical(seqs[i].filename, pos_2, p.end[i]);
    }
}

static uint32_t px_of(uint32_t start, uint32_t pos, double bpp) {                // :401, :405 (the device's dot_px)
    const double v = std::round((double)pos / bpp);
    return start + sat_u32(v);
}

void dotplot_image(DeviceDotplot& device, const std::vector<DotplotInput>& seqs, uint32_t res, uint32_t kmer, const DotplotFont* font,
                   std::vector<uint8_t>& rgb, DotplotStats& st) {
    st = DotplotStats();
    const uint32_t n = (uint32_t)seqs.size();
    if (n == 0) fail("no sequences were loaded");
    if (n > AC_DOTPLOT_MAX_SEQS) fail("too many sequences for one dotplot (at most 32768)");
    for (const DotplotInput& s : seqs) if (s.seq.size() >= 0xFFFFFFFFull) fail("sequence " + s.name + " is too long");
    // create_dotplot's two passes (:184-200): the label size from the first layout, then the layout with the top-left gap it needs.
    // Without a font, reduce_scale keeps the largest size.
    const Sizes sz = get_sizes(res, n);
    const Positions p0 = get_positions(seqs, res, kmer, sz.top_left_gap, sz.border_gap, sz.between_seq_gap);
    const float text_height = reduce_scale(seqs, p0, font, (float)sz.max_font_size, nullptr);
    const uint32_t top_left_gap = sat_u32f(2.0f * text_height) + sz.border_gap;
    const Positions p = get_positions(seqs, res, kmer, top_left_gap, sz.border_gap, sz.between_seq_gap);
    st.bp_per_pixel = p.bpp; st.text_height = text_height;
    rgb.assign((size_t)res * res * 3, 255);                                   // BACKGROUND_COLOUR
    draw_boxes(rgb, res, p, true);
    if (font) draw_labels(rgb, res, seqs, p, sz.text_gap, *font, (float)sz.max_font_size);

    // the sequences for the device, and the windows holding another byte than ACGT for the host (:394-450 literally, for those)
    std::string bytes;
    std::vector<DotplotSeq> ds(n);
    uint64_t wb = 0;
    struct HostWin { uint32_t seq, pos; };
    std::vector<HostWin> hw;
    for (uint32_t s = 0; s < n; ++s) {
        const std::string& q = seqs[s].seq;
        ds[s] = DotplotSeq{bytes.size(), wb, (uint32_t)q.size(), p.start[s]};
        bytes += q;
        if (q.size() < kmer) continue;
        const uint32_t nw = (uint32_t)(q.size() - kmer + 1);
        wb += nw;
        uint32_t last_bad = 0xFFFFFFFFu;                                       // position of the last non-ACGT byte seen
        for (uint32_t x = 0; x < (uint32_t)q.size(); ++x) {
            const char c = q[x];
            if (c != 'A' && c != 'C' && c != 'G' && c != 'T') last_bad = x;
            if (x + 1 >= kmer) {
                const uint32_t j = x + 1 - kmer;
                if (last_bad != 0xFFFFFFFFu && last_bad >= j) hw.push_back(HostWin{s, j});
            }
        }
    }
    st.windows = wb; st.host_windows = hw.size();
    std::unordered_map<uint64_t, uint64_t> host_pix;
    uint64_t host_dots = 0;
    if (!hw.empty()) {
        std::unordered_map<std::string, std::vector<uint32_t>> fwd, rev;       // Kmers.forward / Kmers.reverse over these windows
        auto window = [&](const HostWin& w) { return seqs[w.seq].seq.substr(w.pos, kmer); };
        auto rc = [](const std::string& s) { std::string r(s.size(), 'N'); for (size_t i = 0; i < s.size(); ++i) r[i] = complement(s[s.size() - 1 - i]); return r; };
        for (uint32_t x = 0; x < hw.size(); ++x) { const std::string w = window(hw[x]); fwd[w].push_back(x); rev[rc(w)].push_back(x); }
        for (const HostWin& v : hw) {                                          // v: window j of sequence b
            const std::string w = window(v);
            const uint32_t y = px_of(p.start[v.seq], v.pos, p.bpp);
            for (int forward = 0; forward < 2; ++forward) {
                auto it = (forward ? fwd : rev).find(w);
                if (it == (forward ? fwd : rev).end()) continue;
                for (uint32_t ui : it->second) {
                    const HostWin& u = hw[ui];
                    const uint32_t x = px_of(p.start[u.seq], u.pos, p.bpp);
                    ++host_dots;
                    if (x >= res || y >= res) continue;
                    const uint64_t key = dotplot_key((uint64_t)u.seq * n + v.seq, v.pos, forward != 0);
                    uint64_t& cur = host_pix[(uint64_t)y * res + x];
                    if (key > cur) cur = key;
                }
            }
        }
    }
    std::vector<uint64_t> hidx, hkey;
    hidx.reserve(host_pix.size()); hkey.reserve(host_pix.size());
    for (const auto& e : host_pix) { hidx.push_back(e.first); hkey.push_back(e.second); }
    DotplotRun run;
    device.dotplot((const uint8_t*)bytes.data(), bytes.size(), ds.data(), n, kmer, p.bpp, res, hidx.data(), hkey.data(), hidx.size(), rgb.data(), &run);
    st.groups = run.groups; st.dots = run.dots + host_dots; st.kernel_ms = run.kernel_ms;
    draw_boxes(rgb, res, p, false);                                            // the outlines once more, over the dots (:213-215)
}

// ---- PNG -------------------------------------------------------------------------------------------------------------------------
static void be32(std::string& s, uint32_t v) { const char b[4] = {(char)(v >> 24), (char)(v >> 16), (char)(v >> 8), (char)v}; s.append(b, 4); }
static void chunk(std::string& out, const char* type, const std::string& data) {
    be32(out, (uint32_t)data.size());
    const std::string td = std::string(type, 4) + data;
    out += td;
    be32(out, (uint32_t)crc32(crc32(0L, Z_NULL, 0), (const Bytef*)td.data(), (uInt)td.size()));
}

bool png_write(const std::string& path, const uint8_t* rgb, uint32_t width, uint32_t height) {
    std::string ihdr;
    be32(ihdr, width); be32(ihdr, height);
    ihdr += std::string("\x08\x02\x00\x00\x00", 5);                           // 8-bit RGB, deflate, adaptive filtering, no interlace
    const uint64_t row = (uint64_t)width * 3;
    std::vector<uint8_t> raw((row + 1) * height);
    for (uint32_t y = 0; y < height; ++y) { raw[y * (row + 1)] = 0; memcpy(&raw[y * (row + 1) + 1], rgb + y * row, row); }   // filter type 0 on every row
    uLongf zlen = compressBound((uLong)raw.size());
    std::string z(zlen, '\0');
    if (compress2((Bytef*)&z[0], &zlen, raw.data(), (uLong)raw.size(), 6) != Z_OK) return false;
    z.resize(zlen);
    std::string out("\x89PNG\r\n\x1a\n", 8);
    chunk(out, "IHDR", ihdr); chunk(out, "IDAT", z); chunk(out, "IEND", std::string());
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = fwrite(out.data(), 1, out.size(), f) == out.size();
    return fclose(f) == 0 && ok;
}
