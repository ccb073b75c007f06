// `autocycler dotplot` on the host (dotplot.rs): inputs, layout, boxes, the dots of the windows the device does not take, and the PNG.
// The dots of every window of only ACGT run on the GPU (DeviceDotplot::dotplot).  Citations are file:line in the reference's src/.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "commands.h"

struct DotplotInput { std::string filename, name, seq; };        // FileSeqName and the bytes, uppercased (dotplot.rs:106-110)

struct DotplotStats {
    uint64_t windows = 0, groups = 0, dots = 0, host_windows = 0;
    double bp_per_pixel = 0;
    float text_height = 0, kernel_ms = 0;
};

// check_settings (dotplot.rs:55-60); throws InputError with the reference's message
void dotplot_check_settings(uint32_t res, uint32_t kmer);
// determine_input_type + load_sequences (dotplot.rs:65-80, 113-176): a directory of assemblies, a FASTA file or an Autocycler GFA
// (sequences sorted by (filename, name) then bytes, unitig_graph.rs:372-381).  Refuses two sequences with the same (filename, name).
std::vector<DotplotInput> dotplot_load(const std::string& input, bool verbose);
// A TrueType font for the labels (the subset dotplot needs; see host_dotplot.cpp).  dotplot_font_load throws InputError when the
// file cannot be read or parsed; dotplot_font_default tries a fixed list of standard DejaVuSans.ttf paths and returns null if none exists.
struct DotplotFont;
std::shared_ptr<DotplotFont> dotplot_font_load(const std::string& path);
std::shared_ptr<DotplotFont> dotplot_font_default(std::string* found_path);
// create_dotplot (dotplot.rs:179-221) into rgb (res x res x 3): boxes, labels (none when font is null), dots (device), outlines again
void dotplot_image(DeviceDotplot& device, const std::vector<DotplotInput>& seqs, uint32_t res, uint32_t kmer, const DotplotFont* font,
                   std::vector<uint8_t>& rgb, DotplotStats& st);
// an RGB8 PNG (colour type 2, no interlace, zlib), written to path; false on an I/O error
bool png_write(const std::string& path, const uint8_t* rgb, uint32_t width, uint32_t height);
