// `autocycler clean` (clean.rs:23-149), `autocycler gfa2fasta` (gfa2fasta.rs:23-82) and `autocycler table` (table.rs:24-204): commands
// users run on the outputs of the others.  They work on consensus graphs of a handful of unitigs and on YAML files of a few kilobytes,
// and one of them (remove_low_depth_unitigs) is sequential by definition, so they are host only and need no device.
//
// Two inputs make the reference panic, and are refused here with the reference's kind of error (InputError) instead: a tig that is
// both removed and duplicated, and a tig listed twice in --duplicate.  In both the second operation would look up a unitig that is
// already gone.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "host_graph.h"

// parse_tig_numbers (clean.rs:142-149): spaces removed, split on ',', each item a u32, sorted
std::vector<uint32_t> parse_tig_numbers(const std::string& text);

// UnitigGraph::from_gfa_lines of a GFA given by the user: every loader error is an input error
void load_user_gfa(const std::string& text, HostGraph& g);

// clean.rs:26-45 on a loaded graph: checks the numbers (`name` stands for the input file in the messages), removes, duplicates, drops
// low-depth tigs (min_depth may be null), then, when `merge` is set, merges linear paths and renumbers.  The GFA text is saved with
// use_other_colour and no P lines.  verbose: the reference's report on stderr.
void clean_graph(HostGraph& g, const std::string& name, std::vector<uint32_t> remove, std::vector<uint32_t> duplicate,
                 const double* min_depth, bool merge, bool verbose, std::string& gfa);

// save_graph_to_fasta (gfa2fasta.rs:55-82): counts[0..3) = circular, linear and other sequences written
std::string gfa_fasta_text(const HostGraph& g, uint64_t counts[3]);

// table.rs:24-123: `autocycler_dir` empty prints the header line; fields is the -f text.  Returns the line, newline included.
// verbose: the "not found" warnings on stderr.
std::string table_text(const std::string& autocycler_dir, bool have_dir, const std::string& name, const std::string& fields, uint64_t sigfigs,
                       bool verbose);
extern const char* const TABLE_DEFAULT_FIELDS;    // main.rs:287-293

// format_float_sigfigs (misc.rs:373-386), bit for bit
std::string format_float_sigfigs(double value, uint64_t sigfigs);
