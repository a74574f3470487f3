// lfr_solve_main.cc — native `solve` executable: the command-line surface of the reference's
// multi-view-refinement/solve.cc main() (solve.cc:375-682) above the C ABI.
//
//     solve --matches_file X.pb --output_file Y.pb [--n_threads 8] [--banned_images NAME]...
//
// Same flags (solve.cc:379-385, Boost.Program_options semantics and messages), same `.part.N` handling
// (:416-424), same stdout lines (:484-485,534,549,589,591,606,638,641,670) and exit codes (0; 1 on a
// command-line error, :397-401; -1 = 255 when the input does not parse or the output cannot be
// written, :433-436,674-677).  The work is lfr_wire_walk_matches() (include/lfr_wire.h) over the pairs,
// the graph stage, the solve and the SolutionFile.  The graph stage runs where
// lfr_graph_stage_on_device() (include/lfr_graph.h) says, from the pair level alone:
//   device: lfr_plan_create_from_wire() on the mapped parts (the matches are decoded on the GPU) — or,
//           below the match count lfr_wire_decode_on_device() sets, lfr_wire_decode_matches() +
//           lfr_plan_create_from_matches() —, lfr_plan_solve() on the plan left in HBM, and
//           lfr_plan_encode_solution() for the SolutionFile bytes (encoded on the GPU from the positions
//           in HBM);
//   host:   lfr_wire_decode_matches(), lfr_host_stage_create() (include/lfr_host.h) writing the edge
//           records into page-locked memory, then lfr_solve() / lfr_solve_multi() (include/lfr.h), the
//           output assembly and lfr_wire_encode_solution().
// Both routes give the same bytes and lines.  LFR_GRAPH_STAGE=host|device forces a route (a test and
// measurement hook); on the device route LFR_DEVICE_CUT=1 cuts oversized meta-components on the GPU too.  Opt-in extras: --device D, --gpus N (one process drives N GPUs; host route),
// --fixed_images NAME (repeatable: every node of the image is held constant, as a root is) and
// --initial_solution FILE (start values from a SolutionFile instead of zeros), with
// --keep_initial_solution (every keypoint with an entry in that file is held constant too) — on the device
// route lfr_plan_fix_images() / lfr_plan_start_from_solution() or lfr_plan_keep_solution(), on the host
// route the constant mask and lfr_wire_join_solution() or _entries() handed to the solve — and
// --carry_initial_solution (the output also holds every entry of that file the scene does not refine:
// lfr_plan_encode_solution_carried() on the device route, lfr_wire_encode_solution_carried() on the host
// route's assembly) and --update_initial_solution (every component a keypoint without an entry in that
// file joins is solved from zeros as without the file, every other one is held at the file's values:
// lfr_plan_update_solution() on the device route, lfr_wire_update_solution() handed to the solve on the host
// route) and --previous_matches_file OLD.pb (with --update_initial_solution: a component is also solved again
// when its problem is not the one OLD.pb's run solved: lfr_plan_update_solution_since() with a plan built from
// OLD.pb on the device route, lfr_wire_update_solution_since() on the host route) and --record_file FILE (after
// the SolutionFile, this run's problem record: lfr_plan_problem_record() on the device route,
// lfr_host_problem_record() on the host route, the same bytes) and --earlier_record_file FILE (with
// --update_initial_solution, in place of --previous_matches_file: the record the earlier run wrote;
// lfr_plan_update_solution_since_record() / lfr_wire_update_solution_since_record()) and --query_images NAME
// (repeatable: each query's pairs become a sub-scene with its own ids for the database images, the graph stage
// takes the sub-scene of every id, lfr_host_input::image_group, and only query images are written:
// lfr_plan_encode_solution_images() on the device route) and --joint_queries (with --query_images: queries
// that a kept pair names together share one sub-scene, so sequences and rigs are refined jointly) and
// --additional_scenes FILE (lines `MATCHES_FILE<TAB>OUTPUT_FILE`: every listed scene is one more sub-scene of the
// same run, and each scene's output file holds what its own run writes: lfr_plan_encode_solution_groups() on
// the device route) and --listed_pairs FILE (lines `MATCH_LIST<TAB>OUTPUT_FILE`: the pairs of every match list,
// one `NAME1 NAME2` per line, are taken out of --matches_file, and each list's output file holds what the run on
// a MatchingFile of those pairs in line order writes: lfr_plan_create_from_wire_listed() expands the file's
// matches, decoded once, on the device route) and --versioned_scenes FILE (lines `MATCHES_FILE<TAB>OUTPUT_FILE<TAB>
// INITIAL_SOLUTION<TAB>EARLIER_RECORD<TAB>RECORD_FILE`: a scene batch whose every scene is updated from its own
// solution and record, or solved from zeros without one, and writes its own record: lfr_plan_update_solution_groups()
// and lfr_plan_problem_record_groups() on the device route, lfr_wire_update_solution_groups() and
// lfr_host_problem_record_groups() on the host route) and --task_stream FILE (with --device, --gpus and --n_threads alone:
// one process runs every line of FILE, read as it arrives, as a task, each line's TAB-separated fields its argument
// vector, and prints `# task K: exit C` after each; run_stream()).  `--n_threads` is accepted and
// ignored (the solve runs on the GPU).  local-feature-refinement_b200/cli.py is the same program in
// Python; this one starts in milliseconds instead of importing numpy.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fcntl.h>
#include <fstream>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "../../include/lfr.h"
#include "../../include/lfr_graph.h"
#include "../../include/lfr_host.h"
#include "../../include/lfr_wire.h"
#include "lfr_record.h"

// The graph stage on the GPU is resolved weakly: the same source links against the CPU checker
// (oracle/liblfr_ref.so), which has no plans; there they are NULL and every input takes the host route.
extern "C" {
int lfr_graph_stage_on_device(const lfr_host_input* in, int32_t n_devices) __attribute__((weak));
int lfr_wire_decode_on_device(uint64_t n_matches) __attribute__((weak));
int lfr_plan_create_from_matches(const lfr_host_input* in, const lfr_options* o, const double* initial_positions,
                                 lfr_plan** out, lfr_host_sizes* sizes) __attribute__((weak));
int lfr_plan_create_from_wire(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts,
                              const lfr_options* o, const double* initial_positions, lfr_plan** out,
                              lfr_host_sizes* sizes) __attribute__((weak));
int lfr_plan_create_from_wire_listed(const lfr_host_input* in, const lfr_wire_part* parts, uint32_t n_parts,
                                     const uint64_t* src_pair_ptr, uint64_t n_src_pairs, const uint64_t* pair_src,
                                     const lfr_options* o, const double* initial_positions, lfr_plan** out,
                                     lfr_host_sizes* sizes) __attribute__((weak));
int64_t lfr_plan_encode_solution(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                 const uint64_t* name_off, const float* fact, uint8_t* out, uint64_t cap,
                                 uint64_t* n_outside) __attribute__((weak));
int lfr_plan_fix_images(lfr_plan* plan, const uint8_t* fixed_by_image_id, uint32_t n_images) __attribute__((weak));
int lfr_plan_start_from_solution(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                 const uint8_t* names, const uint64_t* name_off, uint64_t* n_started) __attribute__((weak));
int lfr_plan_keep_solution(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                           const uint8_t* names, const uint64_t* name_off, uint64_t* n_kept) __attribute__((weak));
int lfr_plan_update_solution(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                             const uint8_t* names, const uint64_t* name_off, uint64_t* n_held,
                             uint32_t* n_touched) __attribute__((weak));
int lfr_plan_update_solution_since(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len, uint32_t n_images,
                                   const uint8_t* names, const uint64_t* name_off, const lfr_plan* previous,
                                   uint32_t prev_n_images, const uint8_t* prev_names, const uint64_t* prev_name_off,
                                   uint64_t* n_held, uint32_t* n_touched, uint32_t* n_changed) __attribute__((weak));
int64_t lfr_plan_problem_record(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                const uint64_t* name_off, uint8_t* out, uint64_t cap) __attribute__((weak));
int lfr_plan_update_solution_since_record(lfr_plan* plan, void* stream, const uint8_t* bytes, uint64_t len,
                                          uint32_t n_images, const uint8_t* names, const uint64_t* name_off,
                                          const uint8_t* record, uint64_t record_len, uint64_t* n_held,
                                          uint32_t* n_touched, uint32_t* n_changed) __attribute__((weak));
int64_t lfr_plan_encode_solution_images(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                        const uint64_t* name_off, const float* fact, const uint8_t* written, uint8_t* out,
                                        uint64_t cap, uint64_t* n_outside) __attribute__((weak));
int64_t lfr_plan_encode_solution_carried(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                         const uint64_t* name_off, const float* fact, const uint8_t* file,
                                         uint64_t file_len, uint8_t* out, uint64_t cap, uint64_t* n_outside,
                                         uint64_t* n_carried) __attribute__((weak));
int64_t lfr_plan_encode_solution_groups(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                        const uint64_t* name_off, const float* fact, const uint32_t* group_of_image,
                                        uint32_t n_groups, uint8_t* out, uint64_t cap, uint64_t* group_off,
                                        uint64_t* n_outside) __attribute__((weak));
int lfr_plan_update_solution_groups(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                    const uint64_t* name_off, const uint32_t* group_of_image, uint32_t n_groups,
                                    const uint8_t* const* files, const uint64_t* file_len, const uint8_t* const* records,
                                    const uint64_t* record_len, uint64_t* n_held, uint32_t* n_touched,
                                    uint32_t* n_changed) __attribute__((weak));
int64_t lfr_plan_problem_record_groups(lfr_plan* plan, void* stream, uint32_t n_images, const uint8_t* names,
                                       const uint64_t* name_off, const uint32_t* group_of_image, uint32_t n_groups,
                                       uint8_t* out, uint64_t cap, uint64_t* group_off) __attribute__((weak));
}

namespace {

const char* kUsage =
    "Options:\n"
    "  --help                    print the help\n"
    "  --matches_file arg        path to the matches file\n"
    "  --output_file arg         path to the output file\n"
    "  --n_threads arg (=8)      # threads\n"
    "  --banned_images arg (={}) banned images\n";

struct CliError {
  std::string msg;
};

// The end of the run with exit code `code`; its message is on stderr already.  `lost`: a library call returned
// LFR_ECUDA or LFR_ENODEV, so the CUDA context may be unusable for any later run in the process.
struct Exit {
  int code;
  bool lost = false;
};

[[noreturn]] __attribute__((format(printf, 2, 3))) void fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  std::vfprintf(stderr, fmt, ap);
  va_end(ap);
  throw Exit{code};
}

// Exits 2 after `ERROR: <what> failed (rc): <the library's message>` for a library call that returned `rc`
[[noreturn]] void fail_call(const char* what, int rc) {
  std::fprintf(stderr, "ERROR: %s failed (%d): %s\n", what, rc, lfr_last_error());
  throw Exit{2, rc == LFR_ECUDA || rc == LFR_ENODEV};
}

struct OptionSpec {
  const char* name;
  bool takes, repeat;
};
// solve.cc:379-385 plus the opt-in extras
const OptionSpec kOptions[] = {{"help", false, false},        {"matches_file", true, false}, {"output_file", true, false},
                               {"n_threads", true, false},    {"banned_images", true, true}, {"device", true, false},
                               {"gpus", true, false},         {"fixed_images", true, true},  {"initial_solution", true, false},
                               {"keep_initial_solution", false, false}, {"carry_initial_solution", false, false},
                               {"update_initial_solution", false, false}, {"previous_matches_file", true, false},
                               {"record_file", true, false},  {"earlier_record_file", true, false},
                               {"query_images", true, true},  {"joint_queries", false, false},
                               {"additional_scenes", true, false}, {"listed_pairs", true, false},
                               {"versioned_scenes", true, false}, {"task_stream", true, false}};

// exact name, else unambiguous prefix (Boost.Program_options' default allow_guessing)
const OptionSpec& find_option(const std::string& name) {
  const OptionSpec* hit = nullptr;
  int n_hits = 0;
  for (const OptionSpec& o : kOptions) {
    if (name == o.name) return o;
    if (std::strncmp(o.name, name.c_str(), name.size()) == 0) {
      hit = &o;
      ++n_hits;
    }
  }
  if (n_hits == 1) return *hit;
  if (n_hits > 1) throw CliError{"option '--" + name + "' is ambiguous"};
  throw CliError{"unrecognised option '--" + name + "'"};
}

// The command line.  An absent single option is nullopt, except --initial_solution, which is empty when absent.
struct Options {
  bool help = false, keep_initial_solution = false, carry_initial_solution = false, update_initial_solution = false,
       joint_queries = false;
  std::string matches_file, output_file, initial_solution;
  std::optional<std::string> previous_matches_file, record_file, earlier_record_file, additional_scenes, listed_pairs,
      versioned_scenes, task_stream;
  std::vector<std::string> banned_images, fixed_images, query_images;
  uint64_t device = 0, gpus = 1;
  std::set<std::string> named;  // every option the command line names
};

// Boost.Program_options semantics of solve.cc:387-401: long options, `--name value` or `--name=value`,
// no positional arguments, Boost's error messages
Options parse(int argc, char** argv) {
  std::map<std::string, std::string> single;
  std::map<std::string, std::vector<std::string>> repeated;
  std::set<std::string> flags;
  for (int i = 1; i < argc;) {
    const std::string tok = argv[i++];
    if (tok.size() > 2 && tok.compare(0, 2, "--") == 0) {
      const size_t eq = tok.find('=');
      const std::string name = tok.substr(2, eq == std::string::npos ? std::string::npos : eq - 2);
      const OptionSpec& o = find_option(name);
      if (o.takes) {
        std::string v;
        if (eq != std::string::npos) {
          v = tok.substr(eq + 1);
        } else if (i < argc && !(argv[i][0] == '-' && argv[i][1] != '\0')) {
          v = argv[i++];
        } else {
          throw CliError{std::string("the required argument for option '--") + o.name + "' is missing"};
        }
        if (o.repeat) {
          repeated[o.name].push_back(v);
        } else if (single.count(o.name)) {
          throw CliError{std::string("option '--") + o.name + "' cannot be specified more than once"};
        } else {
          single[o.name] = v;
        }
      } else {
        if (eq != std::string::npos) throw CliError{std::string("option '--") + o.name + "' does not take any arguments"};
        flags.insert(o.name);
      }
    } else if (tok.size() > 1 && tok[0] == '-') {
      throw CliError{"unrecognised option '" + tok + "'"};
    } else {
      throw CliError{"too many positional options have been specified on the command line"};
    }
  }
  Options o;
  o.help = flags.count("help") != 0;
  if (o.help) return o;
  // po::notify: required options, in declaration order; a task stream's tasks name their own files
  for (const char* req : {"matches_file", "output_file"})
    if (!single.count(req) && !single.count("task_stream"))
      throw CliError{std::string("the option '--") + req + "' is required but missing"};
  auto as_uint = [&](const char* name, uint64_t dflt) {  // lexical_cast<size_t>
    const auto it = single.find(name);
    if (it == single.end()) return dflt;
    const std::string& v = it->second;
    bool digits = !v.empty();
    for (char c : v) digits = digits && c >= '0' && c <= '9';
    if (!digits) throw CliError{"the argument ('" + v + "') for option '--" + name + "' is invalid"};
    return (uint64_t)std::strtoull(v.c_str(), nullptr, 10);
  };
  (void)as_uint("n_threads", 8);
  o.device = as_uint("device", 0);
  o.gpus = as_uint("gpus", 1);
  auto given = [&](const char* name) {
    const auto it = single.find(name);
    return it == single.end() ? std::optional<std::string>() : it->second;
  };
  o.matches_file = given("matches_file").value_or("");
  o.output_file = given("output_file").value_or("");
  o.task_stream = given("task_stream");
  o.initial_solution = given("initial_solution").value_or("");
  o.previous_matches_file = given("previous_matches_file");
  o.record_file = given("record_file");
  o.earlier_record_file = given("earlier_record_file");
  o.additional_scenes = given("additional_scenes");
  o.listed_pairs = given("listed_pairs");
  o.versioned_scenes = given("versioned_scenes");
  o.banned_images = repeated["banned_images"];
  o.fixed_images = repeated["fixed_images"];
  o.query_images = repeated["query_images"];
  o.keep_initial_solution = flags.count("keep_initial_solution") != 0;
  o.carry_initial_solution = flags.count("carry_initial_solution") != 0;
  o.update_initial_solution = flags.count("update_initial_solution") != 0;
  o.joint_queries = flags.count("joint_queries") != 0;
  for (const auto& kv : single) o.named.insert(kv.first);
  for (const auto& kv : repeated)  // operator[] above added the repeatable options not given, empty
    if (!kv.second.empty()) o.named.insert(kv.first);
  o.named.insert(flags.begin(), flags.end());
  return o;
}

// The opt-in options the rules between options speak of
enum Opt { kFixed, kStart, kKeep, kCarry, kUpdate, kPrevious, kRecord, kEarlier, kQuery, kJoint, kScenes, kLists, kVersioned,
           kMatches, kOutput, kBanned, kTasks, kNumOpts };
const char* const kOptName[kNumOpts] = {"--fixed_images",          "--initial_solution",    "--keep_initial_solution",
                                        "--carry_initial_solution", "--update_initial_solution", "--previous_matches_file",
                                        "--record_file",           "--earlier_record_file", "--query_images",
                                        "--joint_queries",         "--additional_scenes",   "--listed_pairs",
                                        "--versioned_scenes",      "--matches_file",        "--output_file",
                                        "--banned_images",         "--task_stream"};

// `opt` needs `others[0]`, or excludes each of `others`
struct Rule {
  Opt opt;
  bool needs;
  std::vector<Opt> others;
};
// The start solution, the fixed images, the incremental modes and the queries belong to one scene: a batch
// (--additional_scenes, --listed_pairs) excludes them
const std::vector<Opt> kOneScene = {kFixed, kStart, kKeep, kCarry, kUpdate, kPrevious, kRecord, kEarlier, kQuery, kJoint};
// In order: with two conflicts, the first rule that fires writes the message.
const std::vector<Rule> kRules = {
    {kKeep, true, {kStart}},
    {kCarry, true, {kStart}},
    {kUpdate, true, {kStart}},
    {kUpdate, false, {kKeep}},
    {kPrevious, true, {kUpdate}},
    {kEarlier, true, {kUpdate}},
    {kEarlier, false, {kPrevious}},
    // each query is refined against the scene as it stands; the incremental modes update one scene
    {kQuery, false, {kUpdate, kPrevious, kRecord, kEarlier, kCarry}},
    {kJoint, true, {kQuery}},
    {kLists, false, [] { std::vector<Opt> v = kOneScene; v.push_back(kScenes); return v; }()},
    {kScenes, false, kOneScene},
    // every scene of --versioned_scenes starts from its own solution and record, scene 0 from the ordinary flags;
    // fixed images, kept and carried solutions, earlier MatchingFiles and queries stay one-scene options
    {kVersioned, false, {kFixed, kKeep, kCarry, kPrevious, kQuery, kJoint, kScenes, kLists}},
    // a task stream's command line sets the process alone (--device, --gpus, --n_threads): every task names its own
    // files and options
    {kTasks, false, {kMatches, kOutput, kBanned, kFixed, kStart, kKeep, kCarry, kUpdate, kPrevious, kRecord, kEarlier, kQuery,
                     kJoint, kScenes, kLists, kVersioned}},
};

// Exits 2 after the ERROR line of the first rule the command line breaks
void check_rules(const Options& o) {
  const bool set[kNumOpts] = {!o.fixed_images.empty(),       !o.initial_solution.empty(), o.keep_initial_solution,
                              o.carry_initial_solution,      o.update_initial_solution,   o.previous_matches_file.has_value(),
                              o.record_file.has_value(),     o.earlier_record_file.has_value(), !o.query_images.empty(),
                              o.joint_queries,               o.additional_scenes.has_value(), o.listed_pairs.has_value(),
                              o.versioned_scenes.has_value(), o.named.count("matches_file") != 0,
                              o.named.count("output_file") != 0, !o.banned_images.empty(), o.task_stream.has_value()};
  for (const Rule& r : kRules) {
    if (!set[r.opt]) continue;
    for (const Opt b : r.others) {
      // the task stream excludes every option its command line names, whatever the value (an empty path too)
      const bool on = r.opt == kTasks ? o.named.count(kOptName[b] + 2) != 0 : set[b];
      if (r.needs && !on) fail(2, "ERROR: %s needs %s%s\n", kOptName[r.opt], kOptName[b], b == kStart ? " FILE" : "");
      if (!r.needs && on) fail(2, "ERROR: %s and %s exclude each other\n", kOptName[r.opt], kOptName[b]);
    }
  }
  // a batch's scenes are updated or solved from zeros: a start point alone belongs to one scene
  if (set[kVersioned] && set[kStart] && !set[kUpdate])
    fail(2, "ERROR: %s: %s needs %s\n", kOptName[kVersioned], kOptName[kStart], kOptName[kUpdate]);
}

// How the solve starts (solve.cc:608-612): from zeros, or from --initial_solution joined, kept, or updated (alone,
// since --previous_matches_file, since --earlier_record_file), or with --versioned_scenes every scene updated from its
// own solution and record or from zeros
enum class Start { kZeros, kJoin, kKeep, kUpdate, kUpdateSinceMatches, kUpdateSinceRecord, kScenes };

Start start_mode(const Options& o) {
  if (o.versioned_scenes) return Start::kScenes;
  if (o.initial_solution.empty()) return Start::kZeros;
  if (o.earlier_record_file) return Start::kUpdateSinceRecord;
  if (o.previous_matches_file) return Start::kUpdateSinceMatches;
  if (o.update_initial_solution) return Start::kUpdate;
  return o.keep_initial_solution ? Start::kKeep : Start::kJoin;
}

// keep and the updates hold the nodes with an entry in the start solution constant
bool holds_entries(Start s) { return s != Start::kZeros && s != Start::kJoin; }

// The sub-scenes of the graph stage (lfr_host_input::image_group), with the nouns of the "more than 65535" message
struct Labelling {
  enum Kind { kNone, kQueries, kScenes, kLists } kind;
  const char *option, *members, *list;
  bool batched() const { return kind == kScenes || kind == kLists; }
};

Labelling labelling(const Options& o) {
  if (!o.query_images.empty()) return {Labelling::kQueries, "--query_images", "sub-scenes", "query list"};
  if (o.listed_pairs) return {Labelling::kLists, "--listed_pairs", "lists", "pair list"};
  if (o.additional_scenes) return {Labelling::kScenes, "--additional_scenes", "scenes", "scene list"};
  if (o.versioned_scenes) return {Labelling::kScenes, "--versioned_scenes", "scenes", "scene list"};
  return {Labelling::kNone, nullptr, nullptr, nullptr};
}

bool file_exists(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return f.good();
}

// solve.cc:416-424: the file `path`, or else its pieces `path`.part.0, .part.1, ... up to the first one missing
std::vector<std::string> matching_files(const std::string& path) {
  if (file_exists(path)) return {path};
  std::vector<std::string> files;
  for (int k = 0;; ++k) {
    std::string f = path + ".part." + std::to_string(k);
    if (!file_exists(f)) return files;
    files.push_back(std::move(f));
  }
}

// A file mapped read-only (a Madrid-scale MatchingFile is several GB: no second copy of it in memory).
// Unmapped when released or destroyed, so that no run leaves a mapping behind, whichever way it ends.
struct FileImage {
  const uint8_t* p = nullptr;
  size_t n = 0;
  FileImage() = default;
  FileImage(const FileImage&) = delete;
  FileImage& operator=(const FileImage&) = delete;
  FileImage(FileImage&& o) noexcept : p(o.p), n(o.n) {
    o.p = nullptr;
    o.n = 0;
  }
  ~FileImage() { release(); }
  bool open(const std::string& path) {
    const int fd = ::open(path.c_str(), O_RDONLY);
    if (fd < 0) return false;
    struct stat st;
    if (fstat(fd, &st) != 0) {
      ::close(fd);
      return false;
    }
    n = (size_t)st.st_size;
    if (n) {
      void* m = mmap(nullptr, n, PROT_READ, MAP_PRIVATE, fd, 0);
      ::close(fd);
      if (m == MAP_FAILED) {
        n = 0;
        return false;
      }
      p = static_cast<const uint8_t*>(m);
    } else {
      ::close(fd);
    }
    return true;
  }
  void release() {
    if (p) munmap(const_cast<uint8_t*>(p), n);
    p = nullptr;
    n = 0;
  }
  const uint8_t* data() const { return p; }
  size_t size() const { return n; }
};

// The bytes of the file `path` into `text`; false when it cannot be read
bool read_file(const std::string& path, std::string& text) {
  FileImage f;
  if (!f.open(path)) return false;
  text.assign(reinterpret_cast<const char*>(f.data()), f.size());
  f.release();
  return true;
}

// The lines of `text`, split at '\n'; the last newline is optional
std::vector<std::string> lines_of(const std::string& text) {
  std::vector<std::string> lines;
  for (size_t at = 0; at < text.size();) {
    const size_t end = std::min(text.find('\n', at), text.size());
    lines.push_back(text.substr(at, end - at));
    at = end + 1;
  }
  return lines;
}

// One MatchingFile part after the pair walk: image names as byte ranges of its buffer, the matches as
// the offsets of their length prefixes.
struct Part {
  FileImage buf;
  uint64_t P = 0, M = 0;
  std::vector<uint64_t> pair_ptr, n1_off, n2_off, match_off;
  std::vector<uint32_t> n1_len, n2_len;
  std::vector<float> fact1, fact2;
  // Map `path`, count its pairs and matches and size the pair-level arrays: 0, 2 when the file cannot be mapped,
  // 255 when its bytes do not parse
  int open(const std::string& path) {
    if (!buf.open(path)) return 2;
    if (lfr_wire_scan_matches(buf.data(), buf.size(), &P, &M) != LFR_OK) return 255;
    pair_ptr.resize(P + 1);
    n1_off.resize(P); n2_off.resize(P); n1_len.resize(P); n2_len.resize(P);
    fact1.resize(P); fact2.resize(P);
    return 0;
  }
  lfr_wire_matches pair_level(uint32_t* feat1, uint32_t* feat2, float* sim, float* disp1, float* disp2) {
    lfr_wire_matches w;
    w.n_pairs = P; w.n_matches = M;
    w.pair_ptr = pair_ptr.data(); w.fact1 = fact1.data(); w.fact2 = fact2.data();
    w.name1_off = n1_off.data(); w.name1_len = n1_len.data();
    w.name2_off = n2_off.data(); w.name2_len = n2_len.data();
    w.feat1 = feat1; w.feat2 = feat2; w.sim = sim; w.disp1 = disp1; w.disp2 = disp2;
    return w;
  }
};

// Image names -> ids in order of first appearance
struct NameTable {
  std::vector<std::string> names;
  std::map<std::string, uint32_t> id_of;
  uint32_t intern(const Part& pt, uint64_t off, uint32_t len) {
    std::string s(reinterpret_cast<const char*>(pt.buf.data()) + off, len);
    const auto it = id_of.find(s);
    if (it != id_of.end()) return it->second;
    const uint32_t id = (uint32_t)names.size();
    id_of.emplace(s, id);
    names.push_back(std::move(s));
    return id;
  }
};

using StringPairs = std::vector<std::pair<std::string, std::string>>;

// The nouns of a TAB-separated list file
struct TabList {
  const char *option, *file, *first, *first_empty, *rows;
};
const TabList kSceneList = {"--additional_scenes", "scene list", "MATCHES_FILE", "its matches file is empty", "scenes"};
const TabList kPairList = {"--listed_pairs", "pair list", "MATCH_LIST", "its match list is empty", "lists"};

// The list file of --additional_scenes or --listed_pairs: one `FIRST<TAB>OUTPUT_FILE` per line (raw bytes; the
// last newline is optional), appended to `rows`.  Exits 2 after one ERROR line for an unreadable file, a malformed
// line or two rows (those in `rows` before included) with the same output path.
void read_tab_list(const TabList& kind, const std::string& path, StringPairs& rows) {
  std::string text;
  if (!read_file(path, text)) fail(2, "ERROR: cannot read the %s file '%s'\n", kind.file, path.c_str());
  const std::vector<std::string> lines = lines_of(text);
  for (size_t k = 0; k < lines.size(); ++k) {
    const std::string& l = lines[k];
    const size_t tab = l.find('\t');
    const char* why = l.empty()                                  ? "it is empty"
                      : tab == std::string::npos                 ? "it has no TAB"
                      : l.find('\t', tab + 1) != std::string::npos ? "it has more than one TAB"
                      : tab == 0                                 ? kind.first_empty
                      : tab + 1 == l.size()                      ? "its output file is empty"
                      : l.find('\0') != std::string::npos        ? "it holds a NUL byte"
                                                                 : nullptr;
    if (why) fail(2, "ERROR: %s: line %zu is not %s<TAB>OUTPUT_FILE: %s\n", kind.option, k + 1, kind.first, why);
    rows.emplace_back(l.substr(0, tab), l.substr(tab + 1));
  }
  std::set<std::string> outputs;
  for (const auto& r : rows)
    if (!outputs.insert(r.second).second) fail(2, "ERROR: %s: two %s write '%s'\n", kind.option, kind.rows, r.second.c_str());
}

// The start files of one scene of --versioned_scenes; an empty path is none
struct VersionedRow {
  std::string initial, earlier;
  std::optional<std::string> record;  // none: the scene writes no record (scene 0: no --record_file)
};

// The --versioned_scenes file: one `MATCHES_FILE<TAB>OUTPUT_FILE<TAB>INITIAL_SOLUTION<TAB>EARLIER_RECORD<TAB>RECORD_FILE`
// per line (raw bytes; the last newline is optional; the last three fields may be empty), appended to `rows` and
// `vrows` (scene 0's rows first).  Exits 2 after one ERROR line for an unreadable file, a malformed line, or a file
// that two outputs or records (those of scene 0 included) would write.
void read_versioned_list(const std::string& path, StringPairs& rows, std::vector<VersionedRow>& vrows) {
  std::string text;
  if (!read_file(path, text)) fail(2, "ERROR: cannot read the scene list file '%s'\n", path.c_str());
  const std::vector<std::string> lines = lines_of(text);
  for (size_t k = 0; k < lines.size(); ++k) {
    const std::string& l = lines[k];
    std::vector<std::string> f;
    for (size_t at = 0;;) {
      const size_t tab = l.find('\t', at);
      f.push_back(l.substr(at, tab == std::string::npos ? std::string::npos : tab - at));
      if (tab == std::string::npos) break;
      at = tab + 1;
    }
    const char* why = l.empty()                                ? "it is empty"
                      : f.size() < 5                           ? "it has fewer than four TABs"
                      : f.size() > 5                           ? "it has more than four TABs"
                      : f[0].empty()                           ? "its matches file is empty"
                      : f[1].empty()                           ? "its output file is empty"
                      : l.find('\0') != std::string::npos      ? "it holds a NUL byte"
                      : f[2].empty() && !f[3].empty()          ? "it has an earlier record but no initial solution"
                                                               : nullptr;
    if (why)
      fail(2, "ERROR: --versioned_scenes: line %zu is not MATCHES_FILE<TAB>OUTPUT_FILE<TAB>INITIAL_SOLUTION<TAB>"
              "EARLIER_RECORD<TAB>RECORD_FILE: %s\n", k + 1, why);
    rows.emplace_back(f[0], f[1]);
    vrows.push_back({f[2], f[3], f[4].empty() ? std::optional<std::string>() : f[4]});
  }
  std::set<std::string> written;
  for (size_t i = 0; i < rows.size(); ++i)
    for (const std::string* w : {&rows[i].second, vrows[i].record ? &*vrows[i].record : nullptr})
      if (w && !w->empty() && !written.insert(*w).second) fail(2, "ERROR: --versioned_scenes: two files written are '%s'\n", w->c_str());
}

// The --listed_pairs file: one match list per line (read_tab_list, appended to `rows` after list 0, every pair of
// --matches_file), every match list read and split as compute_match_graph.py:97 splits it (the newline stripped,
// single spaces; exactly two fields).  The lines (NAME1, NAME2) of every list, none for list 0.  Exits 2 after one
// ERROR line for what read_tab_list refuses, an unreadable match list or a malformed line of one, in that order.
std::vector<StringPairs> read_pair_lists(const std::string& path, StringPairs& rows) {
  read_tab_list(kPairList, path, rows);
  std::vector<StringPairs> lists(rows.size());
  for (size_t i = 1; i < rows.size(); ++i) {
    const std::string& list = rows[i].first;
    std::string text;
    if (!read_file(list, text)) fail(2, "ERROR: --listed_pairs: line %zu: cannot read the match list '%s'\n", i, list.c_str());
    const std::vector<std::string> lines = lines_of(text);
    for (size_t j = 0; j < lines.size(); ++j) {
      const std::string& l = lines[j];
      const size_t fields = 1 + (size_t)std::count(l.begin(), l.end(), ' ');
      if (fields != 2)
        fail(2, "ERROR: --listed_pairs: line %zu of the match list '%s' is not NAME1 NAME2: it has %zu fields\n", j + 1,
             list.c_str(), fields);
      const size_t sp = l.find(' ');
      lists[i].emplace_back(l.substr(0, sp), l.substr(sp + 1));
    }
  }
  return lists;
}

// The earlier MatchingFile of --previous_matches_file, decoded on the host: its image names by id (in order of
// first appearance over its parts) and the flat arrays of its lfr_host_input, no image banned.
struct PreviousMatches {
  std::vector<std::string> names;
  std::vector<uint8_t> name_blob;
  std::vector<uint64_t> name_off{0};
  std::vector<uint32_t> pair_img1, pair_img2, feat1, feat2;
  std::vector<uint64_t> pair_ptr{0};
  std::vector<float> sim, disp1, disp2;
  lfr_host_input input() const {
    lfr_host_input in;
    std::memset(&in, 0, sizeof in);
    in.n_pairs = pair_img1.size(); in.n_matches = feat1.size(); in.n_images = (uint32_t)names.size();
    in.pair_img1 = pair_img1.data(); in.pair_img2 = pair_img2.data(); in.pair_ptr = pair_ptr.data();
    in.feat1 = feat1.data(); in.feat2 = feat2.data(); in.sim = sim.data(); in.disp1 = disp1.data(); in.disp2 = disp2.data();
    return in;
  }
};

// Read and decode the earlier MatchingFile `path` (or its .part.N pieces, as --matches_file): 0, 2 when no
// file can be read, 255 when the bytes do not parse.
int read_previous(const std::string& path, PreviousMatches& pm) {
  const std::vector<std::string> files = matching_files(path);
  if (files.empty()) return 2;
  NameTable names;
  for (const std::string& f : files) {
    Part pt;
    if (const int rc = pt.open(f)) return rc;
    const uint64_t m0 = pm.feat1.size();
    pm.feat1.resize(m0 + pt.M); pm.feat2.resize(m0 + pt.M); pm.sim.resize(m0 + pt.M);
    pm.disp1.resize(18 * (m0 + pt.M)); pm.disp2.resize(18 * (m0 + pt.M));
    lfr_wire_matches w = pt.pair_level(pm.feat1.data() + m0, pm.feat2.data() + m0, pm.sim.data() + m0,
                                       pm.disp1.data() + 18 * m0, pm.disp2.data() + 18 * m0);
    if (lfr_wire_decode_matches(pt.buf.data(), pt.buf.size(), &w) != LFR_OK) return 255;
    for (uint64_t p = 0; p < pt.P; ++p) {
      pm.pair_img1.push_back(names.intern(pt, pt.n1_off[p], pt.n1_len[p]));
      pm.pair_img2.push_back(names.intern(pt, pt.n2_off[p], pt.n2_len[p]));
      pm.pair_ptr.push_back(m0 + pt.pair_ptr[p + 1]);
    }
    pt.buf.release();
  }
  pm.names = std::move(names.names);
  for (const std::string& s : pm.names) {
    pm.name_blob.insert(pm.name_blob.end(), s.begin(), s.end());
    pm.name_off.push_back(pm.name_blob.size());
  }
  if (pm.name_blob.empty()) pm.name_blob.push_back(0);
  return 0;
}

// The start of one scene of --versioned_scenes: its solution and earlier record, when it has them
struct SceneStart {
  bool has_file = false, has_record = false;
  std::vector<uint8_t> file, record;
};

// What the start point reads besides the MatchingFiles: the start solution (mapped while the run needs it), the
// earlier MatchingFile and the earlier record; with --versioned_scenes every scene's start, scene 0's copied from
// the first two, and the argument arrays of the grouped update
struct StartInputs {
  FileImage file;
  PreviousMatches previous;
  std::vector<uint8_t> earlier_record;
  std::vector<SceneStart> scenes;
  std::vector<const uint8_t*> files, records;  // NULL: none
  std::vector<uint64_t> file_len, record_len;
  bool any_file = false;
  void point() {
    for (const SceneStart& sc : scenes) {
      files.push_back(sc.has_file ? (sc.file.empty() ? &kEmpty : sc.file.data()) : nullptr);
      file_len.push_back(sc.file.size());
      records.push_back(sc.has_record ? sc.record.data() : nullptr);
      record_len.push_back(sc.record.size());
      any_file = any_file || sc.has_file;
    }
  }
  static constexpr uint8_t kEmpty = 0;  // the bytes of an empty SolutionFile
};

// Read and check the start inputs before any other work, so that their errors come before any output
void read_start_inputs(const Options& o, StartInputs& si) {
  if (!o.initial_solution.empty()) {
    if (!si.file.open(o.initial_solution))
      fail(2, "ERROR: cannot read the initial solution file '%s'\n", o.initial_solution.c_str());
    uint64_t ni = 0, nd = 0;
    if (lfr_wire_decode_solution(si.file.data(), si.file.size(), &ni, &nd, nullptr, nullptr, nullptr, nullptr, nullptr,
                                 nullptr, nullptr) != LFR_OK)
      fail(255, "Failed to parse proto object.\n");  // as for the matches, solve.cc:433-436
  }
  if (o.previous_matches_file) {
    const int rc = read_previous(*o.previous_matches_file, si.previous);
    if (rc == 2) fail(2, "ERROR: cannot read the previous matches file '%s'\n", o.previous_matches_file->c_str());
    if (rc != 0) fail(255, "Failed to parse proto object.\n");
  }
  if (o.earlier_record_file) {
    const std::string& path = *o.earlier_record_file;
    std::string text;
    if (!read_file(path, text)) fail(2, "ERROR: cannot read the earlier record file '%s'\n", path.c_str());
    si.earlier_record.assign(text.begin(), text.end());
    if (!lfr::record::check(si.earlier_record.data(), si.earlier_record.size(), nullptr))
      fail(2, "ERROR: '%s' is not a problem record\n", path.c_str());
  }
}

// --versioned_scenes: every scene's start files read and checked (scene 0's by read_start_inputs(), before),
// in scene order, before any other work.  Exits 2 after one ERROR line naming the list's line.
void read_versioned_starts(const std::vector<VersionedRow>& vrows, StartInputs& si) {
  si.scenes.resize(vrows.size());
  SceneStart& s0 = si.scenes[0];
  s0.has_file = !vrows[0].initial.empty();
  s0.file.assign(si.file.data(), si.file.data() + si.file.size());
  s0.has_record = !vrows[0].earlier.empty();
  s0.record = si.earlier_record;
  for (size_t k = 1; k < vrows.size(); ++k) {
    SceneStart& sc = si.scenes[k];
    const VersionedRow& v = vrows[k];
    std::string text;
    if (!v.initial.empty()) {
      if (!read_file(v.initial, text))
        fail(2, "ERROR: --versioned_scenes: line %zu: cannot read the initial solution file '%s'\n", k, v.initial.c_str());
      sc.file.assign(text.begin(), text.end());
      sc.has_file = true;
      uint64_t ni = 0, nd = 0;
      if (lfr_wire_decode_solution(sc.file.data(), sc.file.size(), &ni, &nd, nullptr, nullptr, nullptr, nullptr, nullptr,
                                   nullptr, nullptr) != LFR_OK)
        fail(2, "ERROR: --versioned_scenes: line %zu: the initial solution file '%s' does not parse\n", k, v.initial.c_str());
    }
    if (!v.earlier.empty()) {
      if (!read_file(v.earlier, text))
        fail(2, "ERROR: --versioned_scenes: line %zu: cannot read the earlier record file '%s'\n", k, v.earlier.c_str());
      sc.record.assign(text.begin(), text.end());
      sc.has_record = true;
      if (!lfr::record::check(sc.record.data(), sc.record.size(), nullptr))
        fail(2, "ERROR: --versioned_scenes: line %zu: '%s' is not a problem record\n", k, v.earlier.c_str());
    }
  }
  si.point();
}

// The pairs of all parts in order, with the batch member (scene) of every pair; image ids in order of first
// appearance over all parts.  With --listed_pairs, select_listed_pairs() makes them the lists' pairs.
struct Pairs {
  std::vector<Part> parts;
  NameTable names;
  uint64_t P = 0, M = 0, M_file = 0;  // M_file: the matches the decode reads, the file's
  std::vector<uint32_t> img1, img2, member;
  std::vector<float> fact1, fact2;
  std::vector<uint64_t> ptr;
  std::vector<uint64_t> src, file_ptr;  // --listed_pairs alone: the file's pair behind every pair, the file's pair_ptr
};

// solve.cc:412-481: the parts of every scene's MatchingFile mapped and walked.  Exits 255 when one does not parse.
Pairs read_pairs(const StringPairs& scenes) {
  Pairs ps;
  std::vector<std::string> files;
  std::vector<uint32_t> part_member;
  for (uint32_t sc = 0; sc < scenes.size(); ++sc)
    for (const std::string& f : matching_files(scenes[sc].first)) {
      files.push_back(f);
      part_member.push_back(sc);
    }
  ps.parts.resize(files.size());
  for (size_t i = 0; i < files.size(); ++i) {
    Part& pt = ps.parts[i];
    bool ok = pt.open(files[i]) == 0;
    if (ok) {
      pt.match_off.resize(pt.M);
      lfr_wire_matches w = pt.pair_level(nullptr, nullptr, nullptr, nullptr, nullptr);
      ok = lfr_wire_walk_matches(pt.buf.data(), pt.buf.size(), &w, pt.match_off.data()) == LFR_OK;
    }
    if (!ok) fail(255, "Failed to parse proto object.\n");  // solve.cc:433-436
  }
  for (const Part& pt : ps.parts) { ps.P += pt.P; ps.M += pt.M; }
  ps.M_file = ps.M;
  ps.img1.resize(ps.P); ps.img2.resize(ps.P); ps.member.resize(ps.P);
  ps.fact1.resize(ps.P); ps.fact2.resize(ps.P);
  ps.ptr.assign(ps.P + 1, 0);
  uint64_t p0 = 0, m0 = 0;
  for (size_t i = 0; i < ps.parts.size(); ++i) {
    const Part& pt = ps.parts[i];
    for (uint64_t p = 0; p < pt.P; ++p) {
      ps.member[p0 + p] = part_member[i];
      ps.img1[p0 + p] = ps.names.intern(pt, pt.n1_off[p], pt.n1_len[p]);
      ps.img2[p0 + p] = ps.names.intern(pt, pt.n2_off[p], pt.n2_len[p]);
      ps.fact1[p0 + p] = pt.fact1[p];
      ps.fact2[p0 + p] = pt.fact2[p];
      ps.ptr[p0 + p + 1] = m0 + pt.pair_ptr[p + 1];
    }
    p0 += pt.P;
    m0 += pt.M;
  }
  return ps;
}

// --listed_pairs: the batch's pairs are the lists' lines, list after list, each the first pair of the file
// with exactly those two names (one map over the pairs, names as bytes); every pair of the file for list 0.
// `rows` holds every list's path first.
// ps.src is the file's pair behind each of them, whose matches are copied to it after the decode.  Exits 2 after
// one ERROR line for a line whose pair the file does not hold.
void select_listed_pairs(Pairs& ps, const StringPairs& rows, const std::vector<StringPairs>& lists) {
  std::unordered_map<uint64_t, uint64_t> first;  // image1 << 32 | image2 -> the first pair
  for (uint64_t p = 0; p < ps.P; ++p) first.emplace((uint64_t)ps.img1[p] << 32 | ps.img2[p], p);
  const auto& id_of = ps.names.id_of;
  std::vector<uint32_t> list_of;
  for (size_t l = 0; l < lists.size(); ++l) {
    if (l == 0) {
      for (uint64_t p = 0; p < ps.P; ++p) {
        ps.src.push_back(p);
        list_of.push_back((uint32_t)l);
      }
      continue;
    }
    for (size_t j = 0; j < lists[l].size(); ++j) {
      const std::string& n1 = lists[l][j].first;
      const std::string& n2 = lists[l][j].second;
      const auto i1 = id_of.find(n1), i2 = id_of.find(n2);
      auto hit = first.end();
      bool reverse = false;
      if (i1 != id_of.end() && i2 != id_of.end()) {
        hit = first.find((uint64_t)i1->second << 32 | i2->second);
        reverse = first.count((uint64_t)i2->second << 32 | i1->second) != 0;
      }
      if (hit == first.end()) {
        std::fprintf(stderr, "ERROR: --listed_pairs: line %zu of the match list '%s': the matches file holds no pair '%s' '%s'",
                     j + 1, rows[l].first.c_str(), n1.c_str(), n2.c_str());
        if (reverse) std::fprintf(stderr, "; it holds only '%s' '%s'", n2.c_str(), n1.c_str());
        fail(2, "\n");
      }
      ps.src.push_back(hit->second);
      list_of.push_back((uint32_t)l);
    }
  }
  const uint64_t Q = ps.src.size();
  std::vector<uint32_t> img1(Q), img2(Q);
  std::vector<float> f1(Q), f2(Q);
  std::vector<uint64_t> ptr(Q + 1, 0);
  for (uint64_t k = 0; k < Q; ++k) {
    const uint64_t p = ps.src[k];
    img1[k] = ps.img1[p]; img2[k] = ps.img2[p]; f1[k] = ps.fact1[p]; f2[k] = ps.fact2[p];
    ptr[k + 1] = ptr[k] + (ps.ptr[p + 1] - ps.ptr[p]);
  }
  ps.img1.swap(img1); ps.img2.swap(img2); ps.fact1.swap(f1); ps.fact2.swap(f2);
  ps.file_ptr.swap(ps.ptr);
  ps.ptr.swap(ptr);
  ps.member.swap(list_of);
  ps.P = Q;
  ps.M = ps.ptr[Q];
}

// The graph stage's input, and everything indexed by its image ids: the original ids, or with sub-scenes one id
// per (sub-scene, image) in order of first appearance
struct Staged {
  lfr_host_input in;
  std::vector<uint8_t> skip;
  std::vector<uint32_t> orig_of, image_group;  // the original image id and the sub-scene of every id
  std::vector<float> image_fact;
  std::vector<uint8_t> fixed, written;
  bool any_fixed = false;
  std::vector<uint8_t> name_blob;
  std::vector<uint64_t> name_off;
  uint64_t e_cap = 0;  // the edge records of the pairs kept
  uint32_t n_ids() const { return (uint32_t)orig_of.size(); }
};

// The pairs as the graph stage takes them (their image ids become stage ids).  Exits 2 after one ERROR line for a
// pair that names two query images without --joint_queries, or for more than 65535 stage ids.
Staged stage(Pairs& ps, const Options& o, const Labelling& lab) {
  Staged st;
  const std::vector<std::string>& names = ps.names.names;
  const bool queries = lab.kind == Labelling::kQueries;
  const uint64_t P = ps.P;
  // banned images (solve.cc:444-446)
  const std::set<std::string> banned(o.banned_images.begin(), o.banned_images.end());
  st.skip.assign(P, 0);
  for (uint64_t p = 0; p < P; ++p) st.skip[p] = (banned.count(names[ps.img1[p]]) || banned.count(names[ps.img2[p]])) ? 1 : 0;

  // --query_images: a kept pair that names a query image belongs to that query's group's sub-scene, and its
  // images get that sub-scene's ids, in order of first appearance; a pair that names none is not solved.  A
  // group is one query, or with --joint_queries a connected component of the queries under the kept pairs
  // that name two of them (with or without matches).  The graph stage then gives every sub-scene what a run
  // on its pairs alone gives (lfr_host_input::image_group).  --additional_scenes: the same rule with every
  // kept pair in its scene's sub-scene, labelled by the scene index, so that scenes that share image names
  // share no node and each meta-component is cut at its own scene's image count.  --listed_pairs: the same with
  // the list index as the label, so a pair listed by two lists is a node set of each.
  std::vector<uint8_t> is_query(names.size(), 0);
  if (lab.kind != Labelling::kNone) {
    const std::set<std::string> query_names(o.query_images.begin(), o.query_images.end());
    for (size_t i = 0; i < names.size(); ++i) is_query[i] = query_names.count(names[i]) ? 1 : 0;
    // the group of every query image: a union-find whose root is the group's lowest image id, its label.  It
    // runs over all pairs before any id is handed out, since a later pair can merge two groups that hold ids.
    std::vector<uint32_t> group_of(names.size());
    for (uint32_t i = 0; i < (uint32_t)names.size(); ++i) group_of[i] = i;
    auto find = [&](uint32_t x) {
      while (group_of[x] != x) x = group_of[x] = group_of[group_of[x]];
      return x;
    };
    for (uint64_t p = 0; queries && p < P; ++p) {
      const uint32_t a = ps.img1[p], b = ps.img2[p];
      if (st.skip[p] || !is_query[a] || !is_query[b]) continue;
      if (!o.joint_queries) fail(2, "ERROR: the pair '%s' - '%s' names two query images\n", names[a].c_str(), names[b].c_str());
      const uint32_t ra = find(a), rb = find(b);
      group_of[std::max(ra, rb)] = std::min(ra, rb);
    }
    std::map<std::pair<uint32_t, uint32_t>, uint32_t> sub_id;  // (group, image) -> stage image id
    auto sub = [&](uint32_t g, uint32_t img) {
      const auto it = sub_id.emplace(std::make_pair(g, img), (uint32_t)st.orig_of.size());
      if (it.second) {
        st.orig_of.push_back(img);
        st.image_group.push_back(g);
      }
      return it.first->second;
    };
    for (uint64_t p = 0; p < P; ++p) {
      const uint32_t a = ps.img1[p], b = ps.img2[p];
      if (st.skip[p] || (queries && !(is_query[a] || is_query[b]))) {
        st.skip[p] = 1;
        ps.img1[p] = ps.img2[p] = 0;  // never read: skipped pairs name no image of the stage
        continue;
      }
      const uint32_t g = queries ? find(is_query[a] ? a : b) : ps.member[p];
      ps.img1[p] = sub(g, a);
      ps.img2[p] = sub(g, b);
    }
    if (st.orig_of.size() > 65535)
      fail(2, "ERROR: %s: the %s hold %zu images, more than 65535; split the %s over several runs\n", lab.option,
           lab.members, st.orig_of.size(), lab.list);
  } else {
    st.orig_of.resize(names.size());
    for (uint32_t i = 0; i < (uint32_t)names.size(); ++i) st.orig_of[i] = i;
  }
  const uint32_t n_ids = st.n_ids();

  // the first fact seen of every image among the pairs kept
  st.image_fact.assign(n_ids, 0.f);
  std::vector<uint8_t> have_fact(n_ids, 0);
  for (uint64_t p = 0; p < P; ++p) {
    if (st.skip[p]) continue;
    st.e_cap += 2 * (ps.ptr[p + 1] - ps.ptr[p]);
    if (!have_fact[ps.img1[p]]) { have_fact[ps.img1[p]] = 1; st.image_fact[ps.img1[p]] = ps.fact1[p]; }
    if (!have_fact[ps.img2[p]]) { have_fact[ps.img2[p]] = 1; st.image_fact[ps.img2[p]] = ps.fact2[p]; }
  }

  // images held fixed (the same name semantics as banned images), and the names by image id as the
  // start-point join and the encoder on the GPU take them (ids of the graph stage: with --query_images a
  // database image's name repeats once per sub-scene, and the joins give every copy the same entries)
  const std::set<std::string> fixed_names(o.fixed_images.begin(), o.fixed_images.end());
  st.fixed.assign(n_ids, 0);
  st.written.assign(n_ids, 0);
  for (uint32_t i = 0; i < n_ids; ++i) {
    st.written[i] = !queries || is_query[st.orig_of[i]];
    if (fixed_names.count(names[st.orig_of[i]])) {
      st.fixed[i] = 1;
      st.any_fixed = true;
    }
  }
  st.name_off.assign(n_ids + 1, 0);
  for (uint32_t i = 0; i < n_ids; ++i) {
    const std::string& nm = names[st.orig_of[i]];
    st.name_blob.insert(st.name_blob.end(), nm.begin(), nm.end());
    st.name_off[i + 1] = st.name_blob.size();
  }

  std::memset(&st.in, 0, sizeof st.in);
  st.in.n_pairs = P; st.in.n_matches = ps.M; st.in.n_images = n_ids;
  st.in.pair_img1 = ps.img1.data(); st.in.pair_img2 = ps.img2.data(); st.in.pair_skip = st.skip.data();
  st.in.pair_ptr = ps.ptr.data();
  st.in.image_group = lab.kind != Labelling::kNone ? st.image_group.data() : nullptr;
  return st;
}

// Which graph stage: the library's size rule, or LFR_GRAPH_STAGE=host|device (a test and measurement hook, not a
// product option).  A library without the stage on the GPU — the CPU checker — takes the host route; forcing the
// device route there is an error, never a silent host run.
bool device_route(const lfr_host_input& in, uint64_t gpus) {
  const bool have_device_stage = lfr_graph_stage_on_device && lfr_wire_decode_on_device && lfr_plan_create_from_matches &&
                                 lfr_plan_create_from_wire && lfr_plan_encode_solution && lfr_plan_fix_images &&
                                 lfr_plan_start_from_solution && lfr_plan_keep_solution && lfr_plan_encode_solution_carried &&
                                 lfr_plan_update_solution && lfr_plan_update_solution_since && lfr_plan_problem_record &&
                                 lfr_plan_update_solution_since_record && lfr_plan_encode_solution_images &&
                                 lfr_plan_encode_solution_groups && lfr_plan_create_from_wire_listed &&
                                 lfr_plan_update_solution_groups && lfr_plan_problem_record_groups;
  const bool on_device = have_device_stage && lfr_graph_stage_on_device(&in, (int32_t)gpus) == 1;
  const char* force = std::getenv("LFR_GRAPH_STAGE");
  if (!force || !*force) return on_device;
  if (std::strcmp(force, "host") == 0) return false;
  if (std::strcmp(force, "device") != 0) fail(2, "ERROR: LFR_GRAPH_STAGE must be 'host' or 'device'\n");
  if (!have_device_stage) fail(2, "ERROR: LFR_GRAPH_STAGE=device: the solve library has no graph stage on the GPU\n");
  if (gpus > 1) fail(2, "ERROR: LFR_GRAPH_STAGE=device: the graph stage on the GPU drives one device (--gpus 1)\n");
  return true;
}

// The decoded matches of every pair
struct Matches {
  std::vector<uint32_t> feat1, feat2;
  std::vector<float> sim, disp1, disp2;
};

// Host route, and the device route below the library's size for the decoder on the GPU: the matches of every part
// decoded into one set of arrays, part after part (the pair level comes out as the walk gave it), each part's
// mapping released after its decode.  With --listed_pairs the file is decoded once and every listed pair's matches
// are then copied into place.  Exits 255 when a part does not parse.
void decode_on_host(Pairs& ps, Matches& m, lfr_host_input& in) {
  const uint64_t M = ps.M_file;
  m.feat1.resize(M); m.feat2.resize(M); m.sim.resize(M); m.disp1.resize(18 * M); m.disp2.resize(18 * M);
  uint64_t m0 = 0;
  for (Part& pt : ps.parts) {
    lfr_wire_matches w = pt.pair_level(m.feat1.data() + m0, m.feat2.data() + m0, m.sim.data() + m0,
                                       m.disp1.data() + 18 * m0, m.disp2.data() + 18 * m0);
    if (lfr_wire_decode_matches(pt.buf.data(), pt.buf.size(), &w) != LFR_OK)
      fail(255, "Failed to parse proto object.\n");  // solve.cc:433-436
    m0 += pt.M;
    pt.buf.release();  // the file image (several GB at Madrid scale) is not needed past the decode
  }
  if (!ps.file_ptr.empty()) {  // --listed_pairs
    Matches e;
    e.feat1.resize(ps.M); e.feat2.resize(ps.M); e.sim.resize(ps.M); e.disp1.resize(18 * ps.M); e.disp2.resize(18 * ps.M);
    for (uint64_t k = 0; k < ps.P; ++k) {
      const uint64_t a = ps.file_ptr[ps.src[k]], c = ps.ptr[k + 1] - ps.ptr[k], b = ps.ptr[k];
      std::copy_n(m.feat1.begin() + a, c, e.feat1.begin() + b);
      std::copy_n(m.feat2.begin() + a, c, e.feat2.begin() + b);
      std::copy_n(m.sim.begin() + a, c, e.sim.begin() + b);
      std::copy_n(m.disp1.begin() + 18 * a, 18 * c, e.disp1.begin() + 18 * b);
      std::copy_n(m.disp2.begin() + 18 * a, 18 * c, e.disp2.begin() + 18 * b);
    }
    m = std::move(e);
  }
  in.feat1 = m.feat1.data(); in.feat2 = m.feat2.data(); in.sim = m.sim.data(); in.disp1 = m.disp1.data(); in.disp2 = m.disp2.data();
}

// Host memory that is page-locked when lfr_host_alloc() gives it (the copies to and from the GPU run at full
// speed) and malloc'ed otherwise, or malloc'ed alone when not `page_locked`; freed the matching way.
struct HostFree {
  bool pinned = false;
  void operator()(void* p) const { pinned ? lfr_host_free(p) : std::free(p); }
};
template <class T>
using HostArray = std::unique_ptr<T[], HostFree>;
template <class T>
HostArray<T> host_array(size_t n, bool page_locked = true) {
  if (void* p = page_locked ? lfr_host_alloc(n * sizeof(T)) : nullptr) return HostArray<T>(static_cast<T*>(p), HostFree{true});
  return HostArray<T>(static_cast<T*>(std::malloc(n ? n * sizeof(T) : 1)), HostFree{false});
}

struct PlanDestroy {
  void operator()(lfr_plan* p) const { lfr_plan_destroy(p); }
};
using PlanPtr = std::unique_ptr<lfr_plan, PlanDestroy>;

// --record_file: this run's problem record (include/lfr_graph.h), from the reference roots, by a size-then-fill
// call `fill(out, cap)`.  Exits 2 when it fails.
template <class Fill>
void problem_record(std::vector<uint8_t>& record, Fill fill) {
  const int64_t need = fill(nullptr, 0);
  record.resize(need > 0 ? (size_t)need : 0);
  const int64_t got = need < 0 ? need : fill(record.data(), record.size());
  if (got < 0 || (uint64_t)got != record.size()) fail_call("the problem record", (int)got);
}

using Clock = std::chrono::steady_clock;

void print_sizes(const lfr_host_sizes& sz) {
  std::printf("# graph nodes: %u\n", sz.n_nodes);                          // solve.cc:484
  std::printf("# graph edges: %llu\n", (unsigned long long)sz.n_edges);    // solve.cc:485
  if (sz.n_nodes) {
    std::printf("# tracks: %u\n", sz.n_tracks);                           // solve.cc:534
    std::printf("max track size: %u\n", sz.max_track_size);               // solve.cc:549
    std::printf("Graph-cut time: %lldms\n", (long long)sz.graph_cut_ms);  // solve.cc:589
    std::printf("# components: %u\n", sz.n_components);                  // solve.cc:591
    std::printf("max component size: %u\n", sz.max_component_size);       // solve.cc:606
  }
  std::fflush(stdout);
}

// "Solver time" from `t_solve` and "Total time" (solve.cc:487-641: the graph work and the solve) from `t_start`
void print_times(Clock::time_point t_start, Clock::time_point t_solve) {
  const Clock::time_point t_end = Clock::now();
  auto ms = [](Clock::duration d) { return (long long)std::chrono::duration_cast<std::chrono::milliseconds>(d).count(); };
  std::printf("Solver time: %lldms\n", ms(t_end - t_solve));  // solve.cc:638
  std::printf("Total time: %lldms\n", ms(t_end - t_start));   // solve.cc:641
}

// What a route gives: the SolutionFile of every output k, bytes[off[k], off[k + 1]), the count of
// solve.cc:666-669 and the problem record (with --versioned_scenes every scene's, record[record_off[k],
// record_off[k + 1]))
struct Result {
  HostArray<uint8_t> bytes;
  std::vector<uint64_t> off;
  uint64_t n_outside = 0;
  std::vector<uint8_t> record;
  std::vector<uint64_t> record_off;
  bool encoded = true;  // false: the host route's encoder failed, which solve.cc:674-677 reports as a write failure
};

// --versioned_scenes: every scene's problem record, by one call `fill(out, cap, group_off)` into a buffer sized for
// the `n_components` of the batch (16 bytes per header and per digest).  Exits 2 when it fails.
template <class Fill>
void problem_records(Result& r, size_t n_scenes, uint64_t n_components, Fill fill) {
  r.record.resize(16 * (n_scenes + n_components));
  r.record_off.assign(n_scenes + 1, 0);
  const int64_t got = fill(r.record.data(), r.record.size(), r.record_off.data());
  if (got < 0 || (uint64_t)got != r.record.size()) fail_call("the problem record", (int)got);
}

// Whether the run writes a problem record: --record_file (given, even with an empty path), or with
// --versioned_scenes any scene's RECORD_FILE
bool writes_records(const std::vector<VersionedRow>& vrows) {
  for (const VersionedRow& v : vrows)
    if (v.record) return true;
  return false;
}

// The device route: the graph stage on the GPU (include/lfr_graph.h), from the mapped parts or from `in`'s decoded
// matches; the problem stays in HBM for the solve and the SolutionFile is encoded there.
Result run_device(const Options& o, Start start, const Labelling& lab, Pairs& ps, const Staged& st, StartInputs& si,
                  size_t n_out, bool record, bool decode_on_device, Clock::time_point t_start) {
  lfr_options opt;
  lfr_options_default(&opt);
  opt.device = (int32_t)o.device;
  // LFR_DEVICE_CUT=1: the recursive cut on the device too (LFR_DBG_DEVICE_CUT; a test and measurement hook)
  if (const char* e = std::getenv("LFR_DEVICE_CUT")) {
    if (std::strcmp(e, "1") == 0) opt.debug_flags |= LFR_DBG_DEVICE_CUT;
  }
  std::vector<lfr_wire_part> wparts;
  for (const Part& pt : ps.parts) wparts.push_back(lfr_wire_part{pt.buf.data(), pt.buf.size(), pt.match_off.data(), pt.M});
  lfr_plan* created = nullptr;
  lfr_host_sizes sz;
  const int rc = decode_on_device && lab.kind == Labelling::kLists
                     ? lfr_plan_create_from_wire_listed(&st.in, wparts.data(), (uint32_t)wparts.size(), ps.file_ptr.data(),
                                                        ps.file_ptr.size() - 1, ps.src.data(), &opt, nullptr, &created, &sz)
                 : decode_on_device
                     ? lfr_plan_create_from_wire(&st.in, wparts.data(), (uint32_t)wparts.size(), &opt, nullptr, &created, &sz)
                     : lfr_plan_create_from_matches(&st.in, &opt, nullptr, &created, &sz);
  PlanPtr plan(created);
  for (Part& pt : ps.parts) pt.buf.release();
  if (rc == LFR_EINVAL && std::strcmp(lfr_last_error(), "malformed Match message") == 0)
    fail(255, "Failed to parse proto object.\n");  // solve.cc:433-436, as the host decode
  if (rc == LFR_EINVAL || rc == LFR_EUNSUPPORTED)  // the input, as the host stage would reject it
    fail(2, "ERROR: the host graph stage rejected the input\n");
  if (rc != LFR_OK) fail_call("the solve", rc);  // no device: the host route's message, from the same device check

  // problem initialisation (solve.cc:608-612) on the plan: the constant mask and the start point
  const uint32_t n_ids = st.n_ids();
  const uint8_t* names = st.name_blob.data();
  const uint64_t* name_off = st.name_off.data();
  const uint8_t* file = si.file.data();
  const uint64_t file_len = si.file.size();
  int rc2 = st.any_fixed ? lfr_plan_fix_images(plan.get(), st.fixed.data(), n_ids) : LFR_OK;
  if (rc2 == LFR_OK && start == Start::kScenes) {
    if (si.any_file)  // every scene from its own file and record, in one call; without any file all start at zero
      rc2 = lfr_plan_update_solution_groups(plan.get(), nullptr, n_ids, names, name_off, st.image_group.data(), (uint32_t)n_out,
                                            si.files.data(), si.file_len.data(), si.records.data(), si.record_len.data(),
                                            nullptr, nullptr, nullptr);
  } else if (rc2 == LFR_OK && start == Start::kUpdateSinceRecord) {
    rc2 = lfr_plan_update_solution_since_record(plan.get(), nullptr, file, file_len, n_ids, names, name_off,
                                                si.earlier_record.data(), si.earlier_record.size(), nullptr, nullptr,
                                                nullptr);
  } else if (rc2 == LFR_OK && start == Start::kUpdateSinceMatches) {
    // the earlier run's graph stage on the device, for the compare only
    const PreviousMatches& pm = si.previous;
    const lfr_host_input pin = pm.input();
    lfr_plan* created_prev = nullptr;
    rc2 = lfr_plan_create_from_matches(&pin, &opt, nullptr, &created_prev, nullptr);
    const PlanPtr prev(created_prev);
    if (rc2 == LFR_OK)
      rc2 = lfr_plan_update_solution_since(plan.get(), nullptr, file, file_len, n_ids, names, name_off, prev.get(),
                                           (uint32_t)pm.names.size(), pm.name_blob.data(), pm.name_off.data(), nullptr,
                                           nullptr, nullptr);
  } else if (rc2 == LFR_OK && start == Start::kUpdate) {
    rc2 = lfr_plan_update_solution(plan.get(), nullptr, file, file_len, n_ids, names, name_off, nullptr, nullptr);
  } else if (rc2 == LFR_OK && start != Start::kZeros) {
    rc2 = (start == Start::kKeep ? lfr_plan_keep_solution : lfr_plan_start_from_solution)(
        plan.get(), nullptr, file, file_len, n_ids, names, name_off, nullptr);
  }
  if (rc2 != LFR_OK) fail_call("the solve", rc2);
  print_sizes(sz);

  if (!o.carry_initial_solution) si.file.release();  // carried into the output otherwise
  const Clock::time_point t_solve = Clock::now();
  if (sz.n_nodes) {
    int rc3 = lfr_plan_solve(plan.get(), nullptr);
    if (rc3 == LFR_OK) rc3 = lfr_plan_download(plan.get(), nullptr, nullptr, nullptr);  // waits for the solve, checks its error flag
    if (rc3 != LFR_OK) fail_call("the solve", rc3);
  }
  print_times(t_start, t_solve);

  Result r;
  if (record && start == Start::kScenes)
    problem_records(r, n_out, sz.n_components, [&](uint8_t* out, uint64_t cap, uint64_t* group_off) {
      return lfr_plan_problem_record_groups(plan.get(), nullptr, n_ids, names, name_off, st.image_group.data(),
                                            (uint32_t)n_out, out, cap, group_off);
    });
  else if (record)
    problem_record(r.record, [&](uint8_t* out, uint64_t cap) {
      return lfr_plan_problem_record(plan.get(), nullptr, n_ids, names, name_off, out, cap);
    });

  // ---- SolutionFile (solve.cc:643-679), encoded on the GPU, names and facts indexed by image id, into
  // page-locked memory sized by the largest encoding: a Displacement record is at most 18 bytes, an Image's
  // header 16 plus its name field
  uint64_t cap = 18ull * sz.n_nodes;
  cap += 27ull * n_ids + st.name_blob.size();
  // carried entries: a file's canonical encoding bounds what it adds; a larger need takes a second call
  if (o.carry_initial_solution) cap += si.file.size();
  r.off.assign(n_out + 1, 0);
  std::vector<uint64_t> outside(n_out, 0);
  const float* fact = st.image_fact.data();
  auto encode = [&](uint8_t* out, uint64_t c) {
    return o.carry_initial_solution
               ? lfr_plan_encode_solution_carried(plan.get(), nullptr, n_ids, names, name_off, fact, si.file.data(),
                                                  si.file.size(), out, c, &r.n_outside, nullptr)
           : lab.kind == Labelling::kQueries
               ? lfr_plan_encode_solution_images(plan.get(), nullptr, n_ids, names, name_off, fact, st.written.data(),
                                                 out, c, &r.n_outside)
           : lab.batched()
               ? lfr_plan_encode_solution_groups(plan.get(), nullptr, n_ids, names, name_off, fact, st.image_group.data(),
                                                 (uint32_t)n_out, out, c, r.off.data(), outside.data())
               : lfr_plan_encode_solution(plan.get(), nullptr, n_ids, names, name_off, fact, out, c, &r.n_outside);
  };
  r.bytes = host_array<uint8_t>(cap);
  int64_t need = encode(r.bytes.get(), cap);
  if (need > 0 && (uint64_t)need > cap) {
    r.bytes.reset();
    cap = (uint64_t)need;
    r.bytes = host_array<uint8_t>(cap);
    need = encode(r.bytes.get(), cap);
  }
  plan.reset();
  if (need < 0 || (uint64_t)need > cap) fail_call("the solve", (int)need);
  if (lab.batched())
    for (uint64_t c : outside) r.n_outside += c;
  else
    r.off[1] = (uint64_t)need;
  return r;
}

// The host route: the host graph stage (solve.cc:438-606) writing the edge records straight into page-locked
// memory, the start point joined on the host, lfr_solve() / lfr_solve_multi() and the output assembly.
Result run_host(const Options& o, Start start, const Labelling& lab, const Pairs& ps, Staged& st, StartInputs& si,
                size_t n_out, bool record, Clock::time_point t_start) {
  const HostArray<lfr_edge> edges_buf = st.e_cap ? host_array<lfr_edge>(st.e_cap) : nullptr;
  lfr_edge* edges = edges_buf.get();
  st.in.edges_out = edges; st.in.edges_out_capacity = st.e_cap;
  lfr_host_stage* hs = nullptr;
  lfr_host_sizes sz;
  if (lfr_host_stage_create(&st.in, &hs, &sz) != LFR_OK) fail(2, "ERROR: the host graph stage rejected the input\n");
  const uint32_t N = sz.n_nodes, C = sz.n_components;
  std::vector<uint32_t> row_ptr((size_t)N + 1, 0), track(N), comp(N), comp_ptr((size_t)C + 1, 0), comp_nodes(N),
      comp_order(C), node_image(N), node_feat(N);
  std::vector<uint8_t> is_root(N);
  const int rc = lfr_host_stage_export(hs, row_ptr.data(), edges, track.data(), comp.data(), is_root.data(),
                                       comp_ptr.data(), comp_nodes.data(), comp_order.data(), node_image.data(),
                                       node_feat.data());
  lfr_host_stage_destroy(hs);
  if (rc != LFR_OK) fail(2, "ERROR: lfr_host_stage_export failed\n");
  // the problem with the reference's is_root (the update since an earlier run and the record read it)
  lfr_problem prob;
  prob.n_nodes = N; prob.n_components = C; prob.n_edges = sz.n_edges;
  prob.row_ptr = row_ptr.data(); prob.edges = edges; prob.track = track.data(); prob.comp = comp.data();
  prob.is_root = is_root.data(); prob.comp_ptr = comp_ptr.data(); prob.comp_nodes = comp_nodes.data();
  print_sizes(sz);

  // ---- the solve (solve.cc:608-635): positions start at zero, or from --initial_solution -----
  const uint32_t n_ids = st.n_ids();
  const uint8_t* names = st.name_blob.data();
  const uint64_t* name_off = st.name_off.data();
  const uint8_t* file = si.file.data();
  const uint64_t file_len = si.file.size();
  HostArray<double> positions_buf;
  double* positions = nullptr;
  // with --fixed_images, --keep_initial_solution or an update: reference roots OR nodes of fixed images OR nodes
  // with an entry in the start solution (kept) or held by the update
  std::vector<uint8_t> is_const;
  const bool any_const = st.any_fixed || holds_entries(start);
  if (N) {
    positions_buf = host_array<double>(2ull * N);
    positions = positions_buf.get();
    std::memset(positions, 0, 2ull * N * sizeof(double));
    std::vector<uint8_t> has_entry(holds_entries(start) ? N : 0, 0);
    if (start == Start::kScenes) {
      if (si.any_file &&
          lfr_wire_update_solution_groups(n_ids, names, name_off, st.image_group.data(), (uint32_t)n_out, si.files.data(),
                                          si.file_len.data(), si.records.data(), si.record_len.data(), &prob,
                                          node_image.data(), node_feat.data(), positions, has_entry.data(), nullptr,
                                          nullptr, nullptr) != LFR_OK)
        fail(2, "ERROR: lfr_wire_update_solution_groups failed\n");
    } else if (start == Start::kUpdateSinceRecord) {
      if (lfr_wire_update_solution_since_record(file, file_len, n_ids, names, name_off, &prob, node_image.data(),
                                                node_feat.data(), si.earlier_record.data(), si.earlier_record.size(),
                                                positions, has_entry.data(), nullptr, nullptr, nullptr) != LFR_OK)
        fail(2, "ERROR: lfr_wire_update_solution_since_record failed\n");
    } else if (start == Start::kUpdateSinceMatches) {
      const lfr_host_input pin = si.previous.input();
      if (lfr_wire_update_solution_since(file, file_len, n_ids, names, name_off, &prob, node_image.data(),
                                         node_feat.data(), &pin, si.previous.name_blob.data(), si.previous.name_off.data(),
                                         positions, has_entry.data(), nullptr, nullptr, nullptr) != LFR_OK)
        fail(2, "ERROR: lfr_wire_update_solution_since failed\n");
    } else if (start == Start::kUpdate) {
      if (lfr_wire_update_solution(file, file_len, n_ids, names, name_off, N, node_image.data(), node_feat.data(),
                                   comp.data(), C, positions, has_entry.data(), nullptr, nullptr) != LFR_OK)
        fail(2, "ERROR: lfr_wire_update_solution failed\n");
    } else if (start != Start::kZeros &&
               (start == Start::kKeep
                    ? lfr_wire_join_solution_entries(file, file_len, n_ids, names, name_off, N, node_image.data(),
                                                     node_feat.data(), positions, nullptr, has_entry.data())
                    : lfr_wire_join_solution(file, file_len, n_ids, names, name_off, N, node_image.data(),
                                             node_feat.data(), positions, nullptr)) != LFR_OK) {
      fail(2, "ERROR: lfr_wire_join_solution failed\n");
    }
    if (any_const) {
      is_const.resize(N);
      for (uint32_t v = 0; v < N; ++v)
        is_const[v] = (is_root[v] || st.fixed[node_image[v]] || (holds_entries(start) && has_entry[v])) ? 1 : 0;
    }
  }
  if (!o.carry_initial_solution) si.file.release();  // carried into the output otherwise
  const Clock::time_point t_solve = Clock::now();
  if (N) {
    lfr_problem solve_prob = prob;
    if (any_const) solve_prob.is_root = is_const.data();
    lfr_options opt;
    lfr_options_default(&opt);
    opt.device = (int32_t)o.device;
    lfr_stats stats;
    std::memset(&stats, 0, sizeof stats);
    int rc3;
    if (o.gpus > 1) {
      std::vector<int32_t> devs((size_t)o.gpus);
      for (size_t i = 0; i < devs.size(); ++i) devs[i] = (int32_t)i;
      rc3 = lfr_solve_multi(&solve_prob, &opt, devs.data(), (int32_t)devs.size(), positions, &stats, nullptr);
    } else {
      rc3 = lfr_solve(&solve_prob, &opt, positions, &stats);
    }
    if (rc3 != LFR_OK) fail_call("the solve", rc3);  // no CPU fallback: without a CUDA device the program stops here
  }
  print_times(t_start, t_solve);

  Result r;
  if (record && start == Start::kScenes)
    problem_records(r, n_out, C, [&](uint8_t* out, uint64_t cap, uint64_t* group_off) {
      return lfr_host_problem_record_groups(&prob, node_image.data(), node_feat.data(), n_ids, names, name_off,
                                            st.image_group.data(), (uint32_t)n_out, out, cap, group_off);
    });
  else if (record)
    problem_record(r.record, [&](uint8_t* out, uint64_t cap) {
      return lfr_host_problem_record(&prob, node_image.data(), node_feat.data(), n_ids, names, name_off, out, cap);
    });

  // ---- SolutionFile (solve.cc:643-679): images by first node appearance, nodes by index.  With --query_images
  // only the query images are written (a database image's keypoints have one value per query): rank -2 marks the
  // images left out; every node still counts towards n_outside
  std::vector<int64_t> rank(n_ids, -1);
  std::vector<uint32_t> img_ids;
  for (uint32_t v = 0; v < N; ++v)
    if (rank[node_image[v]] == -1) {
      if (!st.written[node_image[v]]) {
        rank[node_image[v]] = -2;
        continue;
      }
      rank[node_image[v]] = (int64_t)img_ids.size();
      img_ids.push_back(node_image[v]);
    }
  // with --additional_scenes (--listed_pairs) the images go scene (list) after scene, each one's in the order above
  std::vector<size_t> out_img(n_out + 1, 0);
  if (lab.batched()) {
    std::stable_sort(img_ids.begin(), img_ids.end(),
                     [&](uint32_t x, uint32_t y) { return st.image_group[x] < st.image_group[y]; });
    for (size_t i = 0; i < img_ids.size(); ++i) {
      rank[img_ids[i]] = (int64_t)i;
      ++out_img[st.image_group[img_ids[i]] + 1];
    }
    for (size_t k = 0; k < n_out; ++k) out_img[k + 1] += out_img[k];
  } else {
    out_img[1] = img_ids.size();
  }
  const size_t I = img_ids.size();
  std::vector<uint64_t> img_ptr(I + 1, 0);
  for (uint32_t v = 0; v < N; ++v)
    if (rank[node_image[v]] >= 0) ++img_ptr[(size_t)rank[node_image[v]] + 1];
  for (size_t i = 0; i < I; ++i) img_ptr[i + 1] += img_ptr[i];
  std::vector<uint32_t> feature_idx(img_ptr[I]);
  std::vector<float> di(img_ptr[I]), dj(img_ptr[I]);
  {
    std::vector<uint64_t> fill(img_ptr.begin(), img_ptr.end() - 1);
    for (uint32_t v = 0; v < N; ++v) {
      if (std::fabs(positions[2 * (size_t)v + 1]) > 0.5 || std::fabs(positions[2 * (size_t)v]) > 0.5) ++r.n_outside;  // solve.cc:666-669
      if (rank[node_image[v]] < 0) continue;
      const uint64_t k = fill[(size_t)rank[node_image[v]]]++;
      feature_idx[k] = node_feat[v];
      di[k] = (float)positions[2 * (size_t)v];
      dj[k] = (float)positions[2 * (size_t)v + 1];
    }
  }
  std::vector<uint8_t> out_blob;
  std::vector<uint64_t> out_off(I + 1, 0);
  std::vector<float> fact(I);
  for (size_t i = 0; i < I; ++i) {
    const std::string& s = ps.names.names[st.orig_of[img_ids[i]]];
    out_blob.insert(out_blob.end(), s.begin(), s.end());
    out_off[i + 1] = out_blob.size();
    fact[i] = st.image_fact[img_ids[i]];
  }
  if (out_blob.empty()) out_blob.push_back(0);
  // the images [a, b) of the output order: one output's SolutionFile
  auto encode = [&](size_t a, size_t b, uint8_t* out, uint64_t c) {
    return o.carry_initial_solution
               ? lfr_wire_encode_solution_carried(b - a, img_ptr.data() + a, out_blob.data(), out_off.data() + a,
                                                  fact.data() + a, feature_idx.data(), di.data(), dj.data(),
                                                  si.file.data(), si.file.size(), out, c, nullptr)
               : lfr_wire_encode_solution(b - a, img_ptr.data() + a, out_blob.data(), out_off.data() + a,
                                          fact.data() + a, feature_idx.data(), di.data(), dj.data(), out, c);
  };
  r.off.assign(n_out + 1, 0);
  int64_t need = 0;
  for (size_t k = 0; k < n_out && need >= 0; ++k) {
    const int64_t n = encode(out_img[k], out_img[k + 1], nullptr, 0);
    need = n < 0 ? -1 : need + n;
    r.off[k + 1] = (uint64_t)need;
  }
  r.bytes = host_array<uint8_t>((size_t)std::max<int64_t>(need, 1), false);
  for (size_t k = 0; k < n_out && need >= 0; ++k) {
    const uint64_t n = r.off[k + 1] - r.off[k];
    if (encode(out_img[k], out_img[k + 1], r.bytes.get() + r.off[k], n) != (int64_t)n) need = -1;
  }
  r.encoded = need >= 0;
  return r;
}

// The command line parsed into `o`, or the exit code of a run that ends there: 1 after Boost's error and the usage
// on stderr (solve.cc:397-401), 0 after --help
std::optional<int> parse_command_line(int argc, char** argv, Options& o) {
  try {
    o = parse(argc, argv);
  } catch (const CliError& e) {  // solve.cc:397-401
    std::fprintf(stderr, "ERROR: %s\n\n", e.msg.c_str());
    std::fputs(kUsage, stderr);
    return 1;
  }
  if (o.help) {
    std::fputs("Patch Match graph problem solver\n\n", stdout);
    std::fputs(kUsage, stdout);
    return 0;
  }
  return std::nullopt;
}

// What a process sets once for all its runs.  A one-shot process pays for CUDA's start-up (driver initialisation
// over every visible GPU, context creation: 0.4-0.8 s on an 8-GPU box) more than for all of its work on a
// Fountain-scale scene.  Two measures: only the device that will be used is made visible (unless the caller already
// chose), and the start-up runs on a helper thread while the first input is read, decoded and turned into a graph.
struct Process {
  uint64_t device = 0, gpus = 1;  // the device selection every run takes
  bool started = false;
  std::thread cuda_start;
  void start(const Options& o) {
    device = o.device;
    gpus = o.gpus;
    if (gpus <= 1 && !std::getenv("CUDA_VISIBLE_DEVICES")) {
      setenv("CUDA_VISIBLE_DEVICES", std::to_string(device).c_str(), 1);
      device = 0;
    }
    cuda_start = std::thread([] { lfr_host_free(lfr_host_alloc(64)); });
    started = true;
  }
  void ready() {  // page-locked memory needs the context
    if (cuda_start.joinable()) cuda_start.join();
  }
  ~Process() { ready(); }
};

// One run of the command line `o` under `proc`'s device selection, which it starts when no run has: everything from
// the rules to the record files.  Returns 0 or throws Exit; either way every file, mapping, plan and page-locked
// array it made is released by then (the library's per-device workspaces persist by design).
int run_task(Options o, Process& proc) {
  check_rules(o);
  const Start start = start_mode(o);
  const Labelling lab = labelling(o);

  // the batch's rows, each with its output file second: scene 0 / list 0 is --matches_file / --output_file, then
  // with --additional_scenes every listed scene (each scene's output is what its own run writes: the same command
  // with that scene's two files alone), or with --listed_pairs every listed match list (its output is what the same
  // command writes on a MatchingFile that holds the file's pair for every line of the list, in line order)
  // with --versioned_scenes every listed scene, whose output and record are what its own run writes: the same
  // command with that scene's files alone, updated from its initial solution (and earlier record) when it has one
  StringPairs rows{{o.matches_file, o.output_file}};
  std::vector<StringPairs> lists;
  std::vector<VersionedRow> vrows{{o.initial_solution, o.earlier_record_file.value_or(""), o.record_file}};
  if (o.listed_pairs) lists = read_pair_lists(*o.listed_pairs, rows);
  if (o.additional_scenes) read_tab_list(kSceneList, *o.additional_scenes, rows);
  if (o.versioned_scenes) read_versioned_list(*o.versioned_scenes, rows, vrows);
  StartInputs si;
  read_start_inputs(o, si);
  if (o.versioned_scenes) read_versioned_starts(vrows, si);
  const bool record = writes_records(vrows);

  if (!proc.started) proc.start(o);
  o.device = proc.device;
  o.gpus = proc.gpus;

  Pairs ps = read_pairs(o.listed_pairs ? StringPairs{rows[0]} : rows);  // the lists' pairs are --matches_file's
  if (o.listed_pairs) select_listed_pairs(ps, rows, lists);
  Staged st = stage(ps, o, lab);
  const bool on_device = device_route(st.in, o.gpus);
  // the decoder's threshold sees the file's match count
  const bool decode_on_device = on_device && lfr_wire_decode_on_device(ps.M_file) == 1;
  Matches matches;
  if (!decode_on_device) decode_on_host(ps, matches, st.in);

  proc.ready();
  const Clock::time_point t_start = Clock::now();
  Result r = on_device ? run_device(o, start, lab, ps, st, si, rows.size(), record, decode_on_device, t_start)
                       : run_host(o, start, lab, ps, st, si, rows.size(), record, t_start);
  si.file.release();
  std::printf("# points with at least one coordinate > 0.5: %llu\n", (unsigned long long)r.n_outside);  // solve.cc:670
  std::fflush(stdout);
  bool written = r.encoded;
  for (size_t k = 0; written && k < rows.size(); ++k) {  // in row order; the first failure ends the run
    std::ofstream f(rows[k].second, std::ios::binary | std::ios::trunc);
    written = f.good();
    const uint64_t n = r.off[k + 1] - r.off[k];
    if (written && n) f.write(reinterpret_cast<const char*>(r.bytes.get() + r.off[k]), (std::streamsize)n);
    written = written && f.good();
  }
  if (!written) fail(255, "Failed to write proto object.\n");  // solve.cc:674-677
  if (r.record_off.empty()) r.record_off = {0, r.record.size()};
  for (size_t k = 0; record && k < vrows.size(); ++k) {  // scene order (one scene without --versioned_scenes)
    if (!vrows[k].record) continue;
    const std::string& path = *vrows[k].record;
    std::ofstream f(path, std::ios::binary | std::ios::trunc);
    const uint64_t n = r.record_off[k + 1] - r.record_off[k];
    if (f.good()) f.write(reinterpret_cast<const char*>(r.record.data() + r.record_off[k]), (std::streamsize)n);
    if (!f.good()) fail(255, "ERROR: cannot write the record file '%s'\n", path.c_str());
  }
  return 0;
}

// One task line's argument vector: the line split at TABs (paths with spaces need no quoting); none for an empty line
std::vector<std::string> task_args(const std::string& line) {
  std::vector<std::string> args;
  for (size_t at = 0; !line.empty();) {
    const size_t tab = line.find('\t', at);
    args.push_back(line.substr(at, tab == std::string::npos ? std::string::npos : tab - at));
    if (tab == std::string::npos) break;
    at = tab + 1;
  }
  return args;
}

// The next line of `f` into `line`, without its newline (the last one is optional); false at the end of the file.
// The read blocks until the line is there, so a FIFO or /dev/stdin serves as the file.
bool read_line(std::FILE* f, std::string& line) {
  line.clear();
  int c;
  while ((c = std::getc(f)) != EOF && c != '\n') line.push_back((char)c);
  return c != EOF || !line.empty();
}

// One task of a stream: the run of `args` as a one-shot process would run it, except that the options the stream's
// command line sets once (--task_stream, --device, --gpus) are refused with exit code 2
int run_line(const std::vector<std::string>& args, Process& proc) {
  std::vector<char*> argv{const_cast<char*>("solve")};
  for (const std::string& a : args) argv.push_back(const_cast<char*>(a.c_str()));
  Options o;
  if (const std::optional<int> done = parse_command_line((int)argv.size(), argv.data(), o)) return *done;
  for (const char* name : {"task_stream", "device", "gpus"})
    if (o.named.count(name)) fail(2, "ERROR: --%s is set once, on the task stream's command line\n", name);
  return run_task(o, proc);
}

// --task_stream FILE: one process runs every line of FILE as a task, in order, each as the one-shot run of that
// argument vector would run it, so the start-up is paid once.  After a task its files are closed and `# task K:
// exit C` is on stdout, flushed, before the next line is read: a task can read what the one before wrote, and a
// client can wait for the line.  A failed task ends itself alone, unless a library call returned LFR_ECUDA or
// LFR_ENODEV: the context may then be unusable, and the stream ends with exit code 2.  The end of FILE ends it with 0.
int run_stream(const Options& so) {
  const std::unique_ptr<std::FILE, int (*)(std::FILE*)> f(std::fopen(so.task_stream->c_str(), "rb"), &std::fclose);
  if (!f) fail(2, "ERROR: cannot read the task stream file '%s'\n", so.task_stream->c_str());
  Process proc;
  proc.start(so);
  std::string line;
  for (unsigned long long k = 0; read_line(f.get(), line); ++k) {
    int code;
    bool lost = false;
    try {
      code = run_line(task_args(line), proc);
    } catch (const Exit& e) {
      code = e.code;
      lost = e.lost;
    }
    std::fflush(stderr);
    std::printf("# task %llu: exit %d\n", k, code);
    std::fflush(stdout);
    if (lost) return 2;
  }
  return 0;
}

int run(int argc, char** argv) {
  Options o;
  if (const std::optional<int> done = parse_command_line(argc, argv, o)) return *done;
  if (o.task_stream) {
    check_rules(o);
    return run_stream(o);
  }
  Process proc;  // the one-shot run: the process part and one task
  return run_task(o, proc);
}

}  // namespace

int main(int argc, char** argv) {
  try {
    return run(argc, argv);
  } catch (const Exit& e) {
    return e.code;
  }
}
