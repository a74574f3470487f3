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
// matches, decoded once, on the device route).  `--n_threads` is accepted and
// ignored (the solve runs on the GPU).  local-feature-refinement_b200/cli.py is the same program in
// Python; this one starts in milliseconds instead of importing numpy.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fcntl.h>
#include <fstream>
#include <map>
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
                               {"additional_scenes", true, false}, {"listed_pairs", true, false}};

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

struct Args {
  bool help = false, keep_initial_solution = false, carry_initial_solution = false, update_initial_solution = false,
       joint_queries = false;
  std::map<std::string, std::string> single;
  std::map<std::string, std::vector<std::string>> repeated;
};

// Boost.Program_options semantics of solve.cc:387-401: long options, `--name value` or `--name=value`,
// no positional arguments, Boost's error messages
Args parse(int argc, char** argv) {
  Args a;
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
          a.repeated[o.name].push_back(v);
        } else if (a.single.count(o.name)) {
          throw CliError{std::string("option '--") + o.name + "' cannot be specified more than once"};
        } else {
          a.single[o.name] = v;
        }
      } else {
        if (eq != std::string::npos) throw CliError{std::string("option '--") + o.name + "' does not take any arguments"};
        (std::strcmp(o.name, "help") == 0 ? a.help
         : std::strcmp(o.name, "keep_initial_solution") == 0  ? a.keep_initial_solution
         : std::strcmp(o.name, "carry_initial_solution") == 0 ? a.carry_initial_solution
         : std::strcmp(o.name, "joint_queries") == 0          ? a.joint_queries
                                                              : a.update_initial_solution) = true;
      }
    } else if (tok.size() > 1 && tok[0] == '-') {
      throw CliError{"unrecognised option '" + tok + "'"};
    } else {
      throw CliError{"too many positional options have been specified on the command line"};
    }
  }
  return a;
}

uint64_t as_uint(const Args& a, const char* name, uint64_t dflt) {  // lexical_cast<size_t>
  const auto it = a.single.find(name);
  if (it == a.single.end()) return dflt;
  const std::string& v = it->second;
  bool digits = !v.empty();
  for (char c : v) digits = digits && c >= '0' && c <= '9';
  if (!digits) throw CliError{"the argument ('" + v + "') for option '--" + name + "' is invalid"};
  return std::strtoull(v.c_str(), nullptr, 10);
}

bool file_exists(const std::string& path) {
  std::ifstream f(path, std::ios::binary);
  return f.good();
}

// A file mapped read-only (a Madrid-scale MatchingFile is several GB: no second copy of it in memory).
struct FileImage {
  const uint8_t* p = nullptr;
  size_t n = 0;
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

// One MatchingFile part after the pair walk: image names as byte ranges of its buffer, the matches as
// the offsets of their length prefixes.
struct Part {
  FileImage buf;
  uint64_t P = 0, M = 0;
  std::vector<uint64_t> pair_ptr, n1_off, n2_off, match_off;
  std::vector<uint32_t> n1_len, n2_len;
  std::vector<float> fact1, fact2;
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

// Read and decode the earlier MatchingFile `path` (or its .part.N pieces, as --matches_file): 0, 2 when no
// file can be read, 255 when the bytes do not parse.
int read_previous(const std::string& path, PreviousMatches& pm) {
  std::vector<std::string> files;
  if (file_exists(path)) {
    files.push_back(path);
  } else {
    for (int k = 0;; ++k) {
      const std::string f = path + ".part." + std::to_string(k);
      if (!file_exists(f)) break;
      files.push_back(f);
    }
  }
  if (files.empty()) return 2;
  std::map<std::string, uint32_t> id_of;
  for (const std::string& f : files) {
    Part pt;
    if (!pt.buf.open(f)) return 2;
    if (lfr_wire_scan_matches(pt.buf.data(), pt.buf.size(), &pt.P, &pt.M) != LFR_OK) return 255;
    pt.pair_ptr.resize(pt.P + 1);
    pt.n1_off.resize(pt.P); pt.n2_off.resize(pt.P); pt.n1_len.resize(pt.P); pt.n2_len.resize(pt.P);
    pt.fact1.resize(pt.P); pt.fact2.resize(pt.P);
    const uint64_t m0 = pm.feat1.size();
    pm.feat1.resize(m0 + pt.M); pm.feat2.resize(m0 + pt.M); pm.sim.resize(m0 + pt.M);
    pm.disp1.resize(18 * (m0 + pt.M)); pm.disp2.resize(18 * (m0 + pt.M));
    lfr_wire_matches w = pt.pair_level(pm.feat1.data() + m0, pm.feat2.data() + m0, pm.sim.data() + m0,
                                       pm.disp1.data() + 18 * m0, pm.disp2.data() + 18 * m0);
    if (lfr_wire_decode_matches(pt.buf.data(), pt.buf.size(), &w) != LFR_OK) return 255;
    auto intern = [&](uint64_t off, uint32_t len) {
      std::string s(reinterpret_cast<const char*>(pt.buf.data()) + off, len);
      const auto it = id_of.find(s);
      if (it != id_of.end()) return it->second;
      const uint32_t id = (uint32_t)pm.names.size();
      id_of.emplace(s, id);
      pm.name_blob.insert(pm.name_blob.end(), s.begin(), s.end());
      pm.name_off.push_back(pm.name_blob.size());
      pm.names.push_back(std::move(s));
      return id;
    };
    for (uint64_t p = 0; p < pt.P; ++p) {
      pm.pair_img1.push_back(intern(pt.n1_off[p], pt.n1_len[p]));
      pm.pair_img2.push_back(intern(pt.n2_off[p], pt.n2_len[p]));
      pm.pair_ptr.push_back(m0 + pt.pair_ptr[p + 1]);
    }
    pt.buf.release();
  }
  if (pm.name_blob.empty()) pm.name_blob.push_back(0);
  return 0;
}

// The --additional_scenes list: one `MATCHES_FILE<TAB>OUTPUT_FILE` per line (raw bytes; the last newline is
// optional), appended to `scenes`.  0, or 2 after one ERROR line for an unreadable file, a malformed line or
// two scenes (the first one included) with the same output path.
int read_scene_list(const std::string& path, std::vector<std::pair<std::string, std::string>>& scenes) {
  FileImage f;
  if (!f.open(path)) {
    std::fprintf(stderr, "ERROR: cannot read the scene list file '%s'\n", path.c_str());
    return 2;
  }
  const std::string text(reinterpret_cast<const char*>(f.data()), f.size());
  f.release();
  size_t line = 0;
  for (size_t at = 0; at < text.size();) {
    ++line;
    const size_t end = std::min(text.find('\n', at), text.size());
    const std::string l = text.substr(at, end - at);
    at = end + 1;
    const size_t tab = l.find('\t');
    const char* why = l.empty()                                  ? "it is empty"
                      : tab == std::string::npos                 ? "it has no TAB"
                      : l.find('\t', tab + 1) != std::string::npos ? "it has more than one TAB"
                      : tab == 0                                 ? "its matches file is empty"
                      : tab + 1 == l.size()                      ? "its output file is empty"
                      : l.find('\0') != std::string::npos        ? "it holds a NUL byte"
                                                                 : nullptr;
    if (why) {
      std::fprintf(stderr, "ERROR: --additional_scenes: line %zu is not MATCHES_FILE<TAB>OUTPUT_FILE: %s\n", line, why);
      return 2;
    }
    scenes.emplace_back(l.substr(0, tab), l.substr(tab + 1));
  }
  std::set<std::string> outputs;
  for (const auto& sc : scenes)
    if (!outputs.insert(sc.second).second) {
      std::fprintf(stderr, "ERROR: --additional_scenes: two scenes write '%s'\n", sc.second.c_str());
      return 2;
    }
  return 0;
}

// One --listed_pairs entry: a match list's path, its output file and its lines (NAME1, NAME2); `all` is list 0,
// every pair of --matches_file in file order.
struct PairList {
  std::string path, output;
  std::vector<std::pair<std::string, std::string>> lines;
  bool all = false;
};

// The --listed_pairs file: one `MATCH_LIST<TAB>OUTPUT_FILE` per line (the rules of read_scene_list), appended to
// `lists` after list 0, then every match list read and split as compute_match_graph.py:97 splits it (the
// newline stripped, single spaces; exactly two fields).  0, or 2 after one ERROR line for an unreadable file, a
// malformed line, two lists (the first one included) with the same output path, an unreadable match list or a
// malformed line of one, in that order.
int read_pair_lists(const std::string& path, std::vector<PairList>& lists) {
  FileImage f;
  if (!f.open(path)) {
    std::fprintf(stderr, "ERROR: cannot read the pair list file '%s'\n", path.c_str());
    return 2;
  }
  const std::string text(reinterpret_cast<const char*>(f.data()), f.size());
  f.release();
  size_t line = 0;
  for (size_t at = 0; at < text.size();) {
    ++line;
    const size_t end = std::min(text.find('\n', at), text.size());
    const std::string l = text.substr(at, end - at);
    at = end + 1;
    const size_t tab = l.find('\t');
    const char* why = l.empty()                                  ? "it is empty"
                      : tab == std::string::npos                 ? "it has no TAB"
                      : l.find('\t', tab + 1) != std::string::npos ? "it has more than one TAB"
                      : tab == 0                                 ? "its match list is empty"
                      : tab + 1 == l.size()                      ? "its output file is empty"
                      : l.find('\0') != std::string::npos        ? "it holds a NUL byte"
                                                                 : nullptr;
    if (why) {
      std::fprintf(stderr, "ERROR: --listed_pairs: line %zu is not MATCH_LIST<TAB>OUTPUT_FILE: %s\n", line, why);
      return 2;
    }
    PairList pl;
    pl.path = l.substr(0, tab);
    pl.output = l.substr(tab + 1);
    lists.push_back(std::move(pl));
  }
  std::set<std::string> outputs;
  for (const PairList& pl : lists)
    if (!outputs.insert(pl.output).second) {
      std::fprintf(stderr, "ERROR: --listed_pairs: two lists write '%s'\n", pl.output.c_str());
      return 2;
    }
  for (size_t i = 1; i < lists.size(); ++i) {
    PairList& pl = lists[i];
    FileImage g;
    if (!g.open(pl.path)) {
      std::fprintf(stderr, "ERROR: --listed_pairs: line %zu: cannot read the match list '%s'\n", i, pl.path.c_str());
      return 2;
    }
    const std::string t(reinterpret_cast<const char*>(g.data()), g.size());
    g.release();
    size_t j = 0;
    for (size_t at = 0; at < t.size();) {
      ++j;
      const size_t end = std::min(t.find('\n', at), t.size());
      const std::string l = t.substr(at, end - at);
      at = end + 1;
      const size_t fields = 1 + (size_t)std::count(l.begin(), l.end(), ' ');
      if (fields != 2) {
        std::fprintf(stderr, "ERROR: --listed_pairs: line %zu of the match list '%s' is not NAME1 NAME2: it has %zu fields\n",
                     j, pl.path.c_str(), fields);
        return 2;
      }
      const size_t sp = l.find(' ');
      pl.lines.emplace_back(l.substr(0, sp), l.substr(sp + 1));
    }
  }
  return 0;
}

using Clock = std::chrono::steady_clock;
long long ms_between(Clock::time_point a, Clock::time_point b) {
  return (long long)std::chrono::duration_cast<std::chrono::milliseconds>(b - a).count();
}

}  // namespace

int main(int argc, char** argv) {
  std::string matches_file, output_file, initial_solution, previous_matches_file, record_file, earlier_record_file,
      scene_list, list_file;
  std::vector<std::string> banned_list, fixed_list, query_list;
  uint64_t device = 0, gpus = 1;
  bool keep_start = false, carry_start = false, update_start = false, have_previous = false, have_record = false,
       have_earlier = false, have_query = false, joint = false, have_scenes = false,
       have_lists = false;
  try {
    Args a = parse(argc, argv);
    if (a.help) {
      std::fputs("Patch Match graph problem solver\n\n", stdout);
      std::fputs(kUsage, stdout);
      return 0;
    }
    for (const char* req : {"matches_file", "output_file"})  // po::notify: required options, in declaration order
      if (!a.single.count(req)) throw CliError{std::string("the option '--") + req + "' is required but missing"};
    matches_file = a.single.at("matches_file");
    output_file = a.single.at("output_file");
    (void)as_uint(a, "n_threads", 8);
    device = as_uint(a, "device", 0);
    gpus = as_uint(a, "gpus", 1);
    banned_list = a.repeated["banned_images"];
    fixed_list = a.repeated["fixed_images"];
    have_query = a.repeated.count("query_images") != 0;
    query_list = a.repeated["query_images"];
    joint = a.joint_queries;
    if (a.single.count("initial_solution")) initial_solution = a.single.at("initial_solution");
    keep_start = a.keep_initial_solution;
    carry_start = a.carry_initial_solution;
    update_start = a.update_initial_solution;
    have_previous = a.single.count("previous_matches_file") != 0;
    if (have_previous) previous_matches_file = a.single.at("previous_matches_file");
    have_record = a.single.count("record_file") != 0;
    if (have_record) record_file = a.single.at("record_file");
    have_earlier = a.single.count("earlier_record_file") != 0;
    if (have_earlier) earlier_record_file = a.single.at("earlier_record_file");
    have_scenes = a.single.count("additional_scenes") != 0;
    if (have_scenes) scene_list = a.single.at("additional_scenes");
    have_lists = a.single.count("listed_pairs") != 0;
    if (have_lists) list_file = a.single.at("listed_pairs");
  } catch (const CliError& e) {  // solve.cc:397-401
    std::fprintf(stderr, "ERROR: %s\n\n", e.msg.c_str());
    std::fputs(kUsage, stderr);
    return 1;
  }

  // the start solution is read and checked before any other work, so that its errors come before any output
  FileImage start_file;
  const bool have_start = !initial_solution.empty();
  if (keep_start && !have_start) {
    std::fputs("ERROR: --keep_initial_solution needs --initial_solution FILE\n", stderr);
    return 2;
  }
  if (carry_start && !have_start) {
    std::fputs("ERROR: --carry_initial_solution needs --initial_solution FILE\n", stderr);
    return 2;
  }
  if (update_start && !have_start) {
    std::fputs("ERROR: --update_initial_solution needs --initial_solution FILE\n", stderr);
    return 2;
  }
  if (update_start && keep_start) {
    std::fputs("ERROR: --update_initial_solution and --keep_initial_solution exclude each other\n", stderr);
    return 2;
  }
  if (have_previous && !update_start) {
    std::fputs("ERROR: --previous_matches_file needs --update_initial_solution\n", stderr);
    return 2;
  }
  if (have_earlier && !update_start) {
    std::fputs("ERROR: --earlier_record_file needs --update_initial_solution\n", stderr);
    return 2;
  }
  if (have_earlier && have_previous) {
    std::fputs("ERROR: --earlier_record_file and --previous_matches_file exclude each other\n", stderr);
    return 2;
  }
  if (have_query) {  // each query is refined against the scene as it stands; the incremental modes update one scene
    for (const auto& o : {std::make_pair(update_start, "--update_initial_solution"),
                          std::make_pair(have_previous, "--previous_matches_file"), std::make_pair(have_record, "--record_file"),
                          std::make_pair(have_earlier, "--earlier_record_file"),
                          std::make_pair(carry_start, "--carry_initial_solution")})
      if (o.first) {
        std::fprintf(stderr, "ERROR: --query_images and %s exclude each other\n", o.second);
        return 2;
      }
  }
  if (joint && !have_query) {
    std::fputs("ERROR: --joint_queries needs --query_images\n", stderr);
    return 2;
  }
  // --listed_pairs: list 0 is every pair of --matches_file, written to --output_file; the listed match lists
  // follow.  Each list's output is what its own run writes: the same command on a MatchingFile that holds the
  // file's pair for every line of the list, in line order.
  std::vector<PairList> lists(1);
  lists[0].output = output_file;
  lists[0].all = true;
  if (have_lists) {  // as --additional_scenes, whose batches it excludes too
    for (const auto& o : {std::make_pair(!fixed_list.empty(), "--fixed_images"), std::make_pair(have_start, "--initial_solution"),
                          std::make_pair(keep_start, "--keep_initial_solution"),
                          std::make_pair(carry_start, "--carry_initial_solution"),
                          std::make_pair(update_start, "--update_initial_solution"),
                          std::make_pair(have_previous, "--previous_matches_file"), std::make_pair(have_record, "--record_file"),
                          std::make_pair(have_earlier, "--earlier_record_file"), std::make_pair(have_query, "--query_images"),
                          std::make_pair(joint, "--joint_queries"), std::make_pair(have_scenes, "--additional_scenes")})
      if (o.first) {
        std::fprintf(stderr, "ERROR: --listed_pairs and %s exclude each other\n", o.second);
        return 2;
      }
    const int rc = read_pair_lists(list_file, lists);
    if (rc) return rc;
  }
  // --additional_scenes: the scene of --matches_file / --output_file is scene 0, the listed ones follow; each
  // scene's output is what its own run writes (the same command with that scene's two files alone)
  std::vector<std::pair<std::string, std::string>> scenes{{matches_file, output_file}};
  if (have_scenes) {  // the start solution, the fixed images and the incremental modes belong to one scene
    for (const auto& o : {std::make_pair(!fixed_list.empty(), "--fixed_images"), std::make_pair(have_start, "--initial_solution"),
                          std::make_pair(keep_start, "--keep_initial_solution"),
                          std::make_pair(carry_start, "--carry_initial_solution"),
                          std::make_pair(update_start, "--update_initial_solution"),
                          std::make_pair(have_previous, "--previous_matches_file"), std::make_pair(have_record, "--record_file"),
                          std::make_pair(have_earlier, "--earlier_record_file"), std::make_pair(have_query, "--query_images"),
                          std::make_pair(joint, "--joint_queries")})
      if (o.first) {
        std::fprintf(stderr, "ERROR: --additional_scenes and %s exclude each other\n", o.second);
        return 2;
      }
    const int rc = read_scene_list(scene_list, scenes);
    if (rc) return rc;
  }
  uint32_t S = (uint32_t)scenes.size();  // the batch's members: scenes, or with --listed_pairs the lists
  if (have_start) {
    if (!start_file.open(initial_solution)) {
      std::fprintf(stderr, "ERROR: cannot read the initial solution file '%s'\n", initial_solution.c_str());
      return 2;
    }
    uint64_t ni = 0, nd = 0;
    if (lfr_wire_decode_solution(start_file.data(), start_file.size(), &ni, &nd, nullptr, nullptr, nullptr, nullptr, nullptr,
                                 nullptr, nullptr) != LFR_OK) {
      std::fputs("Failed to parse proto object.\n", stderr);  // as for the matches, solve.cc:433-436
      return 255;
    }
  }
  PreviousMatches previous;
  if (have_previous) {
    const int rc = read_previous(previous_matches_file, previous);
    if (rc == 2) {
      std::fprintf(stderr, "ERROR: cannot read the previous matches file '%s'\n", previous_matches_file.c_str());
      return 2;
    }
    if (rc != 0) {
      std::fputs("Failed to parse proto object.\n", stderr);
      return 255;
    }
  }
  std::vector<uint8_t> earlier_record;
  if (have_earlier) {
    FileImage f;
    if (!f.open(earlier_record_file)) {
      std::fprintf(stderr, "ERROR: cannot read the earlier record file '%s'\n", earlier_record_file.c_str());
      return 2;
    }
    earlier_record.assign(f.data(), f.data() + f.size());
    f.release();
    if (!lfr::record::check(earlier_record.data(), earlier_record.size(), nullptr)) {
      std::fprintf(stderr, "ERROR: '%s' is not a problem record\n", earlier_record_file.c_str());
      return 2;
    }
  }

  // A one-shot process pays for CUDA's start-up (driver initialisation over every visible GPU, context
  // creation: 0.4-0.8 s on an 8-GPU box) more than for all of its work on a Fountain-scale scene.  Two
  // measures: only the device that will be used is made visible (unless the caller already chose),
  // and the start-up runs on a helper thread while the input is read, decoded and turned into a graph.
  if (gpus <= 1 && !std::getenv("CUDA_VISIBLE_DEVICES")) {
    setenv("CUDA_VISIBLE_DEVICES", std::to_string(device).c_str(), 1);
    device = 0;
  }
  std::thread cuda_start([] { lfr_host_free(lfr_host_alloc(64)); });
  struct Joiner {
    std::thread& t;
    ~Joiner() { if (t.joinable()) t.join(); }
  } join_on_exit{cuda_start};

  // ---- solve.cc:412-481: the file, or its .part.N pieces, of every scene -----------------------
  std::vector<std::string> files;
  std::vector<uint32_t> part_scene;
  for (uint32_t sc = 0; sc < S; ++sc) {
    const std::string& mf = scenes[sc].first;
    if (file_exists(mf)) {
      files.push_back(mf);
      part_scene.push_back(sc);
    } else {
      for (int k = 0;; ++k) {
        const std::string f = mf + ".part." + std::to_string(k);
        if (!file_exists(f)) break;
        files.push_back(f);
        part_scene.push_back(sc);
      }
    }
  }
  std::vector<Part> parts(files.size());
  for (size_t i = 0; i < files.size(); ++i) {
    Part& pt = parts[i];
    bool ok = pt.buf.open(files[i]);
    if (ok) ok = lfr_wire_scan_matches(pt.buf.data(), pt.buf.size(), &pt.P, &pt.M) == LFR_OK;
    if (ok) {
      pt.pair_ptr.resize(pt.P + 1);
      pt.n1_off.resize(pt.P); pt.n2_off.resize(pt.P); pt.n1_len.resize(pt.P); pt.n2_len.resize(pt.P);
      pt.fact1.resize(pt.P); pt.fact2.resize(pt.P);
      pt.match_off.resize(pt.M);
      lfr_wire_matches w = pt.pair_level(nullptr, nullptr, nullptr, nullptr, nullptr);
      ok = lfr_wire_walk_matches(pt.buf.data(), pt.buf.size(), &w, pt.match_off.data()) == LFR_OK;
    }
    if (!ok) {
      std::fputs("Failed to parse proto object.\n", stderr);  // solve.cc:433-436
      return 255;
    }
  }

  // image names -> ids in order of first appearance over all parts; the pairs of all parts in order, and the
  // scene of every pair
  std::vector<std::string> names;
  std::map<std::string, uint32_t> id_of;
  auto intern = [&](const Part& pt, uint64_t off, uint32_t len) {
    std::string s(reinterpret_cast<const char*>(pt.buf.data()) + off, len);
    const auto it = id_of.find(s);
    if (it != id_of.end()) return it->second;
    const uint32_t id = (uint32_t)names.size();
    id_of.emplace(s, id);
    names.push_back(std::move(s));
    return id;
  };
  uint64_t P = 0, M = 0;
  for (const Part& pt : parts) { P += pt.P; M += pt.M; }
  std::vector<uint32_t> pair_img1(P), pair_img2(P);
  std::vector<float> pair_fact1(P), pair_fact2(P);
  std::vector<uint64_t> pair_ptr(P + 1, 0);
  std::vector<uint32_t> pair_scene(P);
  {
    uint64_t p0 = 0, m0 = 0;
    for (size_t i = 0; i < parts.size(); ++i) {
      Part& pt = parts[i];
      for (uint64_t p = 0; p < pt.P; ++p) {
        pair_scene[p0 + p] = part_scene[i];
        pair_img1[p0 + p] = intern(pt, pt.n1_off[p], pt.n1_len[p]);
        pair_img2[p0 + p] = intern(pt, pt.n2_off[p], pt.n2_len[p]);
        pair_fact1[p0 + p] = pt.fact1[p];
        pair_fact2[p0 + p] = pt.fact2[p];
        pair_ptr[p0 + p + 1] = m0 + pt.pair_ptr[p + 1];
      }
      p0 += pt.P;
      m0 += pt.M;
    }
  }

  // --listed_pairs: the batch's pairs are the lists' lines, list after list, each the first pair of the file
  // with exactly those two names (one map over the pairs, names as bytes); every pair of the file for list 0.
  // pair_src is the file's pair behind each of them, whose matches are copied to it after the decode.
  const uint64_t M_file = M;  // the matches the decode reads: the file's
  std::vector<uint64_t> pair_src, file_pair_ptr;
  if (have_lists) {
    std::unordered_map<uint64_t, uint64_t> first;  // image1 << 32 | image2 -> the first pair
    for (uint64_t p = 0; p < P; ++p) first.emplace((uint64_t)pair_img1[p] << 32 | pair_img2[p], p);
    std::vector<uint32_t> list_of;
    for (size_t l = 0; l < lists.size(); ++l) {
      if (lists[l].all) {
        for (uint64_t p = 0; p < P; ++p) {
          pair_src.push_back(p);
          list_of.push_back((uint32_t)l);
        }
        continue;
      }
      for (size_t j = 0; j < lists[l].lines.size(); ++j) {
        const std::string& n1 = lists[l].lines[j].first;
        const std::string& n2 = lists[l].lines[j].second;
        const auto i1 = id_of.find(n1), i2 = id_of.find(n2);
        auto hit = first.end();
        bool reverse = false;
        if (i1 != id_of.end() && i2 != id_of.end()) {
          hit = first.find((uint64_t)i1->second << 32 | i2->second);
          reverse = first.count((uint64_t)i2->second << 32 | i1->second) != 0;
        }
        if (hit == first.end()) {
          std::fprintf(stderr, "ERROR: --listed_pairs: line %zu of the match list '%s': the matches file holds no pair '%s' '%s'",
                       j + 1, lists[l].path.c_str(), n1.c_str(), n2.c_str());
          if (reverse) std::fprintf(stderr, "; it holds only '%s' '%s'", n2.c_str(), n1.c_str());
          std::fputs("\n", stderr);
          return 2;
        }
        pair_src.push_back(hit->second);
        list_of.push_back((uint32_t)l);
      }
    }
    const uint64_t Q = pair_src.size();
    std::vector<uint32_t> img1(Q), img2(Q);
    std::vector<float> f1(Q), f2(Q);
    std::vector<uint64_t> ptr(Q + 1, 0);
    for (uint64_t k = 0; k < Q; ++k) {
      const uint64_t p = pair_src[k];
      img1[k] = pair_img1[p]; img2[k] = pair_img2[p]; f1[k] = pair_fact1[p]; f2[k] = pair_fact2[p];
      ptr[k + 1] = ptr[k] + (pair_ptr[p + 1] - pair_ptr[p]);
    }
    pair_img1.swap(img1); pair_img2.swap(img2); pair_fact1.swap(f1); pair_fact2.swap(f2);
    file_pair_ptr.swap(pair_ptr);
    pair_ptr.swap(ptr);
    pair_scene.swap(list_of);
    P = Q;
    M = pair_ptr[Q];
    scenes.clear();  // from here on the batch's members are the lists
    for (const PairList& pl : lists) scenes.emplace_back(pl.path, pl.output);
    S = (uint32_t)scenes.size();
  }
  const bool batched = have_scenes || have_lists;

  // banned images (solve.cc:444-446)
  const std::set<std::string> banned(banned_list.begin(), banned_list.end());
  std::vector<uint8_t> skip(P, 0);
  for (uint64_t p = 0; p < P; ++p)
    skip[p] = (banned.count(names[pair_img1[p]]) || banned.count(names[pair_img2[p]])) ? 1 : 0;

  // --query_images: a kept pair that names a query image belongs to that query's group's sub-scene, and its
  // images get that sub-scene's ids, in order of first appearance; a pair that names none is not solved.  A
  // group is one query, or with --joint_queries a connected component of the queries under the kept pairs
  // that name two of them (with or without matches).  The graph stage then gives every sub-scene what a run
  // on its pairs alone gives (lfr_host_input::image_group).  --additional_scenes: the same rule with every
  // kept pair in its scene's sub-scene, labelled by the scene index, so that scenes that share image names
  // share no node and each meta-component is cut at its own scene's image count.  --listed_pairs: the same with
  // the list index as the label, so a pair listed by two lists is a node set of each.
  // orig_of: the original image id (and name) of every stage image id; the identity without sub-scenes.
  std::vector<uint8_t> is_query(names.size(), 0);
  std::vector<uint32_t> orig_of, image_group;
  if (have_query || batched) {
    const std::set<std::string> queries(query_list.begin(), query_list.end());
    for (size_t i = 0; i < names.size(); ++i) is_query[i] = queries.count(names[i]) ? 1 : 0;
    // the group of every query image: a union-find whose root is the group's lowest image id, its label.  It
    // runs over all pairs before any id is handed out, since a later pair can merge two groups that hold ids.
    std::vector<uint32_t> group_of(names.size());
    for (uint32_t i = 0; i < (uint32_t)names.size(); ++i) group_of[i] = i;
    auto find = [&](uint32_t x) {
      while (group_of[x] != x) x = group_of[x] = group_of[group_of[x]];
      return x;
    };
    for (uint64_t p = 0; have_query && p < P; ++p) {
      const uint32_t a = pair_img1[p], b = pair_img2[p];
      if (skip[p] || !is_query[a] || !is_query[b]) continue;
      if (!joint) {
        std::fprintf(stderr, "ERROR: the pair '%s' - '%s' names two query images\n", names[a].c_str(), names[b].c_str());
        return 2;
      }
      const uint32_t ra = find(a), rb = find(b);
      group_of[std::max(ra, rb)] = std::min(ra, rb);
    }
    std::map<std::pair<uint32_t, uint32_t>, uint32_t> sub_id;  // (group, image) -> stage image id
    auto sub = [&](uint32_t g, uint32_t img) {
      const auto it = sub_id.emplace(std::make_pair(g, img), (uint32_t)orig_of.size());
      if (it.second) {
        orig_of.push_back(img);
        image_group.push_back(g);
      }
      return it.first->second;
    };
    for (uint64_t p = 0; p < P; ++p) {
      const uint32_t a = pair_img1[p], b = pair_img2[p];
      if (skip[p] || (have_query && !(is_query[a] || is_query[b]))) {
        skip[p] = 1;
        pair_img1[p] = pair_img2[p] = 0;  // never read: skipped pairs name no image of the stage
        continue;
      }
      const uint32_t g = have_query ? find(is_query[a] ? a : b) : pair_scene[p];
      pair_img1[p] = sub(g, a);
      pair_img2[p] = sub(g, b);
    }
    if (orig_of.size() > 65535) {
      if (have_query)
        std::fprintf(stderr, "ERROR: --query_images: the sub-scenes hold %zu images, more than 65535; split the query list "
                             "over several runs\n", orig_of.size());
      else if (have_lists)
        std::fprintf(stderr, "ERROR: --listed_pairs: the lists hold %zu images, more than 65535; split the pair list "
                             "over several runs\n", orig_of.size());
      else
        std::fprintf(stderr, "ERROR: --additional_scenes: the scenes hold %zu images, more than 65535; split the scene list "
                             "over several runs\n", orig_of.size());
      return 2;
    }
  } else {
    orig_of.resize(names.size());
    for (uint32_t i = 0; i < (uint32_t)names.size(); ++i) orig_of[i] = i;
  }
  const uint32_t n_ids = (uint32_t)orig_of.size();  // image ids of the graph stage's input

  // the first fact seen of every image among the pairs kept
  std::vector<float> image_fact(n_ids, 0.f);
  std::vector<uint8_t> have_fact(n_ids, 0);
  uint64_t e_cap = 0;
  for (uint64_t p = 0; p < P; ++p) {
    if (skip[p]) continue;
    e_cap += 2 * (pair_ptr[p + 1] - pair_ptr[p]);
    if (!have_fact[pair_img1[p]]) { have_fact[pair_img1[p]] = 1; image_fact[pair_img1[p]] = pair_fact1[p]; }
    if (!have_fact[pair_img2[p]]) { have_fact[pair_img2[p]] = 1; image_fact[pair_img2[p]] = pair_fact2[p]; }
  }

  // images held fixed (the same name semantics as banned images), and the names by image id as the
  // start-point join and the encoder on the GPU take them (ids of the graph stage: with --query_images a
  // database image's name repeats once per sub-scene, and the joins give every copy the same entries)
  const std::set<std::string> fixed_names(fixed_list.begin(), fixed_list.end());
  std::vector<uint8_t> fixed(n_ids, 0), image_written(n_ids, 0);
  bool any_fixed = false;
  for (uint32_t i = 0; i < n_ids; ++i) {
    image_written[i] = !have_query || is_query[orig_of[i]];
    if (fixed_names.count(names[orig_of[i]])) {
      fixed[i] = 1;
      any_fixed = true;
    }
  }
  std::vector<uint8_t> name_blob;
  std::vector<uint64_t> name_off(n_ids + 1, 0);
  for (uint32_t i = 0; i < n_ids; ++i) {
    const std::string& nm = names[orig_of[i]];
    name_blob.insert(name_blob.end(), nm.begin(), nm.end());
    name_off[i + 1] = name_blob.size();
  }

  lfr_host_input in;
  std::memset(&in, 0, sizeof in);
  in.n_pairs = P; in.n_matches = M; in.n_images = n_ids;
  in.pair_img1 = pair_img1.data(); in.pair_img2 = pair_img2.data(); in.pair_skip = skip.data();
  in.pair_ptr = pair_ptr.data();
  in.image_group = have_query || batched ? image_group.data() : nullptr;

  // ---- which graph stage: the library's size rule, or LFR_GRAPH_STAGE=host|device (a test and
  // measurement hook, not a product option).  A library without the stage on the GPU — the CPU checker —
  // takes the host route; forcing the device route there is an error, never a silent host run.
  const bool have_device_stage = lfr_graph_stage_on_device && lfr_wire_decode_on_device && lfr_plan_create_from_matches &&
                                 lfr_plan_create_from_wire && lfr_plan_encode_solution && lfr_plan_fix_images &&
                                 lfr_plan_start_from_solution && lfr_plan_keep_solution && lfr_plan_encode_solution_carried &&
                                 lfr_plan_update_solution && lfr_plan_update_solution_since && lfr_plan_problem_record &&
                                 lfr_plan_update_solution_since_record && lfr_plan_encode_solution_images &&
                                 lfr_plan_encode_solution_groups && lfr_plan_create_from_wire_listed;
  bool on_device = have_device_stage && lfr_graph_stage_on_device(&in, (int32_t)gpus) == 1;
  const char* force = std::getenv("LFR_GRAPH_STAGE");
  if (force && *force) {
    if (std::strcmp(force, "host") == 0) {
      on_device = false;
    } else if (std::strcmp(force, "device") == 0) {
      if (!have_device_stage) {
        std::fprintf(stderr, "ERROR: LFR_GRAPH_STAGE=device: the solve library has no graph stage on the GPU\n");
        return 2;
      }
      if (gpus > 1) {
        std::fprintf(stderr, "ERROR: LFR_GRAPH_STAGE=device: the graph stage on the GPU drives one device (--gpus 1)\n");
        return 2;
      }
      on_device = true;
    } else {
      std::fprintf(stderr, "ERROR: LFR_GRAPH_STAGE must be 'host' or 'device'\n");
      return 2;
    }
  }

  // host route, and the device route below the library's size for the decoder on the GPU: the matches of
  // every part decoded into one set of arrays, part after part (the pair level comes out as the walk gave it).
  // With --listed_pairs the file is decoded once and every listed pair's matches are then copied into place;
  // the decoder's threshold sees the file's match count.
  const bool decode_on_device = on_device && lfr_wire_decode_on_device(M_file) == 1;
  std::vector<uint32_t> feat1, feat2;
  std::vector<float> sim, disp1, disp2;
  if (!decode_on_device) {
    feat1.resize(M_file); feat2.resize(M_file); sim.resize(M_file); disp1.resize(18 * M_file); disp2.resize(18 * M_file);
    uint64_t m0 = 0;
    for (Part& pt : parts) {
      lfr_wire_matches w = pt.pair_level(feat1.data() + m0, feat2.data() + m0, sim.data() + m0, disp1.data() + 18 * m0,
                                         disp2.data() + 18 * m0);
      if (lfr_wire_decode_matches(pt.buf.data(), pt.buf.size(), &w) != LFR_OK) {
        std::fputs("Failed to parse proto object.\n", stderr);  // solve.cc:433-436
        return 255;
      }
      m0 += pt.M;
      pt.buf.release();  // the file image (several GB at Madrid scale) is not needed past the decode
    }
    if (have_lists) {
      std::vector<uint32_t> e1(M), e2(M);
      std::vector<float> es(M), ed1(18 * M), ed2(18 * M);
      for (uint64_t k = 0; k < P; ++k) {
        const uint64_t a = file_pair_ptr[pair_src[k]], c = pair_ptr[k + 1] - pair_ptr[k], b = pair_ptr[k];
        std::copy_n(feat1.begin() + a, c, e1.begin() + b);
        std::copy_n(feat2.begin() + a, c, e2.begin() + b);
        std::copy_n(sim.begin() + a, c, es.begin() + b);
        std::copy_n(disp1.begin() + 18 * a, 18 * c, ed1.begin() + 18 * b);
        std::copy_n(disp2.begin() + 18 * a, 18 * c, ed2.begin() + 18 * b);
      }
      feat1.swap(e1); feat2.swap(e2); sim.swap(es); disp1.swap(ed1); disp2.swap(ed2);
    }
    in.feat1 = feat1.data(); in.feat2 = feat2.data(); in.sim = sim.data(); in.disp1 = disp1.data(); in.disp2 = disp2.data();
  }

  cuda_start.join();  // page-locked memory needs the context
  const Clock::time_point t_start = Clock::now();  // "Total time" (solve.cc:487-641): the graph work and the solve
  lfr_edge* edges = nullptr;
  bool edges_pinned = false;
  lfr_plan* plan = nullptr;
  lfr_host_sizes sz;
  std::vector<uint32_t> row_ptr, track, comp, comp_ptr, comp_nodes, comp_order, node_image, node_feat;
  std::vector<uint8_t> is_root;
  if (on_device) {
    // ---- the matches decoded and the graph stage run on the GPU (include/lfr_graph.h): the problem stays
    // in HBM for the solve and the SolutionFile is encoded there
    lfr_options opt;
    lfr_options_default(&opt);
    opt.device = (int32_t)device;
    // LFR_DEVICE_CUT=1: the recursive cut on the device too (LFR_DBG_DEVICE_CUT; a test and measurement hook)
    if (const char* e = std::getenv("LFR_DEVICE_CUT")) {
      if (std::strcmp(e, "1") == 0) opt.debug_flags |= LFR_DBG_DEVICE_CUT;
    }
    std::vector<lfr_wire_part> wparts;
    for (const Part& pt : parts) wparts.push_back(lfr_wire_part{pt.buf.data(), pt.buf.size(), pt.match_off.data(), pt.M});
    const int rc = decode_on_device && have_lists
                       ? lfr_plan_create_from_wire_listed(&in, wparts.data(), (uint32_t)wparts.size(), file_pair_ptr.data(),
                                                          file_pair_ptr.size() - 1, pair_src.data(), &opt, nullptr, &plan, &sz)
                   : decode_on_device
                       ? lfr_plan_create_from_wire(&in, wparts.data(), (uint32_t)wparts.size(), &opt, nullptr, &plan, &sz)
                       : lfr_plan_create_from_matches(&in, &opt, nullptr, &plan, &sz);
    for (Part& pt : parts) pt.buf.release();
    if (rc == LFR_EINVAL && std::strcmp(lfr_last_error(), "malformed Match message") == 0) {
      std::fputs("Failed to parse proto object.\n", stderr);  // solve.cc:433-436, as the host decode
      return 255;
    }
    if (rc == LFR_EINVAL || rc == LFR_EUNSUPPORTED) {  // the input, as the host stage would reject it
      std::fprintf(stderr, "ERROR: the host graph stage rejected the input\n");
      return 2;
    }
    if (rc != LFR_OK) {  // no device: the host route's message, from the same device check
      std::fprintf(stderr, "ERROR: the solve failed (%d): %s\n", rc, lfr_last_error());
      return 2;
    }
    // problem initialisation (solve.cc:608-612) on the plan: the constant mask and the start point
    int rc2 = any_fixed ? lfr_plan_fix_images(plan, fixed.data(), n_ids) : LFR_OK;
    if (rc2 == LFR_OK && have_earlier) {
      rc2 = lfr_plan_update_solution_since_record(plan, nullptr, start_file.data(), start_file.size(), n_ids,
                                                  name_blob.data(), name_off.data(), earlier_record.data(),
                                                  earlier_record.size(), nullptr, nullptr, nullptr);
    } else if (rc2 == LFR_OK && have_previous) {
      // the earlier run's graph stage on the device, for the compare only
      const lfr_host_input pin = previous.input();
      lfr_plan* prev_plan = nullptr;
      rc2 = lfr_plan_create_from_matches(&pin, &opt, nullptr, &prev_plan, nullptr);
      if (rc2 == LFR_OK)
        rc2 = lfr_plan_update_solution_since(plan, nullptr, start_file.data(), start_file.size(), n_ids,
                                             name_blob.data(), name_off.data(), prev_plan, (uint32_t)previous.names.size(),
                                             previous.name_blob.data(), previous.name_off.data(), nullptr, nullptr, nullptr);
      lfr_plan_destroy(prev_plan);
    } else if (rc2 == LFR_OK && have_start && update_start)
      rc2 = lfr_plan_update_solution(plan, nullptr, start_file.data(), start_file.size(), n_ids,
                                     name_blob.data(), name_off.data(), nullptr, nullptr);
    else if (rc2 == LFR_OK && have_start)
      rc2 = (keep_start ? lfr_plan_keep_solution : lfr_plan_start_from_solution)(
          plan, nullptr, start_file.data(), start_file.size(), n_ids, name_blob.data(), name_off.data(), nullptr);
    if (rc2 != LFR_OK) {
      std::fprintf(stderr, "ERROR: the solve failed (%d): %s\n", rc2, lfr_last_error());
      return 2;
    }
  } else {
    // ---- host graph stage (solve.cc:438-606); the edge records go straight into page-locked memory
    if (e_cap) {
      edges = static_cast<lfr_edge*>(lfr_host_alloc(e_cap * sizeof(lfr_edge)));
      edges_pinned = edges != nullptr;
      if (!edges) edges = static_cast<lfr_edge*>(std::malloc(e_cap * sizeof(lfr_edge)));
    }
    in.edges_out = edges; in.edges_out_capacity = e_cap;
    lfr_host_stage* hs = nullptr;
    if (lfr_host_stage_create(&in, &hs, &sz) != LFR_OK) {
      std::fprintf(stderr, "ERROR: the host graph stage rejected the input\n");
      return 2;
    }
    const uint32_t n = sz.n_nodes, c = sz.n_components;
    row_ptr.assign((size_t)n + 1, 0); track.resize(n); comp.resize(n); comp_ptr.assign((size_t)c + 1, 0);
    comp_nodes.resize(n); comp_order.resize(c); node_image.resize(n); node_feat.resize(n); is_root.resize(n);
    if (lfr_host_stage_export(hs, row_ptr.data(), edges, track.data(), comp.data(), is_root.data(), comp_ptr.data(),
                              comp_nodes.data(), comp_order.data(), node_image.data(), node_feat.data()) != LFR_OK) {
      std::fprintf(stderr, "ERROR: lfr_host_stage_export failed\n");
      return 2;
    }
    lfr_host_stage_destroy(hs);
  }
  const uint32_t N = sz.n_nodes, C = sz.n_components;
  const uint64_t E = sz.n_edges;
  // the host route's problem with the reference's is_root (the update since an earlier run and the record read it)
  auto host_problem = [&] {
    lfr_problem p;
    p.n_nodes = N; p.n_components = C; p.n_edges = E;
    p.row_ptr = row_ptr.data(); p.edges = edges; p.track = track.data(); p.comp = comp.data();
    p.is_root = is_root.data(); p.comp_ptr = comp_ptr.data(); p.comp_nodes = comp_nodes.data();
    return p;
  };
  std::printf("# graph nodes: %u\n", N);                                  // solve.cc:484
  std::printf("# graph edges: %llu\n", (unsigned long long)E);            // solve.cc:485
  if (N) {
    std::printf("# tracks: %u\n", sz.n_tracks);                           // solve.cc:534
    std::printf("max track size: %u\n", sz.max_track_size);               // solve.cc:549
    std::printf("Graph-cut time: %lldms\n", (long long)sz.graph_cut_ms);  // solve.cc:589
    std::printf("# components: %u\n", C);                                 // solve.cc:591
    std::printf("max component size: %u\n", sz.max_component_size);       // solve.cc:606
  }
  std::fflush(stdout);

  // ---- the solve (solve.cc:608-635): positions start at zero, or from --initial_solution -----
  double* positions = nullptr;  // host route: the solve's result; the device route keeps it in HBM
  bool positions_pinned = false;
  // host route with --fixed_images, --keep_initial_solution or --update_initial_solution: reference roots OR
  // nodes of fixed images OR nodes with an entry in the start solution (kept) or held by the update
  std::vector<uint8_t> is_const;
  const bool any_const = any_fixed || keep_start || update_start;
  if (N && !plan) {
    positions = static_cast<double*>(lfr_host_alloc(2ull * N * sizeof(double)));
    positions_pinned = positions != nullptr;
    if (!positions) positions = static_cast<double*>(std::malloc(2ull * N * sizeof(double)));
    std::memset(positions, 0, 2ull * N * sizeof(double));
    std::vector<uint8_t> has_entry(keep_start || update_start ? N : 0, 0);
    if (have_earlier) {
      const lfr_problem cur = host_problem();
      if (lfr_wire_update_solution_since_record(start_file.data(), start_file.size(), n_ids,
                                                name_blob.data(), name_off.data(), &cur, node_image.data(), node_feat.data(),
                                                earlier_record.data(), earlier_record.size(), positions, has_entry.data(),
                                                nullptr, nullptr, nullptr) != LFR_OK) {
        std::fprintf(stderr, "ERROR: lfr_wire_update_solution_since_record failed\n");
        return 2;
      }
    } else if (have_previous) {
      const lfr_problem cur = host_problem();
      const lfr_host_input pin = previous.input();
      if (lfr_wire_update_solution_since(start_file.data(), start_file.size(), n_ids, name_blob.data(),
                                         name_off.data(), &cur, node_image.data(), node_feat.data(), &pin,
                                         previous.name_blob.data(), previous.name_off.data(), positions, has_entry.data(),
                                         nullptr, nullptr, nullptr) != LFR_OK) {
        std::fprintf(stderr, "ERROR: lfr_wire_update_solution_since failed\n");
        return 2;
      }
    } else if (have_start && update_start) {
      if (lfr_wire_update_solution(start_file.data(), start_file.size(), n_ids, name_blob.data(),
                                   name_off.data(), N, node_image.data(), node_feat.data(), comp.data(), C, positions,
                                   has_entry.data(), nullptr, nullptr) != LFR_OK) {
        std::fprintf(stderr, "ERROR: lfr_wire_update_solution failed\n");
        return 2;
      }
    } else if (have_start && (keep_start ? lfr_wire_join_solution_entries(start_file.data(), start_file.size(), n_ids,
                                                                  name_blob.data(), name_off.data(), N, node_image.data(),
                                                                  node_feat.data(), positions, nullptr, has_entry.data())
                                  : lfr_wire_join_solution(start_file.data(), start_file.size(), n_ids,
                                                           name_blob.data(), name_off.data(), N, node_image.data(),
                                                           node_feat.data(), positions, nullptr)) != LFR_OK) {
      std::fprintf(stderr, "ERROR: lfr_wire_join_solution failed\n");
      return 2;
    }
    if (any_const) {
      is_const.resize(N);
      for (uint32_t v = 0; v < N; ++v)
        is_const[v] = (is_root[v] || fixed[node_image[v]] || ((keep_start || update_start) && has_entry[v])) ? 1 : 0;
    }
  }
  if (!carry_start) start_file.release();  // carried into the output otherwise
  const Clock::time_point t_solve = Clock::now();
  if (N && plan) {
    int rc = lfr_plan_solve(plan, nullptr);
    if (rc == LFR_OK) rc = lfr_plan_download(plan, nullptr, nullptr, nullptr);  // waits for the solve, checks its error flag
    if (rc != LFR_OK) {
      std::fprintf(stderr, "ERROR: the solve failed (%d): %s\n", rc, lfr_last_error());
      return 2;
    }
  } else if (N) {
    lfr_problem prob;
    prob.n_nodes = N; prob.n_components = C; prob.n_edges = E;
    prob.row_ptr = row_ptr.data(); prob.edges = edges; prob.track = track.data(); prob.comp = comp.data();
    prob.is_root = any_const ? is_const.data() : is_root.data(); prob.comp_ptr = comp_ptr.data(); prob.comp_nodes = comp_nodes.data();
    lfr_options opt;
    lfr_options_default(&opt);
    opt.device = (int32_t)device;
    lfr_stats st;
    std::memset(&st, 0, sizeof st);
    int rc;
    if (gpus > 1) {
      std::vector<int32_t> devs((size_t)gpus);
      for (size_t i = 0; i < devs.size(); ++i) devs[i] = (int32_t)i;
      rc = lfr_solve_multi(&prob, &opt, devs.data(), (int32_t)devs.size(), positions, &st, nullptr);
    } else {
      rc = lfr_solve(&prob, &opt, positions, &st);
    }
    if (rc != LFR_OK) {  // no CPU fallback: without a CUDA device this is where the program stops
      std::fprintf(stderr, "ERROR: the solve failed (%d): %s\n", rc, lfr_last_error());
      return 2;
    }
  }
  const Clock::time_point t_end = Clock::now();
  std::printf("Solver time: %lldms\n", ms_between(t_solve, t_end));  // solve.cc:638
  std::printf("Total time: %lldms\n", ms_between(t_start, t_end));   // solve.cc:641

  // ---- --record_file: this run's problem record (include/lfr_graph.h), from the reference roots
  std::vector<uint8_t> record_out;
  if (have_record) {
    int64_t got = -1;
    if (plan) {
      const int64_t need_r = lfr_plan_problem_record(plan, nullptr, n_ids, name_blob.data(),
                                                     name_off.data(), nullptr, 0);
      record_out.resize(need_r > 0 ? (size_t)need_r : 0);
      got = need_r < 0 ? need_r
                       : lfr_plan_problem_record(plan, nullptr, n_ids, name_blob.data(), name_off.data(),
                                                 record_out.data(), record_out.size());
    } else {
      const lfr_problem cur = host_problem();
      const int64_t need_r = lfr_host_problem_record(&cur, node_image.data(), node_feat.data(), n_ids,
                                                     name_blob.data(), name_off.data(), nullptr, 0);
      record_out.resize(need_r > 0 ? (size_t)need_r : 0);
      got = need_r < 0 ? need_r
                       : lfr_host_problem_record(&cur, node_image.data(), node_feat.data(), n_ids,
                                                 name_blob.data(), name_off.data(), record_out.data(), record_out.size());
    }
    if (got < 0 || (uint64_t)got != record_out.size()) {
      std::fprintf(stderr, "ERROR: the problem record failed (%d): %s\n", (int)got, lfr_last_error());
      return 2;
    }
  }

  // ---- SolutionFile (solve.cc:643-679): images by first node appearance, nodes by index ------
  uint64_t n_outside = 0;
  int64_t need = 0;
  uint8_t* out = nullptr;
  bool out_pinned = false;
  // scene sc's SolutionFile is out[scene_off[sc], scene_off[sc + 1])
  std::vector<uint64_t> scene_off(S + 1, 0), scene_outside(S, 0);
  if (plan) {
    // encoded on the GPU, names and facts indexed by image id, into page-locked memory sized by the
    // largest encoding: a Displacement record is at most 18 bytes, an Image's header 16 plus its name field
    uint64_t cap = 18ull * N;
    cap += 27ull * n_ids + name_blob.size();
    // carried entries: a file's canonical encoding bounds what it adds; a larger need takes a second call
    if (carry_start) cap += start_file.size();
    auto encode = [&](uint8_t* o, uint64_t c) {
      return carry_start ? lfr_plan_encode_solution_carried(plan, nullptr, n_ids, name_blob.data(),
                                                            name_off.data(), image_fact.data(), start_file.data(),
                                                            start_file.size(), o, c, &n_outside, nullptr)
                         : have_query ? lfr_plan_encode_solution_images(plan, nullptr, n_ids, name_blob.data(), name_off.data(),
                                                                        image_fact.data(), image_written.data(), o, c, &n_outside)
                         : batched ? lfr_plan_encode_solution_groups(plan, nullptr, n_ids, name_blob.data(), name_off.data(),
                                                                         image_fact.data(), image_group.data(), S, o, c,
                                                                         scene_off.data(), scene_outside.data())
                         : lfr_plan_encode_solution(plan, nullptr, n_ids, name_blob.data(), name_off.data(),
                                                    image_fact.data(), o, c, &n_outside);
    };
    out = static_cast<uint8_t*>(lfr_host_alloc(cap));
    out_pinned = out != nullptr;
    if (!out) out = static_cast<uint8_t*>(std::malloc(cap ? cap : 1));
    need = encode(out, cap);
    if (need > 0 && (uint64_t)need > cap) {
      if (out_pinned) lfr_host_free(out); else std::free(out);
      cap = (uint64_t)need;
      out = static_cast<uint8_t*>(lfr_host_alloc(cap));
      out_pinned = out != nullptr;
      if (!out) out = static_cast<uint8_t*>(std::malloc(cap));
      need = encode(out, cap);
    }
    lfr_plan_destroy(plan);
    if (need < 0 || (uint64_t)need > cap) {
      std::fprintf(stderr, "ERROR: the solve failed (%d): %s\n", (int)need, lfr_last_error());
      return 2;
    }
    if (batched)
      for (uint64_t c : scene_outside) n_outside += c;
    else
      scene_off[1] = (uint64_t)need;
  } else {
    // with --query_images only the query images are written (a database image's keypoints have one value
    // per query): rank -2 marks the images left out; every node still counts towards n_outside
    std::vector<int64_t> rank(n_ids, -1);
    std::vector<uint32_t> img_ids;
    for (uint32_t v = 0; v < N; ++v)
      if (rank[node_image[v]] == -1) {
        if (!image_written[node_image[v]]) {
          rank[node_image[v]] = -2;
          continue;
        }
        rank[node_image[v]] = (int64_t)img_ids.size();
        img_ids.push_back(node_image[v]);
      }
    // with --additional_scenes (--listed_pairs) the images go scene (list) after scene, each one's in the order above
    std::vector<size_t> scene_img(S + 1, 0);
    if (batched) {
      std::stable_sort(img_ids.begin(), img_ids.end(),
                       [&](uint32_t x, uint32_t y) { return image_group[x] < image_group[y]; });
      for (size_t i = 0; i < img_ids.size(); ++i) {
        rank[img_ids[i]] = (int64_t)i;
        ++scene_img[image_group[img_ids[i]] + 1];
      }
      for (uint32_t sc = 0; sc < S; ++sc) scene_img[sc + 1] += scene_img[sc];
    } else {
      scene_img[1] = img_ids.size();
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
        if (std::fabs(positions[2 * (size_t)v + 1]) > 0.5 || std::fabs(positions[2 * (size_t)v]) > 0.5) ++n_outside;  // solve.cc:666-669
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
      const std::string& s = names[orig_of[img_ids[i]]];
      out_blob.insert(out_blob.end(), s.begin(), s.end());
      out_off[i + 1] = out_blob.size();
      fact[i] = image_fact[img_ids[i]];
    }
    if (out_blob.empty()) out_blob.push_back(0);
    // the images [a, b) of the output order: one scene's SolutionFile
    auto encode = [&](size_t a, size_t b, uint8_t* o, uint64_t c) {
      return carry_start ? lfr_wire_encode_solution_carried(b - a, img_ptr.data() + a, out_blob.data(), out_off.data() + a,
                                                            fact.data() + a, feature_idx.data(), di.data(), dj.data(),
                                                            start_file.data(), start_file.size(), o, c, nullptr)
                         : lfr_wire_encode_solution(b - a, img_ptr.data() + a, out_blob.data(), out_off.data() + a,
                                                    fact.data() + a, feature_idx.data(), di.data(), dj.data(), o, c);
    };
    for (uint32_t sc = 0; sc < S && need >= 0; ++sc) {
      const int64_t n = encode(scene_img[sc], scene_img[sc + 1], nullptr, 0);
      need = n < 0 ? -1 : need + n;
      scene_off[sc + 1] = (uint64_t)need;
    }
    out = static_cast<uint8_t*>(std::malloc((size_t)std::max<int64_t>(need, 1)));
    for (uint32_t sc = 0; sc < S && need >= 0; ++sc) {
      const uint64_t n = scene_off[sc + 1] - scene_off[sc];
      if (encode(scene_img[sc], scene_img[sc + 1], out + scene_off[sc], n) != (int64_t)n) need = -1;
    }
  }
  start_file.release();
  std::printf("# points with at least one coordinate > 0.5: %llu\n", (unsigned long long)n_outside);  // solve.cc:670
  std::fflush(stdout);
  bool written = need >= 0;
  for (uint32_t sc = 0; written && sc < S; ++sc) {  // in scene order; the first failure ends the run
    std::ofstream f(scenes[sc].second, std::ios::binary | std::ios::trunc);
    written = f.good();
    const uint64_t n = scene_off[sc + 1] - scene_off[sc];
    if (written && n) f.write(reinterpret_cast<const char*>(out + scene_off[sc]), (std::streamsize)n);
    written = written && f.good();
  }
  if (positions_pinned) lfr_host_free(positions); else std::free(positions);
  if (edges_pinned) lfr_host_free(edges); else std::free(edges);
  if (out_pinned) lfr_host_free(out); else std::free(out);
  if (!written) {
    std::fputs("Failed to write proto object.\n", stderr);  // solve.cc:674-677
    return 255;
  }
  if (have_record) {
    std::ofstream f(record_file, std::ios::binary | std::ios::trunc);
    if (f.good()) f.write(reinterpret_cast<const char*>(record_out.data()), (std::streamsize)record_out.size());
    if (!f.good()) {
      std::fprintf(stderr, "ERROR: cannot write the record file '%s'\n", record_file.c_str());
      return 255;
    }
  }
  return 0;
}
