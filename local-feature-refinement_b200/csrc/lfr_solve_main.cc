// lfr_solve_main.cc — native `solve` executable: the command-line surface of the reference's
// multi-view-refinement/solve.cc main() (solve.cc:375-682) above the C ABI.
//
//     solve --matches_file X.pb --output_file Y.pb [--n_threads 8] [--banned_images NAME]...
//
// Same flags (solve.cc:379-385, Boost.Program_options semantics and messages), same `.part.N` handling
// (:416-424), same stdout lines (:484-485,534,549,589,591,606,638,641,670) and exit codes (0; 1 on a
// command-line error, :397-401; -1 = 255 when the input does not parse or the output cannot be
// written, :433-436,674-677).  The work is lfr_wire_walk_matches() (include/lfr_wire.h) over the pairs,
// the graph stage and the solve, then lfr_wire_encode_solution().  The graph stage runs where
// lfr_graph_stage_on_device() (include/lfr_graph.h) says, from the pair level alone:
//   device: lfr_plan_create_from_wire() on the mapped parts (the matches are decoded on the GPU) — or,
//           below the match count lfr_wire_decode_on_device() sets, lfr_wire_decode_matches() +
//           lfr_plan_create_from_matches() —, lfr_plan_solve() + lfr_plan_download() on the plan left
//           in HBM, and lfr_plan_export_graph() for the node -> (image, feature) ids;
//   host:   lfr_wire_decode_matches(), lfr_host_stage_create() (include/lfr_host.h) writing the edge
//           records into page-locked memory, then lfr_solve() / lfr_solve_multi() (include/lfr.h).
// Both routes give the same bytes and lines.  LFR_GRAPH_STAGE=host|device forces a route (a test and
// measurement hook).  Opt-in extras: --device D, --gpus N (one process drives N GPUs; host route).  `--n_threads` is accepted and
// ignored (the solve runs on the GPU).  local-feature-refinement_b200/cli.py is the same program in
// Python; this one starts in milliseconds instead of importing numpy.
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
#include <vector>

#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "../../include/lfr.h"
#include "../../include/lfr_graph.h"
#include "../../include/lfr_host.h"
#include "../../include/lfr_wire.h"

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
int lfr_plan_export_graph(const lfr_plan* plan, uint32_t* row_ptr, lfr_edge* edges, uint32_t* track, uint32_t* comp,
                          uint8_t* is_root, uint32_t* comp_ptr, uint32_t* comp_nodes, uint32_t* comp_order,
                          uint32_t* node_image, uint32_t* node_feat) __attribute__((weak));
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
                               {"gpus", true, false}};

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
  bool help = false;
  std::map<std::string, std::string> single;
  std::vector<std::string> banned;
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
          a.banned.push_back(v);
        } else if (a.single.count(o.name)) {
          throw CliError{std::string("option '--") + o.name + "' cannot be specified more than once"};
        } else {
          a.single[o.name] = v;
        }
      } else {
        if (eq != std::string::npos) throw CliError{std::string("option '--") + o.name + "' does not take any arguments"};
        a.help = true;
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

using Clock = std::chrono::steady_clock;
long long ms_between(Clock::time_point a, Clock::time_point b) {
  return (long long)std::chrono::duration_cast<std::chrono::milliseconds>(b - a).count();
}

}  // namespace

int main(int argc, char** argv) {
  std::string matches_file, output_file;
  std::vector<std::string> banned_list;
  uint64_t device = 0, gpus = 1;
  try {
    const Args a = parse(argc, argv);
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
    banned_list = a.banned;
  } catch (const CliError& e) {  // solve.cc:397-401
    std::fprintf(stderr, "ERROR: %s\n\n", e.msg.c_str());
    std::fputs(kUsage, stderr);
    return 1;
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

  // ---- solve.cc:412-481: the file, or its .part.N pieces ------------------------------------
  std::vector<std::string> files;
  if (file_exists(matches_file)) {
    files.push_back(matches_file);
  } else {
    for (int k = 0;; ++k) {
      const std::string f = matches_file + ".part." + std::to_string(k);
      if (!file_exists(f)) break;
      files.push_back(f);
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

  // image names -> ids in order of first appearance over all parts; the pairs of all parts in order
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
  {
    uint64_t p0 = 0, m0 = 0;
    for (Part& pt : parts) {
      for (uint64_t p = 0; p < pt.P; ++p) {
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

  // banned images (solve.cc:444-446) and the first fact seen of every image among the pairs kept
  const std::set<std::string> banned(banned_list.begin(), banned_list.end());
  std::vector<uint8_t> skip(P, 0);
  std::vector<float> image_fact(names.size(), 0.f);
  std::vector<uint8_t> have_fact(names.size(), 0);
  uint64_t e_cap = 0;
  for (uint64_t p = 0; p < P; ++p) {
    skip[p] = (banned.count(names[pair_img1[p]]) || banned.count(names[pair_img2[p]])) ? 1 : 0;
    if (skip[p]) continue;
    e_cap += 2 * (pair_ptr[p + 1] - pair_ptr[p]);
    if (!have_fact[pair_img1[p]]) { have_fact[pair_img1[p]] = 1; image_fact[pair_img1[p]] = pair_fact1[p]; }
    if (!have_fact[pair_img2[p]]) { have_fact[pair_img2[p]] = 1; image_fact[pair_img2[p]] = pair_fact2[p]; }
  }

  lfr_host_input in;
  std::memset(&in, 0, sizeof in);
  in.n_pairs = P; in.n_matches = M; in.n_images = (uint32_t)names.size();
  in.pair_img1 = pair_img1.data(); in.pair_img2 = pair_img2.data(); in.pair_skip = skip.data();
  in.pair_ptr = pair_ptr.data();

  // ---- which graph stage: the library's size rule, or LFR_GRAPH_STAGE=host|device (a test and
  // measurement hook, not a product option).  A library without the stage on the GPU — the CPU checker —
  // takes the host route; forcing the device route there is an error, never a silent host run.
  const bool have_device_stage = lfr_graph_stage_on_device && lfr_wire_decode_on_device && lfr_plan_create_from_matches &&
                                 lfr_plan_create_from_wire && lfr_plan_export_graph;
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
  // every part decoded into one set of arrays, part after part (the pair level comes out as the walk gave it)
  const bool decode_on_device = on_device && lfr_wire_decode_on_device(M) == 1;
  std::vector<uint32_t> feat1, feat2;
  std::vector<float> sim, disp1, disp2;
  if (!decode_on_device) {
    feat1.resize(M); feat2.resize(M); sim.resize(M); disp1.resize(18 * M); disp2.resize(18 * M);
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
    // in HBM for the solve and only the per-node image / feature ids come back for the SolutionFile
    lfr_options opt;
    lfr_options_default(&opt);
    opt.device = (int32_t)device;
    std::vector<lfr_wire_part> wparts;
    for (const Part& pt : parts) wparts.push_back(lfr_wire_part{pt.buf.data(), pt.buf.size(), pt.match_off.data(), pt.M});
    const int rc = decode_on_device
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
    node_image.resize(sz.n_nodes);
    node_feat.resize(sz.n_nodes);
    if (lfr_plan_export_graph(plan, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                              node_image.data(), node_feat.data()) != LFR_OK) {
      std::fprintf(stderr, "ERROR: lfr_plan_export_graph failed\n");
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

  // ---- the solve (solve.cc:608-635): positions start at zero --------------------------------
  double* positions = nullptr;
  bool positions_pinned = false;
  if (N) {
    positions = static_cast<double*>(lfr_host_alloc(2ull * N * sizeof(double)));
    positions_pinned = positions != nullptr;
    if (!positions) positions = static_cast<double*>(std::malloc(2ull * N * sizeof(double)));
    std::memset(positions, 0, 2ull * N * sizeof(double));
  }
  const Clock::time_point t_solve = Clock::now();
  if (N && plan) {
    int rc = lfr_plan_solve(plan, nullptr);
    if (rc == LFR_OK) rc = lfr_plan_download(plan, nullptr, positions, nullptr);
    if (rc != LFR_OK) {
      std::fprintf(stderr, "ERROR: the solve failed (%d): %s\n", rc, lfr_last_error());
      return 2;
    }
  } else if (N) {
    lfr_problem prob;
    prob.n_nodes = N; prob.n_components = C; prob.n_edges = E;
    prob.row_ptr = row_ptr.data(); prob.edges = edges; prob.track = track.data(); prob.comp = comp.data();
    prob.is_root = is_root.data(); prob.comp_ptr = comp_ptr.data(); prob.comp_nodes = comp_nodes.data();
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
  lfr_plan_destroy(plan);
  std::printf("Solver time: %lldms\n", ms_between(t_solve, t_end));  // solve.cc:638
  std::printf("Total time: %lldms\n", ms_between(t_start, t_end));   // solve.cc:641

  // ---- SolutionFile (solve.cc:643-679): images by first node appearance, nodes by index ------
  std::vector<int64_t> rank(names.size(), -1);
  std::vector<uint32_t> img_ids;
  for (uint32_t v = 0; v < N; ++v)
    if (rank[node_image[v]] < 0) {
      rank[node_image[v]] = (int64_t)img_ids.size();
      img_ids.push_back(node_image[v]);
    }
  const size_t I = img_ids.size();
  std::vector<uint64_t> img_ptr(I + 1, 0);
  for (uint32_t v = 0; v < N; ++v) ++img_ptr[(size_t)rank[node_image[v]] + 1];
  for (size_t i = 0; i < I; ++i) img_ptr[i + 1] += img_ptr[i];
  std::vector<uint32_t> feature_idx(N);
  std::vector<float> di(N), dj(N);
  uint64_t n_outside = 0;
  {
    std::vector<uint64_t> fill(img_ptr.begin(), img_ptr.end() - 1);
    for (uint32_t v = 0; v < N; ++v) {
      const uint64_t k = fill[(size_t)rank[node_image[v]]]++;
      feature_idx[k] = node_feat[v];
      di[k] = (float)positions[2 * (size_t)v];
      dj[k] = (float)positions[2 * (size_t)v + 1];
      if (std::fabs(positions[2 * (size_t)v + 1]) > 0.5 || std::fabs(positions[2 * (size_t)v]) > 0.5) ++n_outside;  // solve.cc:666-669
    }
  }
  std::printf("# points with at least one coordinate > 0.5: %llu\n", (unsigned long long)n_outside);  // solve.cc:670
  std::fflush(stdout);
  std::vector<uint8_t> name_blob;
  std::vector<uint64_t> name_off(I + 1, 0);
  std::vector<float> fact(I);
  for (size_t i = 0; i < I; ++i) {
    const std::string& s = names[img_ids[i]];
    name_blob.insert(name_blob.end(), s.begin(), s.end());
    name_off[i + 1] = name_blob.size();
    fact[i] = image_fact[img_ids[i]];
  }
  if (name_blob.empty()) name_blob.push_back(0);
  const int64_t need = lfr_wire_encode_solution(I, img_ptr.data(), name_blob.data(), name_off.data(), fact.data(),
                                                feature_idx.data(), di.data(), dj.data(), nullptr, 0);
  std::vector<uint8_t> out((size_t)std::max<int64_t>(need, 1));
  bool written = need >= 0 && lfr_wire_encode_solution(I, img_ptr.data(), name_blob.data(), name_off.data(), fact.data(),
                                                       feature_idx.data(), di.data(), dj.data(), out.data(), (uint64_t)need) == need;
  if (written) {
    std::ofstream f(output_file, std::ios::binary | std::ios::trunc);
    written = f.good();
    if (written && need) f.write(reinterpret_cast<const char*>(out.data()), need);
    written = written && f.good();
  }
  if (positions_pinned) lfr_host_free(positions); else std::free(positions);
  if (edges_pinned) lfr_host_free(edges); else std::free(edges);
  if (!written) {
    std::fputs("Failed to write proto object.\n", stderr);  // solve.cc:674-677
    return 255;
  }
  return 0;
}
