// Plan files: the autotuner's tilings (engine.cu autotune_tc) and form_chains' chain-or-separate decisions of a handle,
// written as text and read back by another handle or process, which then times nothing the file covers.
//
//   yolact_b200 plans 1
//   build <yb_build_id()>
//   device <cudaDeviceProp::name>
//   compute_capability <major>.<minor>
//   sms <multiprocessors>
//   precision <f32 | f16tc | f16x3>
//   sk_candidates <0|1>
//   chain_mode <0|1|2>
//   pdl <0|1>
//   entries <n>
//   tiling <key> bn=<> stages=<> grid=<> pair=<> mma_groups=<> pdl_friendly=<> stream_k=<> chain=<>    (n lines,
//   chain <key> <chain | separate>                                                                       any mix)
//   end
//
// Entries are sorted (tilings, then chains, each by key), so a save right after a load writes the loaded bytes.
#include <ctype.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <sstream>

#include "engine.cuh"

#ifndef YB_BUILD_ID
#define YB_BUILD_ID "unversioned"   // yolact_b200/build.py passes a hash of the sources and compiler flags
#endif

namespace yb {

namespace {

constexpr int kPlanVersion = 1;
const char* const kMagic = "yolact_b200 plans ";

[[noreturn]] void bad(const std::string& msg) { throw Error(YB_ERR_INVALID, "plan file: " + msg); }

int parse_int(const std::string& s, const std::string& what) {
  if (s.empty() || s.size() > 10) bad(what + ": '" + s + "' is not an integer");
  char* end = nullptr;
  const long v = strtol(s.c_str(), &end, 10);
  if (*end != '\0' || !(isdigit((unsigned char)s[0]) || (s[0] == '-' && s.size() > 1))) bad(what + ": '" + s + "' is not an integer");
  return (int)v;
}

std::vector<std::string> split_spaces(const std::string& s) {
  std::vector<std::string> out;
  std::string cur;
  for (char c : s) {
    if (c == ' ') {
      out.push_back(cur);
      cur.clear();
    } else {
      cur += c;
    }
  }
  out.push_back(cur);
  return out;
}

const char* const kTilingFields[8] = {"bn", "stages", "grid", "pair", "mma_groups", "pdl_friendly", "stream_k", "chain"};

TcTiling parse_tiling(const std::vector<std::string>& tok, const std::string& where) {
  // tok[0] = "tiling", tok[1] = key, then exactly the eight fields in order
  if (tok.size() != 10) bad(where + ": a tiling has " + std::to_string(tok.size() - 2) + " fields, not 8");
  int v[8];
  for (int i = 0; i < 8; ++i) {
    const std::string& t = tok[2 + i];
    const size_t eq = t.find('=');
    const std::string name = t.substr(0, eq);
    if (eq == std::string::npos || name != kTilingFields[i])
      bad(where + ": field '" + name + "' where '" + kTilingFields[i] + "' belongs");
    v[i] = parse_int(t.substr(eq + 1), where + " field '" + name + "'");
  }
  TcTiling t;
  t.bn = v[0];
  t.stages = v[1];
  t.grid = v[2];
  t.pair = v[3];
  t.mma_groups = v[4];
  t.pdl_friendly = v[5];
  t.stream_k = v[6];
  t.chain = v[7];
  const bool ok_bn = t.bn == 32 || t.bn == 64 || t.bn == 128 || t.bn == 256;
  if (!ok_bn) bad(where + ": field 'bn' must be 32, 64, 128 or 256");
  if (t.stages < 1 || t.stages > 8) bad(where + ": field 'stages' must be 1..8");
  if (t.grid < 1) bad(where + ": field 'grid' must be positive");
  if (t.pair != 0 && t.pair != 1) bad(where + ": field 'pair' must be 0 or 1");
  if (t.mma_groups != 1 && t.mma_groups != 2) bad(where + ": field 'mma_groups' must be 1 or 2");
  if (t.pdl_friendly != 0 && t.pdl_friendly != 1) bad(where + ": field 'pdl_friendly' must be 0 or 1");
  if (t.stream_k != 0 && t.stream_k != 1) bad(where + ": field 'stream_k' must be 0 or 1");
  if (t.chain != 0) bad(where + ": field 'chain' must be 0 (the autotuner plans single launches)");
  return t;
}

bool same_tiling(const TcTiling& a, const TcTiling& b) {
  return a.bn == b.bn && a.stages == b.stages && a.grid == b.grid && a.pair == b.pair && a.mma_groups == b.mma_groups &&
         a.pdl_friendly == b.pdl_friendly && a.stream_k == b.stream_k && a.chain == b.chain;
}

const char* precision_name(int p) {
  return p == YB_PREC_F32 ? "f32" : p == YB_PREC_F16TC ? "f16tc" : p == YB_PREC_F16X3 ? "f16x3" : "unknown";
}

}  // namespace

const char* build_id() { return YB_BUILD_ID; }

PlanFile parse_plan_file(const std::string& text) {
  std::vector<std::string> lines;
  {
    size_t b = 0;
    while (b < text.size()) {
      const size_t e = text.find('\n', b);
      if (e == std::string::npos) bad("truncated: the last line has no newline");
      lines.push_back(text.substr(b, e - b));
      b = e + 1;
    }
  }
  size_t ln = 0;
  auto next = [&](const std::string& what) -> const std::string& {
    if (ln >= lines.size()) bad("truncated: " + what + " is missing");
    return lines[ln++];
  };
  const std::string& first = next("the version line");
  if (first.compare(0, strlen(kMagic), kMagic) != 0) bad("line 1: not a yolact_b200 plan file");
  const std::string ver = first.substr(strlen(kMagic));
  if (ver != std::to_string(kPlanVersion)) bad("field 'version' is '" + ver + "', this library reads " + std::to_string(kPlanVersion));

  PlanFile f;
  auto field = [&](const char* name) -> std::string {
    const std::string& l = next(std::string("header field '") + name + "'");
    const size_t sp = l.find(' ');
    const std::string got = l.substr(0, sp);
    if (got != name) bad("line " + std::to_string(ln) + ": header field '" + got + "' where '" + name + "' belongs");
    if (sp == std::string::npos || sp + 1 >= l.size()) bad("header field '" + std::string(name) + "' has no value");
    return l.substr(sp + 1);
  };
  f.hdr.build = field("build");
  if (f.hdr.build != build_id())
    bad("field 'build' is '" + f.hdr.build + "', this library's build id is '" + build_id() + "'");
  f.hdr.device = field("device");
  f.hdr.cc = field("compute_capability");
  f.hdr.sms = parse_int(field("sms"), "field 'sms'");
  f.hdr.precision = field("precision");
  f.hdr.sk_candidates = parse_int(field("sk_candidates"), "field 'sk_candidates'");
  f.hdr.chain_mode = parse_int(field("chain_mode"), "field 'chain_mode'");
  f.hdr.pdl = parse_int(field("pdl"), "field 'pdl'");
  const int n = parse_int(field("entries"), "field 'entries'");
  if (n < 0) bad("field 'entries' is negative");
  for (int e = 0; e < n; ++e) {
    const std::string where = "line " + std::to_string(ln + 1);
    const std::vector<std::string> tok = split_spaces(next("entry " + std::to_string(e + 1) + " of " + std::to_string(n)));
    if (tok.size() < 2 || tok[1].empty()) bad(where + ": an entry needs a kind and a key");
    const std::string& key = tok[1];
    if (tok[0] == "tiling") {
      const TcTiling t = parse_tiling(tok, where);
      if (!f.tilings.emplace(key, t).second) bad(where + ": duplicate tiling key " + key);
    } else if (tok[0] == "chain") {
      if (tok.size() != 3 || (tok[2] != "chain" && tok[2] != "separate"))
        bad(where + ": a chain entry's value is 'chain' or 'separate'");
      if (!f.chains.emplace(key, tok[2] == "chain").second) bad(where + ": duplicate chain key " + key);
    } else {
      bad(where + ": unknown entry kind '" + tok[0] + "'");
    }
  }
  if (next("the end line") != "end") bad("line " + std::to_string(ln) + ": expected 'end' after " + std::to_string(n) + " entries");
  if (ln != lines.size()) bad("line " + std::to_string(ln + 1) + ": text after the end line");
  return f;
}

std::string write_plan_file(const PlanFile& f) {
  std::ostringstream o;
  o << kMagic << kPlanVersion << "\n";
  o << "build " << f.hdr.build << "\n";
  o << "device " << f.hdr.device << "\n";
  o << "compute_capability " << f.hdr.cc << "\n";
  o << "sms " << f.hdr.sms << "\n";
  o << "precision " << f.hdr.precision << "\n";
  o << "sk_candidates " << f.hdr.sk_candidates << "\n";
  o << "chain_mode " << f.hdr.chain_mode << "\n";
  o << "pdl " << f.hdr.pdl << "\n";
  o << "entries " << f.tilings.size() + f.chains.size() << "\n";
  for (const auto& kv : f.tilings) {
    const TcTiling& t = kv.second;
    o << "tiling " << kv.first << " bn=" << t.bn << " stages=" << t.stages << " grid=" << t.grid << " pair=" << t.pair
      << " mma_groups=" << t.mma_groups << " pdl_friendly=" << t.pdl_friendly << " stream_k=" << t.stream_k
      << " chain=" << t.chain << "\n";
  }
  for (const auto& kv : f.chains) o << "chain " << kv.first << " " << (kv.second ? "chain" : "separate") << "\n";
  o << "end\n";
  return o.str();
}

std::string read_text_file(const std::string& path) {
  FILE* fp = fopen(path.c_str(), "rb");
  if (!fp) throw Error(YB_ERR_INVALID, "plan file: cannot open " + path);
  std::string s;
  char buf[1 << 16];
  size_t n;
  while ((n = fread(buf, 1, sizeof(buf), fp)) > 0) s.append(buf, n);
  const bool err = ferror(fp) != 0;
  fclose(fp);
  if (err) throw Error(YB_ERR_INVALID, "plan file: cannot read " + path);
  return s;
}

// Writes next to `path` and renames over it, so that a reader never sees half a file.
void write_text_file(const std::string& path, const std::string& text) {
  const std::string tmp = path + ".tmp";
  FILE* fp = fopen(tmp.c_str(), "wb");
  if (!fp) throw Error(YB_ERR_INVALID, "plan file: cannot create " + tmp);
  const bool ok = fwrite(text.data(), 1, text.size(), fp) == text.size();
  if (fclose(fp) != 0 || !ok || rename(tmp.c_str(), path.c_str()) != 0) {
    remove(tmp.c_str());
    throw Error(YB_ERR_INVALID, "plan file: cannot write " + path);
  }
}

}  // namespace yb

using namespace yb;

PlanHeader yb_handle::plan_header() const {
  cudaDeviceProp prop;
  YB_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  PlanHeader hd;
  hd.build = build_id();
  hd.device = prop.name;
  hd.cc = std::to_string(prop.major) + "." + std::to_string(prop.minor);
  hd.sms = prop.multiProcessorCount;
  hd.precision = precision_name(cfg.precision);
  hd.sk_candidates = sk_candidates ? 1 : 0;
  hd.chain_mode = chain_mode;
  hd.pdl = pdl ? 1 : 0;
  return hd;
}

void yb_handle::save_plans(const std::string& path) const {
  PlanFile f;
  f.hdr = plan_header();
  for (const auto& kv : tune_cache) f.tilings[kv.first] = kv.second.t;
  for (const auto& kv : chain_cache) f.chains[kv.first] = kv.second.chain;
  write_text_file(path, write_plan_file(f));
}

void yb_handle::load_plans(const std::string& path) {
  const PlanFile f = parse_plan_file(read_text_file(path));
  const PlanHeader mine = plan_header();
  auto refuse = [](const std::string& name, const std::string& theirs, const std::string& ours) {
    bad("field '" + name + "' is '" + theirs + "', this handle's is '" + ours + "'");
  };
  if (f.hdr.device != mine.device) refuse("device", f.hdr.device, mine.device);
  if (f.hdr.cc != mine.cc) refuse("compute_capability", f.hdr.cc, mine.cc);
  if (f.hdr.sms != mine.sms) refuse("sms", std::to_string(f.hdr.sms), std::to_string(mine.sms));
  if (f.hdr.precision != mine.precision) refuse("precision", f.hdr.precision, mine.precision);
  if (f.hdr.sk_candidates != mine.sk_candidates)
    refuse("sk_candidates", std::to_string(f.hdr.sk_candidates), std::to_string(mine.sk_candidates));
  if (f.hdr.chain_mode != mine.chain_mode) refuse("chain_mode", std::to_string(f.hdr.chain_mode), std::to_string(mine.chain_mode));
  if (f.hdr.pdl != mine.pdl) refuse("pdl", std::to_string(f.hdr.pdl), std::to_string(mine.pdl));
  // shapes this handle has planned already must agree before anything is merged
  for (const auto& kv : f.tilings) {
    auto it = tune_cache.find(kv.first);
    if (it != tune_cache.end() && !same_tiling(it->second.t, kv.second))
      bad("tiling " + kv.first + " is '" + tc_tiling_str(kv.second) + "', this handle planned '" +
          tc_tiling_str(it->second.t) + "'");
  }
  for (const auto& kv : f.chains) {
    auto it = chain_cache.find(kv.first);
    if (it != chain_cache.end() && it->second.chain != kv.second)
      bad(std::string("chain ") + kv.first + " is '" + (kv.second ? "chain" : "separate") + "', this handle decided '" +
          (it->second.chain ? "chain" : "separate") + "'");
  }
  for (const auto& kv : f.tilings)
    if (!tune_cache.count(kv.first)) tune_cache[kv.first] = TunedTiling{kv.second, true};
  for (const auto& kv : f.chains)
    if (!chain_cache.count(kv.first)) chain_cache[kv.first] = ChainChoice{kv.second, true};
}
