#include "export_loader.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>

namespace adn {
namespace {

// ---- protobuf wire format ------------------------------------------------------------------
struct Cursor {
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  uint64_t varint() {
    uint64_t r = 0;
    int shift = 0;
    while (p < end) {
      const uint8_t b = *p++;
      r |= uint64_t(b & 0x7F) << shift;
      if (!(b & 0x80)) return r;
      shift += 7;
      if (shift > 63) break;
    }
    ok = false;
    return 0;
  }
};

struct Field {
  uint32_t number;
  uint32_t wire;
  uint64_t value;          // wire 0
  const uint8_t* data;     // wire 1, 2, 5
  size_t size;
};

bool next_field(Cursor& c, Field& f) {
  if (c.p >= c.end || !c.ok) return false;
  const uint64_t key = c.varint();
  if (!c.ok) return false;
  f.number = uint32_t(key >> 3);
  f.wire = uint32_t(key & 7);
  f.value = 0;
  f.data = nullptr;
  f.size = 0;
  switch (f.wire) {
    case 0: f.value = c.varint(); break;
    case 1:
      if (size_t(c.end - c.p) < 8) { c.ok = false; return false; }   // truncated file: an error, not "end of message"
      f.data = c.p; f.size = 8; c.p += 8;
      break;
    case 2: {
      const uint64_t n = c.varint();
      if (!c.ok || n > uint64_t(c.end - c.p)) { c.ok = false; return false; }
      f.data = c.p; f.size = size_t(n); c.p += n;
      break;
    }
    case 5:
      if (size_t(c.end - c.p) < 4) { c.ok = false; return false; }
      f.data = c.p; f.size = 4; c.p += 4;
      break;
    default: c.ok = false; return false;
  }
  return c.ok && c.p <= c.end;
}

// TensorProto: dims(1) data_type(2) float_data(4) name(8) raw_data(9)
bool parse_tensor(const uint8_t* p, size_t n, NamedTensor& t, bool& is_float) {
  Cursor c{p, p + n};
  Field f;
  std::vector<int64_t> dims;
  const uint8_t* raw = nullptr;
  size_t raw_n = 0;
  std::vector<float> floats;
  int dtype = 0;
  while (next_field(c, f)) {
    if (f.number == 1) {
      if (f.wire == 0) dims.push_back(int64_t(f.value));
      else if (f.wire == 2) { Cursor d{f.data, f.data + f.size}; while (d.p < d.end && d.ok) dims.push_back(int64_t(d.varint())); }
    } else if (f.number == 2 && f.wire == 0) {
      dtype = int(f.value);
    } else if (f.number == 4) {
      if (f.wire == 5) { float v; std::memcpy(&v, f.data, 4); floats.push_back(v); }
      else if (f.wire == 2) { const size_t k = f.size / 4; const size_t o = floats.size(); floats.resize(o + k); std::memcpy(floats.data() + o, f.data, k * 4); }
    } else if (f.number == 8 && f.wire == 2) {
      t.name.assign(reinterpret_cast<const char*>(f.data), f.size);
    } else if (f.number == 9 && f.wire == 2) {
      raw = f.data; raw_n = f.size;
    }
  }
  if (!c.ok) return false;
  is_float = (dtype == 1);
  if (!is_float) return true;
  if (raw) { t.data.resize(raw_n / 4); std::memcpy(t.data.data(), raw, raw_n / 4 * 4); }   // little-endian fp32
  else t.data = std::move(floats);
  if (dims.size() == 2) { t.rows = dims[0]; t.cols = dims[1]; }
  else if (dims.size() == 1) { t.rows = dims[0]; t.cols = 1; }
  else { t.rows = int64_t(t.data.size()); t.cols = 1; }
  return int64_t(t.data.size()) == t.rows * t.cols;
}

std::string strip(const std::string& s) {
  std::string r;
  for (char ch : s) if (!std::isspace(static_cast<unsigned char>(ch))) r.push_back(ch);
  return r;
}

// "[a, b]" / "a,b" -> tokens (whitespace stripped like Config::store, config.cpp:200-204)
std::vector<std::string> list_items(const std::string& v) {
  std::string s = strip(v);
  if (!s.empty() && s.front() == '[') s.erase(0, 1);
  if (!s.empty() && s.back() == ']') s.pop_back();
  std::vector<std::string> out;
  std::stringstream ss(s);
  std::string item;
  while (std::getline(ss, item, ',')) out.push_back(item);
  return out;
}

bool read_kv(const std::string& path, std::map<std::string, std::string>& kv) {
  std::ifstream f(path);
  if (!f) return false;
  std::string line;
  while (std::getline(f, line)) {
    const size_t eq = line.find('=');
    if (eq == std::string::npos) continue;
    kv[strip(line.substr(0, eq))] = line.substr(eq + 1);
  }
  return true;
}

bool floats_of(const std::map<std::string, std::string>& kv, const char* key, float* dst, size_t n) {
  auto it = kv.find(key);
  if (it == kv.end()) return false;
  const auto items = list_items(it->second);
  if (items.size() < n) return false;
  for (size_t i = 0; i < n; ++i) dst[i] = float(std::atof(items[i].c_str()));
  return true;
}

}  // namespace

bool read_onnx_initializers(const std::string& path, std::vector<NamedTensor>& out, std::string& err) {
  std::ifstream f(path, std::ios::binary);
  if (!f) { err = "cannot open " + path; return false; }
  std::vector<uint8_t> buf((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  Cursor c{buf.data(), buf.data() + buf.size()};
  Field fld;
  while (next_field(c, fld)) {
    if (fld.number == 7 && fld.wire == 2) {  // ModelProto.graph
      Cursor g{fld.data, fld.data + fld.size};
      Field gf;
      while (next_field(g, gf)) {
        if (gf.number == 5 && gf.wire == 2) {  // GraphProto.initializer
          NamedTensor t;
          bool is_float = false;
          if (!parse_tensor(gf.data, gf.size, t, is_float)) { err = "malformed initializer in " + path; return false; }
          if (is_float) out.push_back(std::move(t));
        }
      }
      if (!g.ok) { err = "malformed graph in " + path; return false; }
    }
  }
  if (!c.ok) { err = "malformed protobuf " + path; return false; }
  if (out.empty()) { err = "no fp32 initializers in " + path; return false; }
  return true;
}

bool load_export_dir(const std::string& dir_in, ExportDir& out, std::string& err) {
  std::string dir = dir_in;
  if (!dir.empty() && dir.back() != '/') dir.push_back('/');
  std::map<std::string, std::string> cfg, info;
  if (!read_kv(dir + "config.ini", cfg)) { err = "cannot read " + dir + "config.ini"; return false; }
  if (!read_kv(dir + "dataset_info.txt", info)) { err = "cannot read " + dir + "dataset_info.txt"; return false; }
  adn_scene& s = out.scene;
  float fov = 0, md = 0;
  if (!floats_of(info, "view_cell_center", s.view_cell_center, 3) || !floats_of(info, "view_cell_size", s.view_cell_size, 3) ||
      !floats_of(info, "depth_range", s.depth_range, 2) || !floats_of(info, "fov", &fov, 1) || !floats_of(info, "max_depth", &md, 1)) {
    err = "dataset_info.txt: missing view_cell_center / view_cell_size / depth_range / fov / max_depth";
    return false;
  }
  s.fov = fov;
  s.max_depth = md;
  // A one-network export (plain NeRF: inFeatures = [RayMarchFromPoses], rayMarchSampler = [LinearlySpacedZNearZFar]) has
  // one-item lists; its network is model0.onnx and goes to the shading slot
  auto sm = cfg.find("rayMarchSampler");
  const auto sitems = sm == cfg.end() ? std::vector<std::string>{} : list_items(sm->second);
  const bool one_net = sitems.size() == 1;
  const size_t n_nets = one_net ? 1 : 2;
  float zn[2] = {0.001f, 0.001f}, zf[2] = {1.0f, 1.0f};
  floats_of(cfg, "zNear", zn, n_nets);
  floats_of(cfg, "zFar", zf, n_nets);
  s.z_near = zn[n_nets - 1];
  s.z_far = zf[n_nets - 1];
  s.n_freq_pos = 10;
  s.n_freq_dir = 4;
  auto pe = cfg.find("posEncArgs");
  if (pe != cfg.end()) {
    const auto items = list_items(pe->second);   // [sampling net, shading net], e.g. [10-4, 10-4] or [2-2, 10-4]
    auto parse = [](const std::string& it, int32_t& pos, int32_t& dir) {
      const size_t dash = it.find('-');
      if (dash == std::string::npos) return;
      pos = std::atoi(it.substr(0, dash).c_str());
      dir = std::atoi(it.substr(dash + 1).c_str());
    };
    if (!items.empty()) parse(items.back(), s.n_freq_pos, s.n_freq_dir);
    if (items.size() >= 2) {
      parse(items.front(), s.n_freq_pos0, s.n_freq_dir0);
      // in adn_scene a sampling-net count of 0 means "the shading net's": a literal 0 bands (e.g. "0-4") is -1 there
      if (s.n_freq_pos0 == 0) s.n_freq_pos0 = -1;
      if (s.n_freq_dir0 == 0) s.n_freq_dir0 = -1;
    }
  }
  // posEnc = [sampling net, shading net] (config.cpp:209-210): nerf, or none -- the identity, whatever posEncArgs says
  // (NoEncoding ignores the band counts); recorded as -1 / -1 (the reference's own convention, features.py:326-328)
  auto penc = cfg.find("posEnc");
  if (penc != cfg.end()) {
    const auto items = list_items(penc->second);
    for (size_t k = 0; k < items.size() && k < 2; ++k) {
      const bool shading = k == 0;   // the last item, then the first
      const std::string& e = items[items.size() - 1 - k];
      if (e == "none") {
        (shading ? s.n_freq_pos : s.n_freq_pos0) = -1;
        (shading ? s.n_freq_dir : s.n_freq_dir0) = -1;
      } else if (e != "nerf") {
        err = "config.ini: posEnc = " + strip(penc->second) + ": only nerf and none are supported";
        return false;
      }
    }
  }
  {
    // the limits of the packed input tiles (adn_create): shading P <= 20 and D <= 10 bands, sampling P0 + D0 <= 20
    const int p = std::max(0, s.n_freq_pos), d = std::max(0, s.n_freq_dir);
    const int p0 = std::max(0, s.n_freq_pos0 ? s.n_freq_pos0 : s.n_freq_pos), d0 = std::max(0, s.n_freq_dir0 ? s.n_freq_dir0 : s.n_freq_dir);
    if (p > 20 || d > 10 || p0 + d0 > 20) {
      err = "config.ini: posEncArgs = " + (pe != cfg.end() ? strip(pe->second) : std::string("?")) +
            " is outside the supported encodings (shading net at most 20-10 bands, sampling net at most 20 bands in all)";
      return false;
    }
  }
  auto ndc = cfg.find("useNDC");
  s.use_ndc = (ndc != cfg.end() && strip(ndc->second) == "True") ? 1 : 0;   // config.cpp:265-266
  if (s.use_ndc) {
    // the reference's export does not record the image size (src/export.py:47-54); accept optional w / h / focal keys,
    // otherwise ndc_rays uses the size of the frame being rendered (featureset.cpp:83-84)
    float v = 0;
    if (floats_of(info, "w", &v, 1)) s.ndc_w = int32_t(v);
    if (floats_of(info, "h", &v, 1)) s.ndc_h = int32_t(v);
  }
  auto th = cfg.find("adaptiveSamplingThreshold");
  out.threshold = th == cfg.end() ? 0.0f : float(std::atof(strip(th->second).c_str()));
  auto ns = cfg.find("numRaymarchSamples");
  if (ns == cfg.end()) { err = "config.ini: numRaymarchSamples missing"; return false; }
  const auto nitems = list_items(ns->second);
  if (nitems.empty()) { err = "config.ini: numRaymarchSamples empty"; return false; }
  out.num_samples = std::atoi(nitems.back().c_str());
  auto check = [&](const char* key, const char* want) {
    auto it = cfg.find(key);
    if (it == cfg.end()) return true;
    const auto items = list_items(it->second);
    return items.empty() || items.back() == want;
  };
  auto value_of = [&](const char* key) {
    auto it = cfg.find(key);
    return it == cfg.end() ? std::string("(missing)") : strip(it->second);
  };
  if (one_net) {
    // LinearlySpacedZNearZFar (src/nerf_raymarch_common.py:293-326; NoDepthRange on NDC scenes, :261-289): K evenly spaced
    // samples from the camera, one NeRF net, the density composite (features.py:564-577).  The depths are warped with
    // dataset_info.txt's depth_range, as the viewer does: src/export.py:50 writes the warped range there, while a Python run
    // without SpherePosDir places them with the dataset's unwarped range (datasets.py:154-159); see INTEGRATION.md.
    auto inf = cfg.find("inFeatures");
    const auto fitems = inf == cfg.end() ? std::vector<std::string>{} : list_items(inf->second);
    if (fitems.size() != 1 || fitems[0] != "RayMarchFromPoses") {
      err = "config.ini: a one-network export needs inFeatures = [RayMarchFromPoses], not " + value_of("inFeatures");
      return false;
    }
    if (s.use_ndc) {
      if (sitems[0] != "LinearlySpacedZNearZFarNoDepthRange" || !check("rayMarchNormalization", "None")) {
        err = "config.ini: a one-network NDC export must use rayMarchSampler = [LinearlySpacedZNearZFarNoDepthRange] and "
              "rayMarchNormalization = [None], not " + value_of("rayMarchSampler") + " / " + value_of("rayMarchNormalization");
        return false;
      }
    } else if (sitems[0] != "LinearlySpacedZNearZFar" || !check("rayMarchNormalization", "InverseSqrtDistCentered") ||
               !check("depthTransform", "log")) {
      err = "config.ini: a one-network export must use rayMarchSampler = [LinearlySpacedZNearZFar], rayMarchNormalization = "
            "[InverseSqrtDistCentered] and depthTransform = log (or LinearlySpacedZNearZFarNoDepthRange / None with useNDC), not " +
            value_of("rayMarchSampler") + " / " + value_of("rayMarchNormalization") + " / " + value_of("depthTransform");
      return false;
    }
    out.sampler = 2;
  } else if (!sitems.empty() && sitems.back() == "FromClassifiedDepth") {
    // FromClassifiedDepth (the DONeRF sampler, src/nerf_raymarch_common.py:606-660) returns z only, so the composite is
    // nerf_raw2outputs without OracleWeights and accumulationMult does not apply; its transform of raw0 is chosen by
    // losses[0] (:625-637)
    if (s.use_ndc || !check("rayMarchNormalization", "InverseSqrtDistCentered") || !check("depthTransform", "log")) {
      err = "config.ini: FromClassifiedDepth exports must use InverseSqrtDistCentered / log and no NDC";
      return false;
    }
    auto lo = cfg.find("losses");
    const auto litems = lo == cfg.end() ? std::vector<std::string>{} : list_items(lo->second);
    const std::string loss0 = litems.empty() ? std::string("") : litems.front();
    if (loss0 == "BCEWithLogitsLoss") {
      out.pdf_transform = 1;
    } else if (loss0 == "CrossEntropyLoss" || loss0 == "CrossEntropyLossWeighted") {
      out.pdf_transform = 2;
    } else {
      err = "config.ini: FromClassifiedDepth with losses[0] = " + (loss0.empty() ? std::string("(missing)") : loss0) +
            " applies no transform to the sampling net's output (pdf_transform 0), which is not supported; "
            "BCEWithLogitsLoss (sigmoid) and CrossEntropyLoss / CrossEntropyLossWeighted (softmax) are";
      return false;
    }
    out.sampler = 1;
  } else if (s.use_ndc) {
    if (!check("rayMarchSampler", "FromClassifiedDepthAdaptiveNoDepthRange") || !check("rayMarchNormalization", "None") ||
        !check("accumulationMult", "alpha")) {
      err = "config.ini: NDC exports must use FromClassifiedDepthAdaptiveNoDepthRange / rayMarchNormalization None / alpha";
      return false;
    }
  } else if (!check("rayMarchSampler", "FromClassifiedDepthAdaptive") || !check("rayMarchNormalization", "InverseSqrtDistCentered") ||
             !check("depthTransform", "log") || !check("accumulationMult", "alpha")) {
    err = "config.ini: only FromClassifiedDepthAdaptive / InverseSqrtDistCentered / log / alpha exports are supported";
    return false;
  }
  if (one_net) {
    if (!read_onnx_initializers(dir + "model0.onnx", out.nets[1], err)) return false;
  } else {
    for (int i = 0; i < 2; ++i)
      if (!read_onnx_initializers(dir + "model" + std::to_string(i) + ".onnx", out.nets[i], err)) return false;
  }
  // The networks' shapes come from the initialisers.  config.ini's layers / layerWidth (src/util/config.py:55-56), when
  // present, must describe the same networks: depth = the number of layers.{i} / pts_linears.{i} weights, width = the
  // input columns of layers.1 (the rows of layers.0 of a one-layer net) / of alpha_linear.
  for (int i = one_net ? 1 : 0; i < 2; ++i) {
    const std::string prefix = i == 0 ? "layers." : "pts_linears.";
    int depth = 0, width = 0, width0 = 0;
    for (const NamedTensor& t : out.nets[i]) {
      if (i == 1 && t.name == "alpha_linear.weight") width = int(t.cols);
      if (t.name.compare(0, prefix.size(), prefix) != 0 || t.name.size() < 7 || t.name.compare(t.name.size() - 7, 7, ".weight") != 0)
        continue;
      const int idx = std::atoi(t.name.c_str() + prefix.size());
      depth = std::max(depth, idx + 1);
      if (i == 0 && idx == 0) width0 = int(t.rows);
      if (i == 0 && idx == 1) width = int(t.cols);
    }
    if (i == 0 && depth == 1) width = width0;
    if (i == 0) {
      // multiDepthFeatures = [D, D] (src/features.py:250-252, nerf_raymarch_common.py:674-676): the depth cells the sampling
      // net classifies; a config without the key trained the reference's default, 128.  Raw / RawSigmoid size the sampling
      // net's output by the first entry and FromClassifiedDepthAdaptive places cells by the second, so they must agree
      // (and with model0.onnx: check_depth_cells).
      int cells = 128;
      auto md = cfg.find("multiDepthFeatures");
      if (md != cfg.end()) {
        const auto items = list_items(md->second);
        const bool two = items.size() == 2 && !items[0].empty() && items[0] == items[1] &&
                         items[0].find_first_not_of("0123456789") == std::string::npos;
        cells = two ? std::atoi(items[0].c_str()) : -1;
        if (cells != 32 && cells != 64 && cells != 128 && cells != 256) {
          err = "config.ini: multiDepthFeatures = " + strip(md->second) + ": need two equal entries, each 32, 64, 128 or 256";
          return false;
        }
      }
      out.depth_cells = cells;
    }
    const std::string onnx = one_net ? "model0.onnx" : "model" + std::to_string(i) + ".onnx";
    for (const auto& [key, have] : {std::pair<const char*, int>{"layers", depth}, {"layerWidth", width}}) {
      auto it = cfg.find(key);
      if (it == cfg.end()) continue;
      const auto items = list_items(it->second);
      if (items.size() != n_nets) continue;
      const int want = std::atoi(items[one_net ? 0 : size_t(i)].c_str());
      if (want != have) {
        err = "config.ini: " + std::string(key) + " = " + strip(it->second) + " but " + onnx + " holds a network with " + key + " " +
              std::to_string(have);
        return false;
      }
    }
  }
  return true;
}

bool check_depth_cells(const ExportDir& ex, std::string& err) {
  if (ex.sampler == 2) return true;   // a one-network export has no sampling net
  int depth = 0, rows = 0;
  for (const NamedTensor& t : ex.nets[0]) {
    if (t.name.compare(0, 7, "layers.") != 0 || t.name.size() < 7 || t.name.compare(t.name.size() - 7, 7, ".weight") != 0) continue;
    const int idx = std::atoi(t.name.c_str() + 7);
    if (idx + 1 > depth) {
      depth = idx + 1;
      rows = int(t.rows);
    }
  }
  if (rows == ex.depth_cells) return true;
  err = "config.ini: multiDepthFeatures gives " + std::to_string(ex.depth_cells) + " depth cells but model0.onnx's last layer has " +
        std::to_string(rows) + " outputs";
  return false;
}

}  // namespace adn
