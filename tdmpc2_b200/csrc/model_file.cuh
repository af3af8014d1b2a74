// Host side of the model file (tdmpc2_model_file_*, include/tdmpc2_b200.h): what `agent.export(fp)` writes
// (tdmpc2_b200/export.py), read without Python.  The layout is safetensors: an 8-byte little-endian header length, a JSON
// header {key: {"dtype", "shape", "data_offsets"}, "__metadata__": {string: string}}, then the raw little-endian data.
// `open` reads the whole file and checks everything a header can state against the dims in its metadata; `upload` lays
// the tensors out in one caller-owned device buffer and fills the pointer structs the planner and the pixel encoder read.
// Included by api.cu after its error helpers (fail, CUDA_TRY, align_up).
#pragma once
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

namespace mfile {

// ---- a JSON reader for what a safetensors header holds: objects, arrays, strings, integers (and the other literals)
struct JVal {
  enum Type { NUL, BOOL, NUM, STR, ARR, OBJ } type = NUL;
  std::string s;
  bool is_uint = false;           // a non-negative integer literal: u holds it exactly
  unsigned long long u = 0;
  std::vector<JVal> arr;
  std::vector<std::pair<std::string, JVal>> obj;
};

class Json {
 public:
  Json(const char* p, const char* end) : p_(p), end_(end) {}
  bool parse(JVal& v, std::string& err) {
    if (!value(v, 0)) { err = err_; return false; }
    ws();
    if (p_ != end_) { err = "trailing bytes after the JSON header"; return false; }
    return true;
  }

 private:
  const char* p_;
  const char* end_;
  std::string err_;
  bool bad(const char* what) { err_ = what; return false; }
  void ws() { while (p_ < end_ && (*p_ == ' ' || *p_ == '\t' || *p_ == '\n' || *p_ == '\r')) ++p_; }
  bool lit(const char* w) {
    const size_t n = strlen(w);
    if (static_cast<size_t>(end_ - p_) < n || memcmp(p_, w, n) != 0) return bad("malformed JSON header");
    p_ += n;
    return true;
  }
  bool str(std::string& s) {
    if (p_ >= end_ || *p_ != '"') return bad("malformed JSON header: a string was expected");
    ++p_;
    s.clear();
    while (p_ < end_ && *p_ != '"') {
      char c = *p_++;
      if (c == '\\') {
        if (p_ >= end_) break;
        c = *p_++;
        switch (c) {
          case '"': case '\\': case '/': s += c; break;
          case 'b': s += '\b'; break;
          case 'f': s += '\f'; break;
          case 'n': s += '\n'; break;
          case 'r': s += '\r'; break;
          case 't': s += '\t'; break;
          case 'u': {             // kept as UTF-8; the keys and values this format needs are ASCII
            if (end_ - p_ < 4) return bad("malformed JSON header: bad \\u escape");
            const unsigned cp = static_cast<unsigned>(strtoul(std::string(p_, 4).c_str(), nullptr, 16));
            p_ += 4;
            if (cp < 0x80) s += static_cast<char>(cp);
            else if (cp < 0x800) { s += static_cast<char>(0xC0 | (cp >> 6)); s += static_cast<char>(0x80 | (cp & 63)); }
            else { s += static_cast<char>(0xE0 | (cp >> 12)); s += static_cast<char>(0x80 | ((cp >> 6) & 63)); s += static_cast<char>(0x80 | (cp & 63)); }
            break;
          }
          default: return bad("malformed JSON header: bad escape");
        }
      } else {
        s += c;
      }
    }
    if (p_ >= end_) return bad("malformed JSON header: unterminated string");
    ++p_;
    return true;
  }
  bool value(JVal& v, int depth) {
    if (depth > 32) return bad("malformed JSON header: nested too deeply");
    ws();
    if (p_ >= end_) return bad("malformed JSON header: unexpected end");
    const char c = *p_;
    if (c == '{') {
      v.type = JVal::OBJ;
      ++p_; ws();
      if (p_ < end_ && *p_ == '}') { ++p_; return true; }
      for (;;) {
        ws();
        std::pair<std::string, JVal> kv;
        if (!str(kv.first)) return false;
        ws();
        if (p_ >= end_ || *p_ != ':') return bad("malformed JSON header: ':' expected");
        ++p_;
        if (!value(kv.second, depth + 1)) return false;
        v.obj.push_back(std::move(kv));
        ws();
        if (p_ < end_ && *p_ == ',') { ++p_; continue; }
        if (p_ < end_ && *p_ == '}') { ++p_; return true; }
        return bad("malformed JSON header: ',' or '}' expected");
      }
    }
    if (c == '[') {
      v.type = JVal::ARR;
      ++p_; ws();
      if (p_ < end_ && *p_ == ']') { ++p_; return true; }
      for (;;) {
        JVal e;
        if (!value(e, depth + 1)) return false;
        v.arr.push_back(std::move(e));
        ws();
        if (p_ < end_ && *p_ == ',') { ++p_; continue; }
        if (p_ < end_ && *p_ == ']') { ++p_; return true; }
        return bad("malformed JSON header: ',' or ']' expected");
      }
    }
    if (c == '"') { v.type = JVal::STR; return str(v.s); }
    if (c == 't') { v.type = JVal::BOOL; return lit("true"); }
    if (c == 'f') { v.type = JVal::BOOL; return lit("false"); }
    if (c == 'n') { v.type = JVal::NUL; return lit("null"); }
    if (c == '-' || (c >= '0' && c <= '9')) {
      const char* b = p_;
      while (p_ < end_ && (strchr("+-.eE", *p_) || (*p_ >= '0' && *p_ <= '9'))) ++p_;
      v.type = JVal::NUM;
      v.s.assign(b, p_);
      v.is_uint = v.s.find_first_not_of("0123456789") == std::string::npos && v.s.size() <= 19;
      if (v.is_uint) v.u = strtoull(v.s.c_str(), nullptr, 10);
      return true;
    }
    return bad("malformed JSON header: unexpected character");
  }
};

struct Tensor {
  std::string dtype;
  std::vector<long long> shape;
  unsigned long long begin = 0, end = 0;     // byte range within the data section
};

// The tensors a model with these dims needs, in upload order, with their shapes (the reference's state-dict keys, then
// the derived tdmpc2.* tensors).  tdmpc2.discount is F64 and stays on the host.
using Shape = std::vector<long long>;
inline void expected_tensors(const tdmpc2_dims& d, bool pixel, const tdmpc2_pixel_dims& px,
                             std::vector<std::pair<std::string, Shape>>& out) {
  const long long L = d.latent_dim, M = d.mlp_dim, A = d.action_dim, T = d.task_dim, B = d.num_bins, nq = d.num_q;
  const long long D = L + T + A;
  auto lin = [&](const std::string& pfx, const Shape& lead, long long in, long long o, bool ln) {
    Shape w = lead, b = lead;
    w.push_back(o); w.push_back(in); b.push_back(o);
    out.emplace_back(pfx + ".weight", w);
    out.emplace_back(pfx + ".bias", b);
    if (ln) { out.emplace_back(pfx + ".ln.weight", b); out.emplace_back(pfx + ".ln.bias", b); }
  };
  auto mlp = [&](const std::string& pfx, const Shape& lead, long long in, long long o, bool ln_last) {
    lin(pfx + ".0", lead, in, M, true);
    lin(pfx + ".1", lead, M, M, true);
    lin(pfx + ".2", lead, M, o, ln_last);
  };
  if (pixel) {
    const long long C = px.in_channels, nc = px.num_channels;
    const long long cin[4] = {C, nc, nc, nc}, k[4] = {7, 5, 3, 3};
    for (int i = 0; i < 4; ++i) {
      const std::string pfx = "_encoder.rgb." + std::to_string(2 * i + 2);
      out.emplace_back(pfx + ".weight", Shape{nc, cin[i], k[i], k[i]});
      out.emplace_back(pfx + ".bias", Shape{nc});
    }
  } else {
    const int n_hidden = d.num_enc_layers - 1 > 1 ? d.num_enc_layers - 1 : 1;   // layers.py:157
    long long in = d.obs_dim + T;
    for (int i = 0; i <= n_hidden; ++i) {
      const long long o = i < n_hidden ? d.enc_dim : L;
      lin("_encoder.state." + std::to_string(i), {}, in, o, true);
      in = o;
    }
  }
  mlp("_dynamics", {}, D, L, true);
  mlp("_reward", {}, D, B, false);
  mlp("_pi", {}, L + T, 2 * A, false);
  mlp("_Qs.params", {nq}, D, B, false);
  if (d.episodic) mlp("_termination", {}, L + T, 1, false);
  if (T > 0) {
    out.emplace_back("_task_emb.weight", Shape{d.num_tasks, T});
    out.emplace_back("_action_masks", Shape{d.num_tasks, A});
  }
  out.emplace_back("tdmpc2.bins", Shape{B});
  if (pixel) out.emplace_back("tdmpc2.grid_base", Shape{64});
  out.emplace_back("tdmpc2.discount", Shape{d.num_tasks});
}

inline std::string shape_str(const Shape& s) {
  std::string o = "[";
  for (size_t i = 0; i < s.size(); ++i) o += (i ? ", " : "") + std::to_string(s[i]);
  return o + "]";
}

}  // namespace mfile

struct tdmpc2_model_file {
  std::vector<unsigned char> bytes;      // the whole file
  size_t data0 = 0;                      // first byte of the data section
  std::map<std::string, mfile::Tensor> tensors;
  tdmpc2_dims dims{};
  tdmpc2_pixel_dims pix{};
  int32_t is_pixel = 0;
  const unsigned char* data(const std::string& k) const { return bytes.data() + data0 + tensors.at(k).begin; }
};

// The dims fields, in tdmpc2_dims order, under the names the metadata uses
static const char* const kMfIntFields[] = {"num_envs", "num_samples", "num_pi_trajs", "num_elites", "horizon", "iterations",
                                           "obs_dim", "action_dim", "latent_dim", "mlp_dim", "enc_dim", "num_enc_layers",
                                           "task_dim", "num_tasks", "num_q", "num_bins", "simnorm_dim", "episodic"};
static const char* const kMfFloatFields[] = {"temperature", "min_std", "max_std", "log_std_min", "log_std_dif"};

static int mf_parse(tdmpc2_model_file* f, const char* path) {
  using namespace mfile;
  const std::vector<unsigned char>& b = f->bytes;
  if (b.size() < 8)
    return fail(TDMPC2_ERR_INVALID, "%s: truncated file: %zu bytes, less than the 8-byte header length", path, b.size());
  unsigned long long hlen = 0;
  for (int i = 7; i >= 0; --i) hlen = (hlen << 8) | b[i];
  if (hlen > b.size() - 8)
    return fail(TDMPC2_ERR_INVALID, "%s: header length %llu runs past the end of the file (%zu bytes)", path, hlen, b.size());
  f->data0 = 8 + static_cast<size_t>(hlen);
  const unsigned long long data_bytes = b.size() - f->data0;
  JVal root;
  std::string err;
  if (!Json(reinterpret_cast<const char*>(b.data() + 8), reinterpret_cast<const char*>(b.data() + f->data0)).parse(root, err))
    return fail(TDMPC2_ERR_INVALID, "%s: %s", path, err.c_str());
  if (root.type != JVal::OBJ) return fail(TDMPC2_ERR_INVALID, "%s: the JSON header is not an object", path);

  // ---- metadata: format, version, dims
  std::map<std::string, std::string> meta;
  for (auto& kv : root.obj) {
    if (kv.first != "__metadata__") continue;
    if (kv.second.type != JVal::OBJ) return fail(TDMPC2_ERR_INVALID, "%s: __metadata__ is not an object", path);
    for (auto& m : kv.second.obj) {
      if (m.second.type != JVal::STR) return fail(TDMPC2_ERR_INVALID, "%s: __metadata__ value '%s' is not a string", path, m.first.c_str());
      meta[m.first] = m.second.s;
    }
  }
  auto field = [&](const char* k) -> const std::string* { auto it = meta.find(k); return it == meta.end() ? nullptr : &it->second; };
  const std::string* fmt = field("format");
  if (!fmt || *fmt != "tdmpc2_b200.model")
    return fail(TDMPC2_ERR_INVALID, "%s: not a tdmpc2_b200 model file: __metadata__ format is '%s', expected 'tdmpc2_b200.model'", path,
                fmt ? fmt->c_str() : "(missing)");
  const std::string* ver = field("version");
  if (!ver || *ver != "1")
    return fail(TDMPC2_ERR_INVALID, "%s: model file version '%s' is not supported: this library reads version 1", path,
                ver ? ver->c_str() : "(missing)");
  const std::string* obs = field("obs");
  if (!obs || (*obs != "state" && *obs != "rgb"))
    return fail(TDMPC2_ERR_INVALID, "%s: __metadata__ obs is '%s', expected 'state' or 'rgb'", path, obs ? obs->c_str() : "(missing)");
  f->is_pixel = *obs == "rgb";
  auto get_int = [&](const char* k, int32_t* out) -> int {
    const std::string* v = field(k);
    if (!v) return fail(TDMPC2_ERR_INVALID, "%s: missing __metadata__ field '%s'", path, k);
    char* e = nullptr;
    errno = 0;
    const long x = strtol(v->c_str(), &e, 10);
    if (v->empty() || *e || errno || x < -0x7fffffffL || x > 0x7fffffffL)
      return fail(TDMPC2_ERR_INVALID, "%s: __metadata__ field '%s' = '%s' is not an int32", path, k, v->c_str());
    *out = static_cast<int32_t>(x);
    return 0;
  };
  auto get_float = [&](const char* k, float* out) -> int {
    const std::string* v = field(k);
    if (!v) return fail(TDMPC2_ERR_INVALID, "%s: missing __metadata__ field '%s'", path, k);
    char* e = nullptr;
    const double x = strtod(v->c_str(), &e);
    if (v->empty() || *e) return fail(TDMPC2_ERR_INVALID, "%s: __metadata__ field '%s' = '%s' is not a number", path, k, v->c_str());
    *out = static_cast<float>(x);
    return 0;
  };
  int32_t* ints = &f->dims.num_envs;        // tdmpc2_dims: 18 int32 fields, then 5 floats
  float* floats = &f->dims.temperature;
  int rc;
  for (int i = 0; i < 18; ++i) if ((rc = get_int(kMfIntFields[i], ints + i))) return rc;
  for (int i = 0; i < 5; ++i) if ((rc = get_float(kMfFloatFields[i], floats + i))) return rc;
  if (f->is_pixel) {
    if ((rc = get_int("pixel.in_channels", &f->pix.in_channels)) || (rc = get_int("pixel.num_channels", &f->pix.num_channels)) ||
        (rc = get_int("pixel.simnorm_dim", &f->pix.simnorm_dim)))
      return rc;
  }
  const tdmpc2_dims& d = f->dims;
  if (d.latent_dim < 1 || d.mlp_dim < 1 || d.action_dim < 1 || d.obs_dim < 1 || d.enc_dim < 1 || d.num_q < 1 || d.num_bins < 1 ||
      d.task_dim < 0 || d.num_tasks < 1 || d.num_enc_layers < 0 || d.num_enc_layers > 64 || (d.episodic != 0 && d.episodic != 1) ||
      (f->is_pixel && (d.num_enc_layers != 0 || f->pix.in_channels < 1 || f->pix.num_channels < 1)) ||
      (!f->is_pixel && d.num_enc_layers < 1))
    return fail(TDMPC2_ERR_INVALID, "%s: the dims in __metadata__ do not describe a model", path);

  // ---- tensor entries: dtype, offsets inside the data section, no overlap, size = dtype x shape
  for (auto& kv : root.obj) {
    if (kv.first == "__metadata__") continue;
    const char* k = kv.first.c_str();
    if (kv.second.type != JVal::OBJ) return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': entry is not an object", path, k);
    Tensor t;
    const JVal *dt = nullptr, *sh = nullptr, *off = nullptr;
    for (auto& e : kv.second.obj) {
      if (e.first == "dtype") dt = &e.second;
      else if (e.first == "shape") sh = &e.second;
      else if (e.first == "data_offsets") off = &e.second;
    }
    if (!dt || dt->type != JVal::STR || !sh || sh->type != JVal::ARR || !off || off->type != JVal::ARR || off->arr.size() != 2 ||
        !off->arr[0].is_uint || !off->arr[1].is_uint)
      return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': entry needs dtype, shape and two data_offsets", path, k);
    t.dtype = dt->s;
    const std::string want = kv.first == "tdmpc2.discount" ? "F64" : "F32";
    if (t.dtype != want)
      return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': dtype %s, expected %s", path, k, t.dtype.c_str(), want.c_str());
    unsigned long long numel = 1;
    for (auto& s : sh->arr) {
      if (!s.is_uint || s.u > (1ull << 40)) return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': bad shape", path, k);
      t.shape.push_back(static_cast<long long>(s.u));
      numel *= s.u;
      if (numel > (1ull << 40)) return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': bad shape", path, k);
    }
    t.begin = off->arr[0].u;
    t.end = off->arr[1].u;
    if (t.begin > t.end || t.end > data_bytes)
      return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': data_offsets [%llu, %llu] out of range: the data section holds %llu bytes "
                  "(truncated file?)", path, k, t.begin, t.end, data_bytes);
    const unsigned long long need = numel * (t.dtype == "F64" ? 8 : 4);
    if (t.end - t.begin != need)
      return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s': data_offsets span %llu bytes, its dtype and shape need %llu", path, k,
                  t.end - t.begin, need);
    if (!f->tensors.emplace(kv.first, t).second) return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s' appears twice", path, k);
  }
  std::vector<std::pair<unsigned long long, const std::string*>> order;
  for (auto& kv : f->tensors) order.emplace_back(kv.second.begin, &kv.first);
  std::sort(order.begin(), order.end());
  for (size_t i = 1; i < order.size(); ++i) {
    const Tensor& prev = f->tensors[*order[i - 1].second];
    if (order[i].first < prev.end)
      return fail(TDMPC2_ERR_INVALID, "%s: tensors '%s' and '%s' overlap in the data section", path, order[i - 1].second->c_str(),
                  order[i].second->c_str());
  }

  // ---- every tensor the dims need, with the shape they need
  std::vector<std::pair<std::string, Shape>> want;
  expected_tensors(d, f->is_pixel != 0, f->pix, want);
  for (auto& w : want) {
    auto it = f->tensors.find(w.first);
    if (it == f->tensors.end()) return fail(TDMPC2_ERR_INVALID, "%s: missing tensor '%s'", path, w.first.c_str());
    if (it->second.shape != w.second)
      return fail(TDMPC2_ERR_INVALID, "%s: tensor '%s' has shape %s, the dims need %s", path, w.first.c_str(),
                  shape_str(it->second.shape).c_str(), shape_str(w.second).c_str());
  }
  return 0;
}

extern "C" int tdmpc2_model_file_open(const char* path, tdmpc2_model_file** out) {
  if (!path || !out) return fail(TDMPC2_ERR_INVALID, "null argument");
  *out = nullptr;
  FILE* fp = fopen(path, "rb");
  if (!fp) return fail(TDMPC2_ERR_INVALID, "%s: cannot open: %s", path, strerror(errno));
  tdmpc2_model_file* f = new tdmpc2_model_file();
  unsigned char buf[1 << 16];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, fp)) > 0) f->bytes.insert(f->bytes.end(), buf, buf + n);
  const bool read_error = ferror(fp) != 0;
  fclose(fp);
  if (read_error) { delete f; return fail(TDMPC2_ERR_INVALID, "%s: read error", path); }
  const int rc = mf_parse(f, path);
  if (rc) { delete f; return rc; }
  *out = f;
  return 0;
}

extern "C" void tdmpc2_model_file_close(tdmpc2_model_file* f) { delete f; }

extern "C" int tdmpc2_model_file_dims(const tdmpc2_model_file* f, tdmpc2_dims* dims, tdmpc2_pixel_dims* pixel, int32_t* is_pixel) {
  if (!f || !dims) return fail(TDMPC2_ERR_INVALID, "null argument");
  *dims = f->dims;
  if (pixel) *pixel = f->pix;
  if (is_pixel) *is_pixel = f->is_pixel;
  return 0;
}

// dims may differ from the file's in num_envs and the planning block; every field that shapes the model must agree
static int mf_check_dims(const tdmpc2_model_file* f, const tdmpc2_dims* d) {
  if (!f || !d) return fail(TDMPC2_ERR_INVALID, "null argument");
  const tdmpc2_dims& m = f->dims;
  const int32_t* a = &m.obs_dim;            // obs_dim .. episodic: the model-shape int32 fields
  const int32_t* b = &d->obs_dim;
  for (int i = 0; i < 12; ++i)
    if (a[i] != b[i]) return fail(TDMPC2_ERR_INVALID, "dims.%s = %d, the model file has %d", kMfIntFields[6 + i], b[i], a[i]);
  if (m.log_std_min != d->log_std_min || m.log_std_dif != d->log_std_dif)
    return fail(TDMPC2_ERR_INVALID, "dims.log_std_min / log_std_dif differ from the model file's");
  if (d->horizon < 1) return fail(TDMPC2_ERR_INVALID, "dims.horizon must be >= 1");
  return 0;
}

// The device layout: every tensor but tdmpc2.discount, then discount_pow [num_tasks, H + 1], each 256-byte aligned.
static size_t mf_layout(const tdmpc2_model_file* f, const tdmpc2_dims& d, std::map<std::string, size_t>* offs) {
  std::vector<std::pair<std::string, mfile::Shape>> want;
  mfile::expected_tensors(f->dims, f->is_pixel != 0, f->pix, want);
  size_t off = 0;
  for (auto& w : want) {
    if (w.first == "tdmpc2.discount") continue;
    const mfile::Tensor& t = f->tensors.at(w.first);
    if (offs) (*offs)[w.first] = off;
    off = align_up(off + (t.end - t.begin), 256);
  }
  if (offs) (*offs)["discount_pow"] = off;
  return align_up(off + static_cast<size_t>(d.num_tasks) * (d.horizon + 1) * 4, 256);
}

extern "C" int tdmpc2_model_file_device_bytes(const tdmpc2_model_file* f, const tdmpc2_dims* dims, size_t* out) {
  if (!out) return fail(TDMPC2_ERR_INVALID, "null argument");
  const int rc = mf_check_dims(f, dims);
  if (rc) return rc;
  *out = mf_layout(f, *dims, nullptr);
  return 0;
}

extern "C" int tdmpc2_model_file_upload(const tdmpc2_model_file* f, const tdmpc2_dims* dims, void* device_buf, tdmpc2_weights* w,
                                        tdmpc2_conv_weights* conv, const float** grid_base, void* stream_) {
  int rc = mf_check_dims(f, dims);
  if (rc) return rc;
  if (!device_buf || !w) return fail(TDMPC2_ERR_INVALID, "null argument");
  if (reinterpret_cast<uintptr_t>(device_buf) & 255) return fail(TDMPC2_ERR_INVALID, "device_buf must be 256-byte aligned");
  if (f->is_pixel && (!conv || !grid_base)) return fail(TDMPC2_ERR_INVALID, "a pixel model needs conv and grid_base");
  std::map<std::string, size_t> offs;
  const size_t bytes = mf_layout(f, *dims, &offs);
  std::vector<unsigned char> stage(bytes, 0);
  for (auto& o : offs) {
    if (o.first == "discount_pow") continue;
    const mfile::Tensor& t = f->tensors.at(o.first);
    memcpy(stage.data() + o.second, f->data(o.first), t.end - t.begin);
  }
  // discount_pow: planner.py's discount_table, bit for bit.  Single-task: a double running product cast to fp32 per step;
  // multi-task: fp32 products of the fp32-cast discounts.
  const tdmpc2_dims& d = *dims;
  const unsigned char* gsrc = f->data("tdmpc2.discount");
  float* pow_out = reinterpret_cast<float*>(stage.data() + offs["discount_pow"]);
  for (int k = 0; k < d.num_tasks; ++k) {
    double g;
    memcpy(&g, gsrc + 8 * k, 8);
    float* row = pow_out + static_cast<size_t>(k) * (d.horizon + 1);
    row[0] = 1.0f;
    if (d.task_dim > 0) {
      const float gf = static_cast<float>(g);
      float p = 1.0f;
      for (int t = 1; t <= d.horizon; ++t) { p = p * gf; row[t] = p; }
    } else {
      double p = 1.0;
      for (int t = 1; t <= d.horizon; ++t) { p = p * g; row[t] = static_cast<float>(p); }
    }
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  CUDA_TRY(cudaMemcpyAsync(device_buf, stage.data(), bytes, cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  unsigned char* base = static_cast<unsigned char*>(device_buf);
  auto ptr = [&](const std::string& k) -> const float* {
    auto it = offs.find(k);
    return it == offs.end() ? nullptr : reinterpret_cast<const float*>(base + it->second);
  };
  auto lin = [&](const std::string& pfx) {
    tdmpc2_linear l;
    l.weight = ptr(pfx + ".weight"); l.bias = ptr(pfx + ".bias");
    l.ln_weight = ptr(pfx + ".ln.weight"); l.ln_bias = ptr(pfx + ".ln.bias");
    return l;
  };
  memset(w, 0, sizeof *w);
  for (int i = 0; i < TDMPC2_MAX_ENC_LAYERS && offs.count("_encoder.state." + std::to_string(i) + ".weight"); ++i) {
    w->enc[i] = lin("_encoder.state." + std::to_string(i));
    w->num_enc = i + 1;
  }
  for (int i = 0; i < 3; ++i) {
    const std::string s = "." + std::to_string(i);
    w->dynamics[i] = lin("_dynamics" + s);
    w->reward[i] = lin("_reward" + s);
    w->pi[i] = lin("_pi" + s);
    w->qs[i] = lin("_Qs.params" + s);
    if (d.episodic) w->termination[i] = lin("_termination" + s);
  }
  w->task_emb = ptr("_task_emb.weight");
  w->action_masks = ptr("_action_masks");
  w->bins = ptr("tdmpc2.bins");
  w->discount_pow = ptr("discount_pow");
  if (f->is_pixel) {
    for (int i = 0; i < 4; ++i) {
      const std::string pfx = "_encoder.rgb." + std::to_string(2 * i + 2);
      conv->weight[i] = ptr(pfx + ".weight");
      conv->bias[i] = ptr(pfx + ".bias");
    }
    *grid_base = ptr("tdmpc2.grid_base");
  } else {
    if (conv) memset(conv, 0, sizeof *conv);
    if (grid_base) *grid_base = nullptr;
  }
  return 0;
}
