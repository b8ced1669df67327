// caffe_proto_io.cpp -- see caffe_proto_io.hpp.
#include "caffe_proto_io.hpp"

#include "hdf5_io.hpp"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

namespace cosb {
namespace {

// ------------------------------------------------------------------ encoder
enum WireType : uint32_t { kVarint = 0, kFixed64 = 1, kLen = 2, kFixed32 = 5 };

size_t varint_size(uint64_t v) {
  size_t n = 1;
  while (v >= 0x80) {
    v >>= 7;
    ++n;
  }
  return n;
}

void put_varint(std::string* s, uint64_t v) {
  while (v >= 0x80) {
    s->push_back(static_cast<char>((v & 0x7f) | 0x80));
    v >>= 7;
  }
  s->push_back(static_cast<char>(v));
}

void put_tag(std::string* s, uint32_t field, WireType wt) { put_varint(s, (static_cast<uint64_t>(field) << 3) | wt); }

void put_string(std::string* s, uint32_t field, const std::string& v) {
  put_tag(s, field, kLen);
  put_varint(s, v.size());
  s->append(v);
}

// BlobProto header = everything except the raw float payload:
//   shape (field 7) + tag/len of the packed data field (5)
std::string blob_header(const BlobView& b) {
  std::string dims;
  for (int64_t d : b.shape) put_varint(&dims, static_cast<uint64_t>(d));
  std::string shape;  // BlobShape { dim = 1 packed }
  put_tag(&shape, 1, kLen);
  put_varint(&shape, dims.size());
  shape += dims;
  std::string h;
  put_tag(&h, 7, kLen);
  put_varint(&h, shape.size());
  h += shape;
  put_tag(&h, 5, kLen);
  put_varint(&h, b.count * sizeof(float));
  return h;
}

uint64_t blob_size(const BlobView& b) { return blob_header(b).size() + b.count * sizeof(float); }

bool write_all(FILE* f, const void* p, size_t n) { return n == 0 || fwrite(p, 1, n, f) == n; }

bool write_blob(FILE* f, uint32_t field, const BlobView& b) {  // as a length-delimited sub-message
  std::string pre;
  put_tag(&pre, field, kLen);
  put_varint(&pre, blob_size(b));
  pre += blob_header(b);
  return write_all(f, pre.data(), pre.size()) && write_all(f, b.data, b.count * sizeof(float));  // little-endian host
}

bool check_views(const std::vector<BlobView>& blobs, std::string* err) {
  for (const BlobView& b : blobs) {
    uint64_t n = 1;
    for (int64_t d : b.shape) n *= static_cast<uint64_t>(d);
    if (b.shape.empty()) n = b.count;
    if (n != b.count || (b.count && !b.data)) {
      *err = "blob '" + b.layer_name + "': shape does not match its element count";
      return false;
    }
  }
  return true;
}

// ------------------------------------------------------------------ decoder
struct Reader {
  const unsigned char* p;
  const unsigned char* end;
  bool ok = true;
  uint64_t varint() {
    uint64_t v = 0;
    int shift = 0;
    while (p < end && shift < 64) {
      unsigned char c = *p++;
      v |= static_cast<uint64_t>(c & 0x7f) << shift;
      if (!(c & 0x80)) return v;
      shift += 7;
    }
    ok = false;
    return 0;
  }
  bool next(uint32_t* field, uint32_t* wt) {
    if (p >= end || !ok) return false;
    uint64_t t = varint();
    *field = static_cast<uint32_t>(t >> 3);
    *wt = static_cast<uint32_t>(t & 7);
    return ok;
  }
  Reader sub() {  // length-delimited payload
    uint64_t n = varint();
    Reader r{p, p, ok};
    if (!ok || n > static_cast<uint64_t>(end - p)) {
      ok = false;
      r.ok = false;
      return r;
    }
    r.end = p + n;
    p += n;
    return r;
  }
  void skip(uint32_t wt) {
    switch (wt) {
      case kVarint: varint(); break;
      case kFixed64: if (end - p >= 8) p += 8; else ok = false; break;
      case kLen: sub(); break;
      case kFixed32: if (end - p >= 4) p += 4; else ok = false; break;
      default: ok = false;
    }
  }
};

bool parse_blob(Reader r, ParsedBlob* out) {
  int64_t legacy[4] = {0, 0, 0, 0};
  bool has_legacy = false;
  uint32_t f, wt;
  while (r.next(&f, &wt)) {
    if (f == 7 && wt == kLen) {  // BlobShape
      Reader s = r.sub();
      uint32_t f2, wt2;
      while (s.next(&f2, &wt2)) {
        if (f2 == 1 && wt2 == kLen) {
          Reader d = s.sub();
          while (d.p < d.end && d.ok) out->shape.push_back(static_cast<int64_t>(d.varint()));
          if (!d.ok) return false;
        } else if (f2 == 1 && wt2 == kVarint) {
          out->shape.push_back(static_cast<int64_t>(s.varint()));
        } else {
          s.skip(wt2);
        }
      }
      if (!s.ok) return false;
    } else if (f == 5 && wt == kLen) {  // packed float data
      Reader d = r.sub();
      if (!d.ok || (d.end - d.p) % 4) return false;
      size_t n = static_cast<size_t>(d.end - d.p) / 4;
      size_t old = out->data.size();
      out->data.resize(old + n);
      memcpy(out->data.data() + old, d.p, n * 4);
    } else if (f == 5 && wt == kFixed32) {  // un-packed float
      if (r.end - r.p < 4) return false;
      float v;
      memcpy(&v, r.p, 4);
      r.p += 4;
      out->data.push_back(v);
    } else if (f >= 1 && f <= 4 && wt == kVarint) {  // legacy num/channels/height/width
      legacy[f - 1] = static_cast<int64_t>(r.varint());
      has_legacy = true;
    } else {
      r.skip(wt);
    }
  }
  if (!r.ok) return false;
  if (out->shape.empty() && has_legacy) out->shape.assign(legacy, legacy + 4);
  return true;
}

bool slurp(const std::string& path, std::vector<unsigned char>* buf, std::string* err) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) {
    *err = "cannot open '" + path + "'";
    return false;
  }
  fseek(f, 0, SEEK_END);
  long n = ftell(f);
  fseek(f, 0, SEEK_SET);
  buf->resize(n > 0 ? static_cast<size_t>(n) : 0);
  bool ok = n >= 0 && (n == 0 || fread(buf->data(), 1, buf->size(), f) == buf->size());
  fclose(f);
  if (!ok) *err = "cannot read '" + path + "'";
  return ok;
}

}  // namespace

bool write_caffemodel(const std::string& path, const std::string& net_name, const std::vector<BlobView>& blobs,
                      std::string* err) {
  if (!check_views(blobs, err)) return false;
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) {
    *err = "cannot open '" + path + "' for writing";
    return false;
  }
  bool ok = true;
  std::string head;
  put_string(&head, 1, net_name);  // NetParameter.name
  ok = write_all(f, head.data(), head.size());
  for (size_t i = 0; ok && i < blobs.size();) {
    size_t j = i;
    while (j < blobs.size() && blobs[j].layer_name == blobs[i].layer_name) ++j;
    // LayerParameter { name = 1, type = 2, blobs = 7... }
    std::string lp;
    put_string(&lp, 1, blobs[i].layer_name);
    put_string(&lp, 2, blobs[i].layer_type);
    uint64_t body = lp.size();
    for (size_t k = i; k < j; ++k) {
      uint64_t bs = blob_size(blobs[k]);
      body += 1 + varint_size(bs) + bs;  // tag of field 7 is one byte
    }
    std::string pre;
    put_tag(&pre, 100, kLen);  // NetParameter.layer
    put_varint(&pre, body);
    pre += lp;
    ok = write_all(f, pre.data(), pre.size());
    for (size_t k = i; ok && k < j; ++k) ok = write_blob(f, 7, blobs[k]);
    i = j;
  }
  ok = (fclose(f) == 0) && ok;
  if (!ok) *err = "short write to '" + path + "'";
  return ok;
}

namespace {
bool blob_from_h5(const H5Node& d, const std::string& path, ParsedBlob* b, std::string* err) {
  if (d.kind != H5Node::kFloat32) {
    *err = "'" + path + "': dataset '" + d.name + "' is not float32";
    return false;
  }
  b->shape = d.shape;
  b->data = d.f32;
  return true;
}
// datasets "0", "1", ... of a group, in numeric order (the B-tree returns them in strcmp order: "0","1","10","2").
// With gaps (a model's layer group), an index below the largest without a dataset is a blob marked absent:
// Net::ToHDF5 skips a param a layer shares.  Without (the solverstate's history), every index must be there.
bool numbered_blobs(const H5Node& g, const std::string& path, bool gaps, std::vector<ParsedBlob>* out,
                    std::string* err) {
  size_t n = g.children.size();
  if (gaps) {
    n = 0;
    for (const auto& c : g.children) {
      const bool index = !c->name.empty() && c->name.size() < 10 &&
                         c->name.find_first_not_of("0123456789") == std::string::npos;
      if (!index) {
        *err = "'" + path + "': group '" + g.name + "' has dataset '" + c->name + "', which is not a blob index";
        return false;
      }
      n = std::max(n, static_cast<size_t>(atol(c->name.c_str())) + 1);
    }
  }
  for (size_t j = 0; j < n; ++j) {
    ParsedBlob b;
    const H5Node* d = g.find(std::to_string(j));
    if (!d && !gaps) {
      *err = "'" + path + "': group '" + g.name + "' has no dataset '" + std::to_string(j) + "'";
      return false;
    }
    if (!d) b.present = false;
    else if (!blob_from_h5(*d, path, &b, err)) return false;
    out->push_back(std::move(b));
  }
  return true;
}
}  // namespace

bool read_caffemodel(const std::string& path, std::string* net_name, std::vector<ParsedLayer>* layers,
                     std::string* err) {
  if (h5_is_hdf5(path)) {  // Net::CopyTrainedLayersFromHDF5 (net.cpp:805-851): group "data", one subgroup per layer
    H5Node root;
    if (!h5_read(path, &root, err)) return false;
    const H5Node* data = root.find("data");
    if (!data || data->kind != H5Node::kGroup) {
      *err = "'" + path + "' has no 'data' group: not a Caffe HDF5 model";
      return false;
    }
    if (net_name) net_name->clear();
    for (const auto& L : data->children) {
      if (L->kind != H5Node::kGroup) continue;
      ParsedLayer pl;
      pl.name = L->name;
      if (!numbered_blobs(*L, path, true, &pl.blobs, err)) return false;
      layers->push_back(std::move(pl));
    }
    return true;
  }
  std::vector<unsigned char> buf;
  if (!slurp(path, &buf, err)) return false;
  Reader r{buf.data(), buf.data() + buf.size(), true};
  uint32_t f, wt;
  bool saw_v1 = false;
  while (r.next(&f, &wt)) {
    if (f == 1 && wt == kLen) {
      Reader s = r.sub();
      if (net_name) net_name->assign(reinterpret_cast<const char*>(s.p), s.end - s.p);
    } else if (f == 100 && wt == kLen) {
      Reader lr = r.sub();
      ParsedLayer L;
      uint32_t f2, wt2;
      while (lr.next(&f2, &wt2)) {
        if ((f2 == 1 || f2 == 2) && wt2 == kLen) {
          Reader s = lr.sub();
          (f2 == 1 ? L.name : L.type).assign(reinterpret_cast<const char*>(s.p), s.end - s.p);
        } else if (f2 == 7 && wt2 == kLen) {
          ParsedBlob b;
          if (!parse_blob(lr.sub(), &b)) {
            *err = "'" + path + "': malformed BlobProto in layer '" + L.name + "'";
            return false;
          }
          L.blobs.push_back(std::move(b));
        } else {
          lr.skip(wt2);
        }
      }
      if (!lr.ok) {  // a truncated / malformed LayerParameter must not yield a silently partial layer list
        *err = "'" + path + "': malformed LayerParameter" + (L.name.empty() ? std::string() : " '" + L.name + "'");
        return false;
      }
      layers->push_back(std::move(L));
    } else {
      if (f == 2 && wt == kLen) saw_v1 = true;  // V1LayerParameter layers
      r.skip(wt);
    }
  }
  if (!r.ok) {
    *err = "'" + path + "' is not a NetParameter binaryproto";
    return false;
  }
  if (layers->empty() && saw_v1) {
    *err = "'" + path + "' uses V1 'layers' (pre-2015 Caffe); upgrade it with upgrade_net_proto_binary";
    return false;
  }
  return true;
}

bool write_solverstate(const std::string& path, int iter, int current_step, const std::string& learned_net,
                       const std::vector<BlobView>& history, std::string* err) {
  if (!check_views(history, err)) return false;
  FILE* f = fopen(path.c_str(), "wb");
  if (!f) {
    *err = "cannot open '" + path + "' for writing";
    return false;
  }
  std::string head;
  put_tag(&head, 1, kVarint);
  put_varint(&head, static_cast<uint64_t>(static_cast<int64_t>(iter)));
  put_string(&head, 2, learned_net);
  bool ok = write_all(f, head.data(), head.size());
  for (size_t i = 0; ok && i < history.size(); ++i) ok = write_blob(f, 3, history[i]);
  std::string tail;
  put_tag(&tail, 4, kVarint);
  put_varint(&tail, static_cast<uint64_t>(static_cast<int64_t>(current_step)));
  ok = ok && write_all(f, tail.data(), tail.size());
  ok = (fclose(f) == 0) && ok;
  if (!ok) *err = "short write to '" + path + "'";
  return ok;
}

bool write_caffemodel_h5(const std::string& path, const std::vector<BlobView>& blobs, std::string* err) {
  if (!check_views(blobs, err)) return false;
  H5Node root;
  H5Node* data = root.add_group("data");
  H5Node* layer = nullptr;
  int j = 0;
  for (size_t i = 0; i < blobs.size(); ++i) {  // consecutive views with one layer_name = that layer's blobs 0, 1, ...
    if (i == 0 || blobs[i].layer_name != blobs[i - 1].layer_name) {
      layer = data->add_group(blobs[i].layer_name);
      j = 0;
    }
    std::vector<int64_t> shape = blobs[i].shape;
    if (shape.empty()) shape.assign(1, static_cast<int64_t>(blobs[i].count));
    const int name = blobs[i].param_index >= 0 ? blobs[i].param_index : j;
    ++j;
    layer->add_float(std::to_string(name), shape, blobs[i].data, blobs[i].count);
  }
  return h5_write(path, root, err);
}

bool write_solverstate_h5(const std::string& path, int iter, int current_step, const std::string& learned_net,
                          const std::vector<BlobView>& history, std::string* err) {
  if (!check_views(history, err)) return false;
  H5Node root;  // sgd_solver.cpp:288-299
  root.add_int("iter", iter);
  root.add_string("learned_net", learned_net);
  root.add_int("current_step", current_step);
  H5Node* h = root.add_group("history");
  for (size_t i = 0; i < history.size(); ++i) {
    std::vector<int64_t> shape = history[i].shape;
    if (shape.empty()) shape.assign(1, static_cast<int64_t>(history[i].count));
    h->add_float(std::to_string(i), shape, history[i].data, history[i].count);
  }
  return h5_write(path, root, err);
}

bool read_solverstate(const std::string& path, int* iter, int* current_step, std::string* learned_net,
                      std::vector<ParsedBlob>* history, std::string* err) {
  if (h5_is_hdf5(path)) {  // SGDSolver::RestoreSolverStateFromHDF5 (sgd_solver.cpp:325-347)
    H5Node root;
    if (!h5_read(path, &root, err)) return false;
    const H5Node *it = root.find("iter"), *cs = root.find("current_step"), *ln = root.find("learned_net"),
                 *h = root.find("history");
    if (!it || it->kind != H5Node::kInt32 || it->i32.empty() || !cs || cs->kind != H5Node::kInt32 || cs->i32.empty() ||
        !h || h->kind != H5Node::kGroup) {
      *err = "'" + path + "' is not a SolverState HDF5 file (iter / current_step / history missing)";
      return false;
    }
    if (iter) *iter = it->i32[0];
    if (current_step) *current_step = cs->i32[0];
    if (learned_net) *learned_net = (ln && ln->kind == H5Node::kString) ? ln->str : std::string();
    return numbered_blobs(*h, path, false, history, err);
  }
  std::vector<unsigned char> buf;
  if (!slurp(path, &buf, err)) return false;
  Reader r{buf.data(), buf.data() + buf.size(), true};
  uint32_t f, wt;
  *iter = 0;
  *current_step = 0;
  bool saw_iter = false;
  while (r.next(&f, &wt)) {
    if (f == 1 && wt == kVarint) {
      *iter = static_cast<int>(static_cast<int64_t>(r.varint()));
      saw_iter = true;
    } else if (f == 2 && wt == kLen) {
      Reader s = r.sub();
      if (learned_net) learned_net->assign(reinterpret_cast<const char*>(s.p), s.end - s.p);
    } else if (f == 3 && wt == kLen) {
      ParsedBlob b;
      if (!parse_blob(r.sub(), &b)) {
        *err = "'" + path + "': malformed history BlobProto";
        return false;
      }
      history->push_back(std::move(b));
    } else if (f == 4 && wt == kVarint) {
      *current_step = static_cast<int>(static_cast<int64_t>(r.varint()));
    } else {
      r.skip(wt);
    }
  }
  if (!r.ok || (!saw_iter && history->empty())) {
    *err = "'" + path + "' is not a SolverState binaryproto";
    return false;
  }
  return true;
}

bool read_blobproto(const std::string& path, ParsedBlob* blob, std::string* err) {
  std::vector<unsigned char> buf;
  if (!slurp(path, &buf, err)) return false;
  *blob = ParsedBlob();
  int64_t n = 1;
  const bool parsed = parse_blob(Reader{buf.data(), buf.data() + buf.size(), true}, blob);
  for (int64_t d : blob->shape) n = d < 0 ? -1 : n * d;
  if (!parsed || blob->shape.empty() || n != static_cast<int64_t>(blob->data.size())) {
    *err = "'" + path + "' is not a BlobProto with float data matching its shape";
    return false;
  }
  return true;
}

}  // namespace cosb
