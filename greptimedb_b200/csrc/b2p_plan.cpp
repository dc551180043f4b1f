// b2p_plan.cpp — host side of GpuPromRangeExec (see b2p_plan.hpp) and its C entry points.
// Pure host C++: everything numeric goes through the C ABI (b2p_range_eval / b2p_group_aggregate).
#include "b2p_plan.hpp"
#include "b2p_regex.hpp"

#include <algorithm>
#include <cctype>
#include <cfloat>
#include <charconv>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <map>
#include <numeric>
#include <unordered_map>

namespace b2p {

namespace {

struct NameId {
  const char* name;
  int id;
};
// UDF display names, src/promql/src/functions/*.rs (`display_name = prom_*`) and planner.rs:2183-2221
const NameId kFns[] = {
    {"prom_rate", B2P_FN_RATE}, {"prom_increase", B2P_FN_INCREASE}, {"prom_delta", B2P_FN_DELTA},
    {"prom_irate", B2P_FN_IRATE}, {"prom_idelta", B2P_FN_IDELTA}, {"prom_resets", B2P_FN_RESETS},
    {"prom_changes", B2P_FN_CHANGES}, {"prom_count_over_time", B2P_FN_COUNT_OVER_TIME},
    {"prom_sum_over_time", B2P_FN_SUM_OVER_TIME}, {"prom_avg_over_time", B2P_FN_AVG_OVER_TIME},
    {"prom_min_over_time", B2P_FN_MIN_OVER_TIME}, {"prom_max_over_time", B2P_FN_MAX_OVER_TIME},
    {"prom_last_over_time", B2P_FN_LAST_OVER_TIME}, {"prom_present_over_time", B2P_FN_PRESENT_OVER_TIME},
    {"prom_absent_over_time", B2P_FN_ABSENT_OVER_TIME}, {"prom_stdvar_over_time", B2P_FN_STDVAR_OVER_TIME},
    {"prom_stddev_over_time", B2P_FN_STDDEV_OVER_TIME}, {"prom_deriv", B2P_FN_DERIV},
    {"prom_predict_linear", B2P_FN_PREDICT_LINEAR}, {"prom_quantile_over_time", B2P_FN_QUANTILE_OVER_TIME},
    {"prom_double_exponential_smoothing", B2P_FN_HOLT_WINTERS}, {"prom_holt_winters", B2P_FN_HOLT_WINTERS},
};
const NameId kAggs[] = {{"sum", B2P_AGG_SUM},       {"avg", B2P_AGG_AVG},       {"count", B2P_AGG_COUNT},
                        {"min", B2P_AGG_MIN},       {"max", B2P_AGG_MAX},       {"stddev", B2P_AGG_STDDEV},
                        {"stdvar", B2P_AGG_STDVAR}};

bool starts_with(const char* s, const char* p) { return std::strncmp(s, p, std::strlen(p)) == 0; }

bool bit_set(const uint8_t* bits, int64_t i) { return bits == nullptr || ((bits[i >> 3] >> (i & 7)) & 1); }

// an Int64 cell's value: the int64_t whose bits the grid's 8-byte slot holds
int64_t bits_i64(double v) {
  int64_t b;
  std::memcpy(&b, &v, sizeof b);
  return b;
}

constexpr int64_t kArrowFlagNullable = 2;  // ARROW_FLAG_NULLABLE of the C Data Interface

// Throws the PlanError of a failed b2p_* call, with the call's message: arguments the call rejects (B2P_E_INVALID,
// B2P_E_TOO_LARGE) as `invalid`, input out of series order (B2P_E_UNSORTED) as Internal, anything else as Execution.
void check(int rc, ErrorKind invalid = ErrorKind::Plan) {
  if (rc == B2P_OK) return;
  if (rc == B2P_E_INVALID || rc == B2P_E_TOO_LARGE) throw PlanError(invalid, b2p_last_error());
  throw PlanError(rc == B2P_E_UNSORTED ? ErrorKind::Internal : ErrorKind::Execution, b2p_last_error());
}

// Field f of r read as Float64 from here on.  Only an Int64 field's cells change: they are coerced on the device
// ((double)i64, b2p_i64_to_f64), as DataFusion coerces an Int64 column under a Float64 projection, aggregate or
// scalar(); Int32 and Count cells already hold their value as a double, and converting them would misread them.
void field_to_f64(b2p_ctx* ctx, NodeResult& r, uint32_t f) {
  if (r.types[f] == ValueType::Int64 && r.grid() > 0)
    check(b2p_i64_to_f64(ctx, reinterpret_cast<const int64_t*>(r.field(f)), r.grid(), r.field(f)));
  r.types[f] = ValueType::Float64;
}
void to_f64(b2p_ctx* ctx, NodeResult& r) {
  for (uint32_t f = 0; f < r.F; ++f) field_to_f64(ctx, r, f);
}

// r's steps: the grid start + k * interval <= end
void set_grid(NodeResult& r, Millisecond start, Millisecond end, Millisecond interval) {
  r.T = b2p_num_steps(start, end, interval);
  r.Tw = (uint32_t)((r.T + 31) / 32);
  r.eval_ts.resize((size_t)r.T);
  for (int64_t k = 0; k < r.T; ++k) r.eval_ts[(size_t)k] = start + k * interval;
}

// The shapes of child result a node may refuse (DESIGN §1 a24-a27).  Int32: DataFusion's integer result types are not
// pinned by the reference tree for a node that reads the number other than element-wise.  Counted: a count_values
// result, whose counted value the reference carries as a column this layer does not model above it.
enum class Shape { MultiField, Int32, Int64, IdKeyed, Counted };

// A node's contract with its one child, checked before the node's work: the first listed shape the child has is a Plan
// error with its text (an empty text accepts the shape after all)
void check_child(const NodeResult& c, std::initializer_list<std::pair<Shape, std::string>> refused) {
  for (const auto& [shape, text] : refused) {
    const bool hit = shape == Shape::MultiField ? c.F > 1
                     : shape == Shape::Int32    ? c.has(ValueType::Int32)
                     : shape == Shape::Int64    ? c.has(ValueType::Int64)
                     : shape == Shape::IdKeyed  ? c.labels.id_keyed
                                                : c.columns == Columns::CountTagsTimeLabel;
    if (hit && !text.empty()) throw PlanError(ErrorKind::Plan, text);
  }
}

// dense ids of keys, in first-insertion order
struct KeyIds {
  std::unordered_map<std::string, uint32_t> ids;
  uint32_t add(const std::string& k) { return ids.emplace(k, (uint32_t)ids.size()).first->second; }
  uint32_t find(const std::string& k) const {
    const auto it = ids.find(k);
    return it == ids.end() ? B2P_NO_KEY : it->second;
  }
};

// ---- export helpers: an ArrowArray whose buffers live in a heap object ---------------------------------
struct OwnedColumn {
  std::vector<int64_t> i64;
  std::vector<int32_t> i32;
  std::vector<double> f64;
  std::vector<int32_t> offsets;
  std::string chars;
  std::vector<uint8_t> validity;  // Utf8 tags: bit i clear = row i is NULL (allocated at the first NULL)
  int64_t nulls = 0;
  const void* buffers[3] = {nullptr, nullptr, nullptr};
};
struct OwnedBatch {
  std::vector<std::unique_ptr<OwnedColumn>> cols;
  std::vector<ArrowArray> child_arrays;
  std::vector<ArrowArray*> child_ptrs;
  const void* buffers[1] = {nullptr};
};
struct OwnedSchema {
  std::vector<std::string> names, formats;
  std::vector<ArrowSchema> children;
  std::vector<ArrowSchema*> child_ptrs;
};

void release_child_array(ArrowArray* a) { a->release = nullptr; }
void release_batch(ArrowArray* a) {
  if (!a || !a->release) return;
  delete static_cast<OwnedBatch*>(a->private_data);
  a->release = nullptr;
}
void release_child_schema(ArrowSchema* s) { s->release = nullptr; }
void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  delete static_cast<OwnedSchema*>(s->private_data);
  s->release = nullptr;
}

}  // namespace

int function_id_from_name(const std::string& n) {
  for (const auto& f : kFns)
    if (n == f.name) return f.id;
  return -1;
}
// str::parse::<f64>() of Rust's std for a label value: optional sign, decimal digits with optional fraction and
// exponent, or inf / infinity / nan in any case — nothing else (no surrounding white space, no hex floats, no locale
// decimal comma: strtod would accept those).  Anything that does not parse is NaN (histogram_fold.rs:791-796).
double parse_f64_like_rust(const std::string& v) {
  const double nan = std::nan("");
  if (v.empty()) return nan;
  size_t i = 0;
  bool neg = false;
  if (v[0] == '+' || v[0] == '-') {
    neg = v[0] == '-';
    i = 1;
  }
  if (i >= v.size()) return nan;
  auto ieq = [&](const char* w) {
    size_t n = std::strlen(w);
    if (v.size() - i != n) return false;
    for (size_t k = 0; k < n; ++k)
      if (std::tolower((unsigned char)v[i + k]) != w[k]) return false;
    return true;
  };
  if (ieq("inf") || ieq("infinity")) return neg ? -HUGE_VAL : HUGE_VAL;
  if (ieq("nan")) return nan;
  bool digits = false, dot = false, exp = false;
  for (size_t k = i; k < v.size(); ++k) {
    const char ch = v[k];
    if (ch >= '0' && ch <= '9') {
      digits = true;
    } else if (ch == '.' && !dot && !exp) {
      dot = true;
    } else if ((ch == 'e' || ch == 'E') && digits && !exp) {
      exp = true;
      if (k + 1 < v.size() && (v[k + 1] == '+' || v[k + 1] == '-')) ++k;
      if (k + 1 >= v.size()) return nan;  // exponent without digits
      digits = true;
      for (size_t q = k + 1; q < v.size(); ++q)
        if (v[q] < '0' || v[q] > '9') return nan;
      break;
    } else {
      return nan;
    }
  }
  if (!digits) return nan;
  double out = 0.0;
  const auto r = std::from_chars(v.data() + i, v.data() + v.size(), out, std::chars_format::general);
  if (r.ec != std::errc() || r.ptr != v.data() + v.size()) {
    if (r.ec == std::errc::result_out_of_range) out = HUGE_VAL;  // Rust saturates to inf (and to 0 on underflow)
    else return nan;
  }
  return neg ? -out : out;
}

int aggregate_id_from_name(const std::string& n) {
  for (const auto& f : kAggs)
    if (n == f.name) return f.id;
  return -1;
}

// ---- RecordBatch -------------------------------------------------------------------------------------
RecordBatch::RecordBatch(ArrowArray* array, ArrowSchema* schema) {
  if (!array || !schema || !array->release || !schema->release)
    throw PlanError(ErrorKind::Internal, "RecordBatch: released or NULL Arrow C structs");
  array_ = *array;
  schema_ = *schema;
  array->release = nullptr;  // moved
  schema->release = nullptr;
  if (!schema_.format || std::strcmp(schema_.format, "+s") != 0 || array_.n_children != schema_.n_children) {
    array_.release(&array_);
    schema_.release(&schema_);
    throw PlanError(ErrorKind::Execution, "RecordBatch: expected a struct array (format \"+s\")");
  }
}
RecordBatch::~RecordBatch() {
  if (array_.release) array_.release(&array_);
  if (schema_.release) schema_.release(&schema_);
}
int RecordBatch::find(const std::string& name) const {
  for (int64_t i = 0; i < schema_.n_children; ++i)
    if (schema_.children[i]->name && name == schema_.children[i]->name) return (int)i;
  return -1;
}

// ---- Labels --------------------------------------------------------------------------------------------
int Labels::column(const std::string& name) const {
  const auto it = std::find(names.begin(), names.end(), name);
  return it == names.end() ? -1 : (int)(it - names.begin());
}

std::vector<int> Labels::columns(const std::vector<std::string>& ns) const {
  std::vector<int> cols;
  for (const std::string& n : ns) cols.push_back(column(n));
  return cols;
}

Label Labels::value(int c, uint32_t r) const {
  if (c < 0) return std::nullopt;
  return id_keyed ? Label(std::to_string(ids[r])) : values[(size_t)c][r];
}

// NULL is "-"; a string is its length, ':' and its bytes.  No encoding is a prefix of another, so no two tuples share one.
void Labels::key(uint32_t r, const std::vector<int>& cols, std::string& key) const {
  key.clear();
  auto put = [&](const std::string& v) {
    key += std::to_string(v.size());
    key.push_back(':');
    key += v;
  };
  for (int c : cols) {
    if (c >= 0 && id_keyed) {
      put(std::to_string(ids[r]));
    } else if (c >= 0 && values[(size_t)c][r]) {
      put(*values[(size_t)c][r]);
    } else {
      key.push_back('-');
    }
  }
}

Labels Labels::gather(const std::vector<uint32_t>& rows) const {
  Labels out;
  out.names = names;
  out.id_keyed = id_keyed;
  out.tsid = tsid;
  if (id_keyed || tsid)
    for (uint32_t r : rows) out.ids.push_back(ids[r]);
  out.values.resize(values.size());
  for (size_t t = 0; t < values.size(); ++t) {
    out.values[t].reserve(rows.size());
    for (uint32_t r : rows) out.values[t].push_back(values[t][r]);
  }
  return out;
}

// "" first, then NULL, then every other string in byte order, the order this plan layer's sorted output has always had.
// The reference's aggregate sorts NULLs last instead (planner.rs:443, `sort(true, false)`); DESIGN.md §2 lists this as
// a known divergence.
bool Labels::less(const Label& a, const Label& b) {
  auto rank = [](const Label& v) { return !v ? 1 : v->empty() ? 0 : 2; };
  if (rank(a) != rank(b)) return rank(a) < rank(b);
  return rank(a) == 2 && *a < *b;
}

namespace {

// The rows of `in` grouped by their tuple over `cols`, for output in label order (the by-label aggregate, HistogramFold)
struct Groups {
  std::vector<uint32_t> id;     // [row] its group, numbered in order of first appearance
  std::vector<uint32_t> first;  // [group] its first row
  std::vector<uint32_t> rank;   // [group] its place in label order
  Labels labels;               // [place] the group's tuple over `cols` (ids as decimal strings)
};

Groups group_rows(const Labels& in, const std::vector<int>& cols, uint32_t rows) {
  Groups g;
  g.id.resize(rows);
  KeyIds ids;
  std::vector<uint32_t>& first = g.first;
  std::string key;
  for (uint32_t r = 0; r < rows; ++r) {
    in.key(r, cols, key);
    g.id[r] = ids.add(key);
    if (g.id[r] == first.size()) first.push_back(r);
  }
  const uint32_t G = (uint32_t)first.size();
  Labels tuples;  // [group]
  tuples.values.resize(cols.size());
  for (size_t t = 0; t < cols.size(); ++t) {
    tuples.names.push_back(in.names[(size_t)cols[t]]);
    for (uint32_t f : first) tuples.values[t].push_back(in.value(cols[t], f));
  }
  std::vector<uint32_t> order(G);
  std::iota(order.begin(), order.end(), 0u);
  std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
    for (const std::vector<Label>& col : tuples.values) {
      if (Labels::less(col[x], col[y])) return true;
      if (Labels::less(col[y], col[x])) return false;
    }
    return false;
  });
  g.rank.resize(G);
  for (uint32_t q = 0; q < G; ++q) g.rank[order[q]] = q;
  g.labels = tuples.gather(order);
  return g;
}

// keep_tsid (planner.rs:347-416): an aggregate other than count_values keeps first_value(__tsid) as __tsid when its
// child carries __tsid and it groups on the child's full label set (a metric-engine leaf's declared label columns)
bool keeps_tsid(const Labels& in, std::vector<int> cols) {
  if (!in.tsid) return false;
  std::sort(cols.begin(), cols.end());
  cols.erase(std::unique(cols.begin(), cols.end()), cols.end());
  return cols.size() == in.names.size() && (cols.empty() || cols.front() >= 0);
}

// ---- the group-label agreement of a sharded node (b2p_group_keys_merge's block layout, include/b200promql.h) ----
constexpr uint32_t kNullTag = 0xFFFFFFFFu, kFlagTsid = 1u;

// a block: the rank's row count and field types, then its groups in Labels order, each its tuple over the group
// columns and, with kFlagTsid, its __tsid
struct KeyBlock {
  uint32_t n_labels = 0, flags = 0;
  uint64_t n_rows = 0;
  std::vector<uint8_t> types;              // [field] enum ValueType
  std::vector<std::vector<Label>> tuples;  // [group][label]
  std::vector<uint64_t> ids;               // [group] with kFlagTsid
};

// What every rank of a sharded node agrees: the global group table in Labels order (with ids where kept), this rank's
// groups -> global ids, the rows of all ranks and the field types of the ranks that have rows
struct Agreement {
  Labels labels;
  uint32_t n_groups = 0;
  std::vector<uint32_t> l2g;  // [this rank's place] -> global id
  uint64_t n_rows = 0;
  std::vector<ValueType> types;
};

bool tuple_less(const std::vector<Label>& a, const std::vector<Label>& b) {
  for (size_t t = 0; t < a.size(); ++t) {
    if (Labels::less(a[t], b[t])) return true;
    if (Labels::less(b[t], a[t])) return false;
  }
  return false;
}

template <class T>
void put(std::string& out, T v) {
  out.append(reinterpret_cast<const char*>(&v), sizeof v);  // (little-endian hosts only, as the project's targets are)
}

// `groups` [place] (Labels order), with their ids when `tsid`; the block of a rank with n_rows rows of these types
std::string serialize_keys(const Labels& groups, uint32_t G, bool tsid, uint64_t n_rows,
                           const std::vector<ValueType>& types) {
  std::string out;
  put<uint32_t>(out, G);
  put<uint32_t>(out, (uint32_t)groups.values.size());
  put<uint32_t>(out, tsid ? kFlagTsid : 0u);
  put<uint32_t>(out, (uint32_t)types.size());
  put<uint64_t>(out, n_rows);
  for (ValueType t : types) put<uint8_t>(out, (uint8_t)t);
  for (uint32_t g = 0; g < G; ++g) {
    if (tsid) put<uint64_t>(out, groups.ids[g]);
    for (const std::vector<Label>& col : groups.values) {
      const Label& v = col[g];
      put<uint32_t>(out, v ? (uint32_t)v->size() : kNullTag);
      if (v) out += *v;
    }
  }
  return out;
}

KeyBlock parse_keys(const uint8_t* p, uint64_t size, int rank) {
  auto bad = [&](const char* what) {
    return PlanError(ErrorKind::Plan, "b2p_group_keys_merge: block " + std::to_string(rank) + " " + what);
  };
  uint64_t at = 0;
  auto get = [&](auto& v) {
    if (size - at < sizeof v) throw bad("is truncated");
    std::memcpy(&v, p + at, sizeof v);
    at += sizeof v;
  };
  KeyBlock b;
  uint32_t G = 0, F = 0;
  get(G);
  get(b.n_labels);
  get(b.flags);
  get(F);
  get(b.n_rows);
  if (b.flags & ~kFlagTsid) throw bad("has unknown flags");
  if ((G == 0) != (b.n_rows == 0)) throw bad("has rows without groups or groups without rows");
  if (F > size - at) throw bad("is truncated");
  b.types.resize(F);
  for (uint8_t& t : b.types) {
    get(t);
    if (t > (uint8_t)ValueType::Count) throw bad("has an unknown field type");
  }
  for (uint32_t g = 0; g < G; ++g) {
    if (b.flags & kFlagTsid) get(b.ids.emplace_back());
    std::vector<Label> t(b.n_labels);
    for (Label& v : t) {
      uint32_t n = 0;
      get(n);
      if (n == kNullTag) continue;
      if (size - at < n) throw bad("is truncated");
      v = std::string(reinterpret_cast<const char*>(p + at), n);
      at += n;
    }
    if (!b.tuples.empty() && !tuple_less(b.tuples.back(), t)) throw bad("is not strictly in label order");
    b.tuples.push_back(std::move(t));
  }
  if (at != size) throw bad("is longer than its groups");
  return b;
}

// The R-way merge: the global table in Labels order without duplicates (a duplicate keeps the lowest rank's id), and
// l2g [block rank's groups] -> global id.  The heads are scanned in rank order and replaced on a strictly smaller tuple
// only, so the table is a function of the blocks alone, whichever rank merges.  The field types are those of the ranks
// with rows, which must agree (a rank without rows has read no batch, so its types are only a default).
Agreement merge_keys(const std::vector<KeyBlock>& blocks, int rank) {
  const KeyBlock& b0 = blocks.at(0);
  Agreement a;
  a.labels.tsid = (b0.flags & kFlagTsid) != 0;
  a.labels.values.resize(b0.n_labels);
  const KeyBlock* typed = nullptr;
  for (size_t r = 0; r < blocks.size(); ++r) {
    const KeyBlock& b = blocks[r];
    if (b.n_labels != b0.n_labels || b.flags != b0.flags || b.types.size() != b0.types.size())
      throw PlanError(ErrorKind::Plan, "b2p_group_keys_merge: block " + std::to_string(r) +
                                           " is unlike block 0 in its labels, flags or fields");
    a.n_rows += b.n_rows;
    if (!b.n_rows) continue;
    if (typed && typed->types != b.types)
      throw PlanError(ErrorKind::Plan, "a sharded node's ranks read different value types (block " + std::to_string(r) +
                                           " against the first rank with rows)");
    if (!typed) typed = &b;
  }
  for (uint8_t t : (typed ? typed : &b0)->types) a.types.push_back((ValueType)t);
  a.l2g.assign(blocks.at((size_t)rank).tuples.size(), 0u);
  std::vector<size_t> head(blocks.size(), 0);
  for (;; ++a.n_groups) {
    int m = -1;
    for (size_t r = 0; r < blocks.size(); ++r)
      if (head[r] < blocks[r].tuples.size() && (m < 0 || tuple_less(blocks[r].tuples[head[r]], blocks[m].tuples[head[m]])))
        m = (int)r;
    if (m < 0) break;
    const std::vector<Label>& t = blocks[m].tuples[head[m]];
    for (size_t c = 0; c < t.size(); ++c) a.labels.values[c].push_back(t[c]);
    if (a.labels.tsid) a.labels.ids.push_back(blocks[m].ids[head[m]]);
    for (size_t r = 0; r < blocks.size(); ++r) {  // every head equal to t (none is smaller)
      if (head[r] >= blocks[r].tuples.size() || (r != (size_t)m && tuple_less(t, blocks[r].tuples[head[r]]))) continue;
      if ((int)r == rank) a.l2g[head[r]] = a.n_groups;
      ++head[r];
    }
  }
  return a;
}

// The agreement of a sharded node over r's rows grouped as `groups` (their ids when `groups.labels.tsid`): this rank's
// block exchanged over the context's communicator and merged.  r takes the agreed field types, so a rank that read no
// batch folds with the types of the ranks that did, and every rank makes the same collective calls.
Agreement agree_groups(b2p_ctx* ctx, const Groups& groups, NodeResult& r) {
  int32_t rank = 0;
  const int32_t R = b2p_comm_ranks(ctx, &rank);
  const std::string mine = serialize_keys(groups.labels, (uint32_t)groups.first.size(), groups.labels.tsid, r.rows,
                                          r.types);
  std::vector<uint64_t> sizes((size_t)R);
  check(b2p_group_keys_sizes(ctx, mine.size(), sizes.data()), ErrorKind::Execution);
  std::vector<uint8_t> all((size_t)std::accumulate(sizes.begin(), sizes.end(), uint64_t(0)));
  check(b2p_group_keys_allgather(ctx, mine.data(), sizes.data(), all.data()), ErrorKind::Execution);
  std::vector<KeyBlock> blocks;
  uint64_t off = 0;
  for (int32_t q = 0; q < R; ++q) {
    blocks.push_back(parse_keys(all.data() + off, sizes[(size_t)q], q));
    off += sizes[(size_t)q];
  }
  Agreement a = merge_keys(blocks, rank);
  a.labels.names = groups.labels.names;
  r.types = a.types;
  return a;
}

// Groups over the global table of a sharded node: the ids become global ids, the places the identity (the global ids
// are already in label order)
void take_global(Groups& groups, Agreement& a) {
  for (uint32_t& id : groups.id) id = a.l2g[groups.rank[id]];
  groups.rank.resize(a.n_groups);
  std::iota(groups.rank.begin(), groups.rank.end(), 0u);
  groups.labels = std::move(a.labels);
}

// Aggregators beyond enum b2p_agg that the aggregate node offers
constexpr int kAggGroup = B2P_AGG_STDVAR + 1, kAggQuantile = B2P_AGG_STDVAR + 2;

// The by-label aggregate of r's [rows x T] grids (the leaf's aggregate stage and AggregatePlan): r's rows grouped by
// their tuple over `cols` (of r.labels), folded on the device in row order, become one row per group in label order,
// a group having a cell at step k iff one of its rows has.  op: enum b2p_agg, kAggGroup (1.0 wherever count is
// non-zero) or kAggQuantile (param = φ).  Each field is folded by its own call over the same group ids; the counts
// depend on the shared validity alone, so field 0's decide the cells.  Sets the rows, labels, grids, types and column
// layout, drops a counted column; keeps T, the fields and the time index.  A group keeps its first member's __tsid
// where keeps_tsid says so.  `sharded` (a sharded node over a communicator): the groups are the global table every rank
// agrees (agree_groups), and each fold merges every rank's partials, so every rank ends with the same result.
void aggregate_rows(b2p_ctx* ctx, int op, double param, const std::vector<int>& cols, NodeResult& r, bool sharded = false) {
  Groups groups = group_rows(r.labels, cols, r.rows);
  if (keeps_tsid(r.labels, cols)) {
    groups.labels.tsid = true;
    groups.labels.ids.resize(groups.first.size());
    for (size_t g = 0; g < groups.first.size(); ++g) groups.labels.ids[groups.rank[g]] = r.labels.ids[groups.first[g]];
  }
  if (sharded) {
    Agreement a = agree_groups(ctx, groups, r);
    take_global(groups, a);
  }
  const uint32_t G = (uint32_t)groups.rank.size(), Tw = r.Tw, F = r.F;
  const size_t T = (size_t)r.T;
  std::vector<double> gval((size_t)F * G * T);
  std::vector<uint32_t> gcnt((size_t)G * T), fcnt(F > 1 ? (size_t)G * T : 0);
  // an Int64 field stays Int64 under sum, min and max (DataFusion's Int64 accumulators); the others give Float64
  const bool int_result = op == B2P_AGG_SUM || op == B2P_AGG_MIN || op == B2P_AGG_MAX;
  std::vector<ValueType> types(F, ValueType::Float64);
  for (uint32_t f = 0; f < F; ++f) {
    const bool i64 = r.types[f] == ValueType::Int64 && op != kAggQuantile && op != kAggGroup;
    // the sharded Int64 avg / stddev / stdvar / count read the Float64 coercion, which is what K3 reads in one pass
    if (op == kAggQuantile || (sharded && i64 && !int_result)) field_to_f64(ctx, r, f);
    if (int_result && r.types[f] == ValueType::Int64) types[f] = ValueType::Int64;
    if (G == 0 || T == 0) continue;  // (G and T are the same on every rank)
    double* gv = gval.data() + (size_t)f * G * T;
    uint32_t* gc = f == 0 ? gcnt.data() : fcnt.data();
    const int agg = op == kAggGroup ? B2P_AGG_COUNT : op;
    if (sharded)
      check(op == kAggQuantile ? b2p_quantile_allreduce(ctx, param, r.field(f), r.valid.data(), groups.id.data(), r.rows,
                                                        G, (uint64_t)T, gv, gc)
            : i64 && int_result ? b2p_group_aggregate_allreduce_i64(ctx, agg, reinterpret_cast<const int64_t*>(r.field(f)),
                                                                    r.valid.data(), groups.id.data(), r.rows, G,
                                                                    (uint64_t)T, gv, gc)
                                : b2p_group_aggregate_allreduce(ctx, agg, r.field(f), r.valid.data(), groups.id.data(),
                                                                r.rows, G, (uint64_t)T, gv, gc),
            ErrorKind::Execution);
    else
      check(op == kAggQuantile ? b2p_group_quantile(ctx, param, r.field(f), r.valid.data(), groups.id.data(), r.rows, G,
                                                    (uint64_t)T, gv, gc)
            : i64 ? b2p_group_aggregate_i64(ctx, agg, reinterpret_cast<const int64_t*>(r.field(f)), r.valid.data(),
                                            groups.id.data(), r.rows, G, (uint64_t)T, gv, gc)
                  : b2p_group_aggregate(ctx, agg, r.field(f), r.valid.data(), groups.id.data(), r.rows, G, (uint64_t)T,
                                        gv, gc),
            ErrorKind::Execution);
  }
  r.types = std::move(types);
  r.labels = std::move(groups.labels);
  r.columns = Columns::TagsTimeValue;
  r.cell_order.clear();
  r.counted.reset();
  r.val.assign((size_t)F * G * T, 0.0);
  r.valid.assign((size_t)G * Tw, 0u);
  for (uint32_t g = 0; g < G; ++g) {
    const uint32_t row = groups.rank[g];
    for (size_t k = 0; k < T; ++k) {
      if (gcnt[g * T + k] == 0) continue;
      for (uint32_t f = 0; f < F; ++f)
        r.val[((size_t)f * G + row) * T + k] = op == kAggGroup ? 1.0 : gval[((size_t)f * G + g) * T + k];
      r.valid[(size_t)row * Tw + (k >> 5)] |= 1u << (k & 31);
    }
  }
  r.rows = G;
}

// The HistogramFold index over `rows` rows labelled `in` (histogram_fold.rs:754-820): rows that agree on every tag but
// column `le` form one histogram, histograms in label order; each histogram's buckets in ascending le order (parsed as
// le.parse::<f64>().unwrap_or(NaN), :791-796, NULL as NaN), NaN bounds last, ties in row order: the order of
// b2p_histogram_shard_index, which the sharded fold uses too.  The CSR hist_off / bucket_series / bucket_le is what
// b2p_histogram_fold[_dev] and b2p_range_histogram_fold take.
struct HistogramIndex {
  Groups hist;  // the histograms; hist.labels are their tags without le
  std::vector<uint32_t> hist_off, bucket_series;
  std::vector<double> bucket_le;
};

// the histograms of `rows` rows labelled `in`: the rows grouped by their tags without column `le`
Groups histogram_groups(const Labels& in, int le, uint32_t rows) {
  std::vector<int> cols;
  for (int t = 0; t < (int)in.names.size(); ++t)
    if (t != le) cols.push_back(t);
  return group_rows(in, cols, rows);
}

// each row's parsed bound
std::vector<double> bucket_bounds(const Labels& in, int le, uint32_t rows) {
  std::vector<double> sle(rows);
  for (uint32_t s = 0; s < rows; ++s) {
    const Label& v = in.values[(size_t)le][s];
    sle[s] = v ? parse_f64_like_rust(*v) : std::nan("");
  }
  return sle;
}

HistogramIndex histogram_index(const Labels& in, int le, uint32_t rows) {
  HistogramIndex ix;
  ix.hist = histogram_groups(in, le, rows);
  const uint32_t H = (uint32_t)ix.hist.rank.size();
  const std::vector<double> sle = bucket_bounds(in, le, rows);
  std::vector<uint32_t> place(rows), rank(rows, 0u), row(rows);
  std::iota(row.begin(), row.end(), 0u);
  for (uint32_t s = 0; s < rows; ++s) place[s] = ix.hist.rank[ix.hist.id[s]];
  ix.hist_off.resize((size_t)H + 1);
  ix.bucket_series.resize(rows);
  ix.bucket_le.resize(rows);
  check(b2p_histogram_shard_index(place.data(), sle.data(), rank.data(), row.data(), rows, H, ix.hist_off.data(),
                                  ix.bucket_series.data(), ix.bucket_le.data()));
  return ix;
}

// histogram_quantile over r's rows sharded across ranks: the histograms are agreed (agree_groups, which also gives r
// the field types of the ranks with rows), refuse(r, n_hist) raises what the node refuses on those agreed types on every
// rank alike, then fold(row_hist, row_le, n_hist, out, out_valid) folds each histogram on one rank and replicates the
// result (a b2p_*histogram_fold_allgather call; not made when there is no histogram or step, the same on every rank).
// r becomes the [n_hist x T] rows in label order, the same on every rank.
template <class Refuse, class Fold>
void fold_sharded(b2p_ctx* ctx, int le, NodeResult& r, Refuse&& refuse, Fold&& fold) {
  Groups hist = histogram_groups(r.labels, le, r.rows);
  Agreement a = agree_groups(ctx, hist, r);
  refuse(r, a.n_groups);
  take_global(hist, a);
  const uint32_t H = (uint32_t)hist.rank.size();
  const std::vector<double> sle = bucket_bounds(r.labels, le, r.rows);
  std::vector<double> out((size_t)H * (size_t)r.T, 0.0);
  std::vector<uint32_t> out_valid((size_t)H * r.Tw, 0u);
  if (H > 0 && r.T > 0) check(fold(hist.id.data(), sle.data(), H, out.data(), out_valid.data()), ErrorKind::Execution);
  r.val = std::move(out);
  r.valid = std::move(out_valid);
  r.labels = std::move(hist.labels);
  r.rows = H;
}

}  // namespace

namespace {
bool contains(const std::vector<std::string>& v, const std::string& x) { return std::find(v.begin(), v.end(), x) != v.end(); }
// the metric engine's series id column (DATA_SCHEMA_TSID_COLUMN_NAME)
const char* const kTsid = "__tsid";
}  // namespace

// ---- PromRangePlan -------------------------------------------------------------------------------------
PromRangePlan::PromRangePlan(b2p_ctx* ctx, PromRangePlanArgs args) : PlanNode(ctx), args_(std::move(args)) {
  require("GpuPromRangeExec", {});
  fn_id_ = args_.function.empty() ? -1 : function_id_from_name(args_.function);
  if (fn_id_ < 0 && !args_.function.empty())
    throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: unknown range function " + args_.function);
  agg_id_ = -1;
  if (!args_.aggregate.empty()) {
    agg_id_ = aggregate_id_from_name(args_.aggregate);
    if (agg_id_ < 0) throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: unsupported aggregator " + args_.aggregate);
  }
  // a leaf keyed on __tsid alone may be a metric-engine leaf whose by-columns name its label columns, which come
  // later: it checks them at set_label_columns() and push()
  if (args_.tag_columns != std::vector<std::string>{kTsid}) check_key_columns();
  if (args_.interval <= 0) throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: interval must be positive");
  const std::vector<std::string>& fields = args_.field_columns;
  if (fields.empty() || fields.size() > B2P_MAX_FIELDS)
    throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: between 1 and " + std::to_string(B2P_MAX_FIELDS) +
                                         " field columns are required, got " + std::to_string(fields.size()));
  if (args_.time_index.empty()) throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: time index and field column are required");
  for (size_t f = 0; f < fields.size(); ++f) {
    if (fields[f].empty()) throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: time index and field column are required");
    if (std::find(fields.begin(), fields.begin() + (long)f, fields[f]) != fields.begin() + (long)f)
      throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: field column " + fields[f] + " is given twice");
  }
  // with several fields the aggregate stage would name every field's column alike (sum(prom_rate)): AggregatePlan over
  // this node is the multi-field route
  if (fields.size() > 1 && agg_id_ >= 0)
    throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: the aggregate stage takes one field column; use an aggregate node");
  val_.resize(fields.size());
  present_.resize(fields.size());
  series_.names = args_.tag_columns;
  series_.values.resize(args_.tag_columns.size());
}

// the label columns of a metric-engine leaf, the tag columns of any other
void PromRangePlan::check_key_columns() const {
  const std::vector<std::string>& keys = args_.label_columns.empty() ? args_.tag_columns : args_.label_columns;
  for (const auto& b : args_.by_columns)
    if (agg_id_ >= 0 && !contains(keys, b))
      throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: by-column " + b + " is not a tag column");
  if (args_.histogram && !contains(keys, args_.le_column))
    throw PlanError(ErrorKind::Plan, "HistogramFold: le column " + args_.le_column + " is not a tag column");
}

void PromRangePlan::set_label_columns(std::vector<std::string> names) {
  if (args_.tag_columns != std::vector<std::string>{kTsid})
    throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: label columns need the one tag column to be the UInt64 id __tsid");
  if (have_last_) throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: label columns must be set before the first batch");
  if (names.empty()) throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: at least one label column is required");
  for (size_t i = 0; i < names.size(); ++i) {
    const std::string& n = names[i];
    if (n.empty() || n == args_.time_index || n == args_.tag_columns[0] || contains(args_.field_columns, n))
      throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: label column \"" + n +
                                           "\" is named like the time index, a field column or the id column");
    if (std::find(names.begin(), names.begin() + (long)i, n) != names.begin() + (long)i)
      throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: label column " + n + " is given twice");
  }
  args_.label_columns = std::move(names);
  series_ = Labels();
  series_.names = args_.label_columns;
  series_.values.resize(series_.names.size());
  series_.tsid = true;
  check_key_columns();
}

void PromRangePlan::set_histogram(const std::string& le_column, double quantile) {
  if (!contains(args_.label_columns.empty() ? args_.tag_columns : args_.label_columns, le_column))
    throw PlanError(ErrorKind::Plan, "HistogramFold: le column " + le_column + " is not a tag column");
  if (!args_.aggregate.empty())
    throw PlanError(ErrorKind::Plan, "HistogramFold over an aggregate is not supported by this node");
  if (args_.field_columns.size() > 1)
    throw PlanError(ErrorKind::Plan, "HistogramFold over several field columns is not supported by this node");
  args_.histogram = true;
  args_.le_column = le_column;
  args_.quantile = quantile;
}

void PromRangePlan::push(std::unique_ptr<RecordBatch> batch) {
  const RecordBatch& b = *batch;
  const int64_t n = b.num_rows();
  if (n == 0) return;  // an empty batch is skipped (never parks the stream, SURVEY appendix C-11)
  check_key_columns();
  const int ti = b.find(args_.time_index);
  if (ti < 0) throw PlanError(ErrorKind::Plan, "No field named " + args_.time_index);  // field_not_found
  const size_t F = args_.field_columns.size();
  std::vector<int> fi(F);
  for (size_t f = 0; f < F; ++f) {
    fi[f] = b.find(args_.field_columns[f]);
    if (fi[f] < 0) throw PlanError(ErrorKind::Plan, "No field named " + args_.field_columns[f]);
  }
  const char* tfmt = b.field(ti).format;
  if (!(starts_with(tfmt, "tsm:") || std::strcmp(tfmt, "l") == 0))
    throw PlanError(ErrorKind::Execution, "Time index Column downcast to TimestampMillisecondArray failed");
  // Float64, or for the instant selector Int64 (BIGINT): its cells are copied as they are, and read as integers by the
  // nodes above.  A range function over an Int64 column stays on the CPU.
  std::vector<ValueType> types(F);
  for (size_t f = 0; f < F; ++f) {
    const char* fmt = b.field(fi[f]).format;
    const bool int_ok = fn_id_ < 0 && !args_.histogram && agg_id_ < 0;
    if (std::strcmp(fmt, "g") != 0 && !(int_ok && std::strcmp(fmt, "l") == 0))
      throw PlanError(ErrorKind::Execution, "field column " + args_.field_columns[f] + " is not Float64");
    types[f] = fmt[0] == 'l' ? ValueType::Int64 : ValueType::Float64;
  }
  if (types_.empty()) types_ = types;
  if (types != types_)
    throw PlanError(ErrorKind::Execution, "GpuPromRangeExec: a field column changed its type between batches");
  const ArrowArray& ta = b.column(ti);
  const int64_t* tsv = static_cast<const int64_t*>(ta.buffers[1]) + ta.offset + b.offset();

  // tag columns: Utf8 (int32 offsets) tuple, or a single UInt64 id
  struct TagCol {
    const int32_t* off;
    const char* data;
    const uint8_t* valid;
    int64_t base;
    const uint64_t* ids;
  };
  const bool metric_engine = !args_.label_columns.empty();
  auto column = [&](int ci) {  // a Utf8 column (offsets, data) or the UInt64 id column
    const ArrowArray& ca = b.column(ci);
    TagCol tc{};
    tc.base = ca.offset + b.offset();
    tc.valid = ca.null_count != 0 ? static_cast<const uint8_t*>(ca.buffers[0]) : nullptr;
    if (std::strcmp(b.field(ci).format, "u") == 0) {
      tc.off = static_cast<const int32_t*>(ca.buffers[1]);
      tc.data = static_cast<const char*>(ca.buffers[2]);
    } else {
      tc.ids = static_cast<const uint64_t*>(ca.buffers[1]);
    }
    return tc;
  };
  std::vector<TagCol> tcols;
  for (size_t t = 0; t < args_.tag_columns.size(); ++t) {
    const int ci = b.find(args_.tag_columns[t]);
    if (ci < 0) throw PlanError(ErrorKind::Plan, "No field named " + args_.tag_columns[t]);
    const char* fmt = b.field(ci).format;
    if (std::strcmp(fmt, "L") == 0 && args_.tag_columns.size() == 1) {
      if (!metric_engine) {
        series_.id_keyed = true;
        series_.values.clear();
      }
    } else if (metric_engine) {
      throw PlanError(ErrorKind::Plan, "GpuPromRangeExec: label columns need the tag column " + args_.tag_columns[t] +
                                           " to be a UInt64 id");
    } else if (std::strcmp(fmt, "u") != 0) {
      throw PlanError(ErrorKind::Execution, "tag column " + args_.tag_columns[t] + " must be Utf8 (or one UInt64 id)");
    }
    tcols.push_back(column(ci));
  }
  // a metric-engine leaf's label columns: read at the first row of each series only
  std::vector<TagCol> lcols;
  for (const std::string& l : args_.label_columns) {
    const int ci = b.find(l);
    if (ci < 0) throw PlanError(ErrorKind::Plan, "No field named " + l);
    if (std::strcmp(b.field(ci).format, "u") != 0) throw PlanError(ErrorKind::Execution, "label column " + l + " must be Utf8");
    lcols.push_back(column(ci));
  }
  auto utf8_at = [&](const TagCol& tc, int64_t row) -> Label {
    const int64_t r = tc.base + row;
    if (!bit_set(tc.valid, r)) return std::nullopt;
    return std::string(tc.data + tc.off[r], (size_t)(tc.off[r + 1] - tc.off[r]));
  };
  auto tag_at = [&](size_t t, int64_t row) -> Label { return utf8_at(tcols[t], row); };

  // Columns are taken over in bulk (the Arrow values buffers are already the device layout): one memcpy per column
  // and batch, no per-row growth.  SeriesDivide only has to find the rows where a new series starts
  // (find_first_diff_row compares adjacent rows, series_divide.rs:658-667, and the first row of a batch with the last
  // row of the previous one, :636-645); the result is the offsets array the device kernels take — the 4 B/row id
  // column is never built nor shipped.
  const size_t row_base = ts_.size();
  ts_.insert(ts_.end(), tsv, tsv + n);
  for (size_t f = 0; f < F; ++f) {
    const ArrowArray& fa = b.column(fi[f]);
    const int64_t base = fa.offset + b.offset();
    const double* fv = static_cast<const double*>(fa.buffers[1]) + base;
    const uint8_t* fvalid = fa.null_count != 0 ? static_cast<const uint8_t*>(fa.buffers[0]) : nullptr;
    std::vector<double>& v = val_[f];
    v.insert(v.end(), fv, fv + n);
    if (F == 1 && types_[0] == ValueType::Float64) {
      if (fvalid) {  // a NULL field value cannot be inside a window: treat it like the NaN the filter drops
        for (int64_t row = 0; row < n; ++row)
          if (!bit_set(fvalid, base + row)) v[row_base + (size_t)row] = std::nan("");
      }
      continue;
    }
    // several fields, or an Int64 field: the device decides per function what a NULL slot means
    // (b2p_range_eval_fields), so the slots go down as one bitmap per field, rows from bit 0; a field without a NULL so
    // far has none
    std::vector<uint8_t>& bits = present_[f];
    if (!fvalid && bits.empty()) continue;
    const size_t total = row_base + (size_t)n;
    if (bits.empty()) bits.assign((row_base + 7) / 8, 0xFF);
    bits.resize((total + 7) / 8, 0xFF);
    for (int64_t row = 0; row < n; ++row) {
      const size_t at = row_base + (size_t)row;
      if (bit_set(fvalid, base + row)) bits[at >> 3] |= (uint8_t)(1u << (at & 7));
      else bits[at >> 3] &= (uint8_t)~(1u << (at & 7));
    }
  }
  auto start_series = [&](int64_t row) {
    offsets_.push_back((uint64_t)(row_base + (size_t)row));
    ++num_series_;
  };
  if (series_.id_keyed || series_.tsid) {
    const uint64_t* ids = tcols[0].ids + tcols[0].base;
    auto open_id_series = [&](int64_t row) {
      series_.ids.push_back(ids[row]);
      for (size_t l = 0; l < lcols.size(); ++l) series_.values[l].push_back(utf8_at(lcols[l], row));
      start_series(row);
    };
    int64_t row = 0;
    if (!have_last_ || ids[0] != last_id_) open_id_series(0);
    for (row = 1; row < n; ++row)
      if (ids[row] != ids[row - 1]) open_id_series(row);  // (a tight compare loop the compiler vectorises)
    last_id_ = ids[n - 1];
  } else if (!tcols.empty()) {
    // adjacent-row compare on the raw Utf8 buffers; label strings are only materialised for the first row of a series
    auto same_as_prev = [&](int64_t row) -> bool {  // row >= 1
      for (const TagCol& tc : tcols) {
        const int64_t r = tc.base + row;
        const bool v = bit_set(tc.valid, r), pv = bit_set(tc.valid, r - 1);
        if (v != pv) return false;
        if (!v) continue;
        const int32_t len = tc.off[r + 1] - tc.off[r];
        if (len != tc.off[r] - tc.off[r - 1]) return false;
        if (std::memcmp(tc.data + tc.off[r], tc.data + tc.off[r - 1], (size_t)len) != 0) return false;
      }
      return true;
    };
    auto same_as_last_key = [&]() -> bool {  // first row of this batch against the previous batch's last row
      for (size_t t = 0; t < tcols.size(); ++t)
        if (tag_at(t, 0) != last_key_[t]) return false;
      return true;
    };
    auto open_series = [&](int64_t row) {
      for (size_t t = 0; t < tcols.size(); ++t) series_.values[t].push_back(tag_at(t, row));
      start_series(row);
    };
    if (!have_last_ || !same_as_last_key()) open_series(0);
    for (int64_t row = 1; row < n; ++row)
      if (!same_as_prev(row)) open_series(row);
    last_key_.resize(tcols.size());
    for (size_t t = 0; t < tcols.size(); ++t) last_key_[t] = tag_at(t, n - 1);
  } else if (!have_last_) {
    start_series(0);  // no tag columns: the whole input is one series (series_divide.rs:624-627)
  }
  have_last_ = true;
}

void PromRangePlan::compute(NodeResult& r) {
  b2p_range_params p{};
  p.fn_id = fn_id_;
  p.filter_nan = args_.need_filter_out_nan ? 1 : 0;
  p.start = args_.start;
  p.end = args_.end;
  p.interval = args_.interval;
  p.range = args_.range;
  p.offset = args_.offset;
  p.param0 = args_.param0;
  p.param1 = args_.param1;
  r = NodeResult();
  set_grid(r, p.start, p.end, p.interval);  // also when there are no series: scalar() of such a node has a NaN row at every step
  const int64_t T = r.T;
  const uint32_t Tw = r.Tw;
  check_key_columns();
  const uint32_t S = (uint32_t)num_series_;
  offsets_.resize((size_t)S);          // (a previous execute() appended the end marker)
  offsets_.push_back((uint64_t)ts_.size());
  // timestamp(): one Float64 value whatever the fields, DEFAULT_FIELD_COLUMN (planner.rs:951-965); no value is read
  const uint32_t F = timestamp_ ? 1u : (uint32_t)args_.field_columns.size();
  const bool sharded = sharded_ && sharded_run("GpuPromRangeExec");
  const bool fold_on_device = args_.histogram && fn_id_ >= 0;  // the dense matrix then never reaches the host
  const size_t cells = (size_t)S * (size_t)T;
  std::vector<double> dense(fold_on_device ? 0 : F * cells);
  std::vector<uint32_t> valid(fold_on_device ? 0 : (size_t)S * Tw);
  const bool int0 = !timestamp_ && !types_.empty() && types_[0] == ValueType::Int64;  // (only the instant selector)
  if (S > 0 && T > 0 && timestamp_)
    check(b2p_instant_timestamp(ctx_, p.start, p.end, p.interval, args_.lookback_delta, p.offset, ts_.data(), nullptr,
                                offsets_.data(), ts_.size(), S, dense.data(), valid.data()));
  else if (S > 0 && T > 0 && !fold_on_device && F == 1 && !int0)
    check(fn_id_ >= 0 ? b2p_range_eval(ctx_, &p, ts_.data(), val_[0].data(), nullptr, offsets_.data(), ts_.size(), S,
                                       dense.data(), valid.data(), nullptr)
                      : b2p_instant_select(ctx_, p.start, p.end, p.interval, args_.lookback_delta, p.offset, ts_.data(),
                                           val_[0].data(), nullptr, offsets_.data(), ts_.size(), S, dense.data(),
                                           valid.data()));  // InstantManipulate
  if (S > 0 && T > 0 && !timestamp_ && (F > 1 || int0)) {
    std::vector<const double*> vals(F);
    std::vector<double*> outs(F);
    std::vector<const uint8_t*> present(F);
    bool any_null = false;
    for (uint32_t f = 0; f < F; ++f) {
      vals[f] = val_[f].data();
      outs[f] = dense.data() + f * cells;
      present_[f].resize(present_[f].empty() ? 0 : (ts_.size() + 7) / 8, 0xFF);
      present[f] = present_[f].empty() ? nullptr : present_[f].data();
      any_null = any_null || present[f];
    }
    const uint8_t* const* nulls = any_null ? present.data() : nullptr;
    check(fn_id_ >= 0 ? b2p_range_eval_fields(ctx_, &p, ts_.data(), vals.data(), nulls, (int32_t)F, nullptr,
                                              offsets_.data(), ts_.size(), S, outs.data(), valid.data())
          : int0      ? b2p_instant_select_fields_i64(ctx_, p.start, p.end, p.interval, args_.lookback_delta, p.offset,
                                                      ts_.data(), vals.data(), nulls, (int32_t)F, nullptr,
                                                      offsets_.data(), ts_.size(), S, outs.data(), valid.data())
                      : b2p_instant_select_fields(ctx_, p.start, p.end, p.interval, args_.lookback_delta, p.offset,
                                                  ts_.data(), vals.data(), nulls, (int32_t)F, nullptr, offsets_.data(),
                                                  ts_.size(), S, outs.data(), valid.data()));
  }
  r.F = F;
  r.types = timestamp_ || types_.empty() ? std::vector<ValueType>(F, ValueType::Float64) : types_;
  r.time_index = args_.time_index;
  for (const std::string& field : args_.field_columns)
    r.value_names.push_back(fn_id_ >= 0 ? args_.function + "(" + args_.time_index + "_range," + field + ")" : field);
  if (timestamp_) r.value_names = {"value"};

  if (args_.histogram) {
    // HistogramFold (histogram_fold.rs:754-820): group the series by their tags without `le`, order each group's
    // buckets by le ascending (parsed as f64, "+Inf" last), one output row per (group, eval ts)
    if (series_.id_keyed) throw PlanError(ErrorKind::Plan, "HistogramFold needs the le tag column, not a tsid key");
    if (sharded) {
      // b2p_range_histogram_fold_allgather: the range function writes into the sharded fold's grid on the device
      r.labels = series_;
      r.rows = S;
      const auto refuse = [&](const NodeResult&, uint32_t H) {
        if (H > 0 && T > 0 && fn_id_ < 0)
          throw PlanError(ErrorKind::Plan, "HistogramFold over an instant selector is not supported by this node");
      };
      fold_sharded(ctx_, series_.column(args_.le_column), r, refuse,
                   [&](const uint32_t* row_hist, const double* row_le, uint32_t H, double* out, uint32_t* out_valid) {
                     return b2p_range_histogram_fold_allgather(ctx_, &p, ts_.data(), val_[0].data(), nullptr,
                                                               offsets_.data(), ts_.size(), S, args_.quantile,
                                                               row_hist, row_le, H, out, out_valid);
                   });
      return;
    }
    HistogramIndex ix = histogram_index(series_, series_.column(args_.le_column), S);
    const uint32_t H = (uint32_t)ix.hist.rank.size();
    r.val.assign((size_t)H * (size_t)T, 0.0);
    r.valid.assign((size_t)H * Tw, 0u);
    if (H > 0 && T > 0) {
      if (fn_id_ < 0) throw PlanError(ErrorKind::Plan, "HistogramFold over an instant selector is not supported by this node");
      check(b2p_range_histogram_fold(ctx_, &p, ts_.data(), val_[0].data(), nullptr, offsets_.data(), ts_.size(), S,
                                     args_.quantile, ix.hist_off.data(), ix.bucket_series.data(), ix.bucket_le.data(),
                                     H, r.val.data(), r.valid.data()));
    }
    r.labels = std::move(ix.hist.labels);
    r.rows = H;
  } else {
    // rows of Filter(prom_fn IS NOT NULL): {time_index (eval ts), prom_fn(...), tags...}, series-major order
    r.labels = series_;
    // a range function's and timestamp()'s projection lists time, value and tags: __tsid stays only on the instant
    // selector, which passes every column through (planner.rs:1055-1058, 2714)
    if (fn_id_ >= 0 || timestamp_) r.labels.drop_tsid();
    r.val = std::move(dense);
    r.valid = std::move(valid);
    r.rows = S;
    if (agg_id_ >= 0) {
      // prom_aggr_expr_to_plan: group keys = by-labels + eval ts; output sorted by (labels asc, ts asc).  Over an id key
      // the by-label is the id's decimal string, so those rows sort as strings ("10" before "9").
      aggregate_rows(ctx_, agg_id_, 0.0, series_.columns(args_.by_columns), r, sharded);
      r.value_names = {args_.aggregate + "(" + (fn_id_ >= 0 ? args_.function : args_.field_columns[0]) + ")"};
    }
  }
}

namespace {

// as DataFusion displays the operators in a projection's name (Operator::Eq is "=")
const char* const kOpSymbols[] = {"+", "-", "*", "/", "%", "^", "atan2", "=", "!=", ">", "<", ">=", "<="};

bool is_comparison(int op) { return op >= B2P_OP_EQ && op <= B2P_OP_LE; }

void check_op(int op, bool return_bool) {
  if (op < B2P_OP_ADD || op > B2P_OP_LE) throw PlanError(ErrorKind::Plan, "unknown binary operator " + std::to_string(op));
  if (return_bool && !is_comparison(op))
    throw PlanError(ErrorKind::Plan, "bool modifier can only be used on comparison operators");
}

// a number literal as DataFusion displays it in a column name: Float64(100), Float64(0.5)
std::string float_literal(double x) {
  char buf[64];
  const auto res = std::to_chars(buf, buf + sizeof buf, x);
  return "Float64(" + std::string(buf, res.ptr) + ")";
}

// the tags a matching modifier keeps: those listed in `labels` for On, those not listed for Ignoring, all for None
std::vector<std::string> narrow_tags(const std::vector<std::string>& tags, Matching m, const std::vector<std::string>& labels) {
  std::vector<std::string> out;
  for (const std::string& t : tags) {
    const bool listed = std::find(labels.begin(), labels.end(), t) != labels.end();
    if (m == Matching::On ? listed : !(m == Matching::Ignoring && listed)) out.push_back(t);
  }
  return out;
}

void export_result(const NodeResult& r, ArrowArray* out, ArrowSchema* out_schema) {
  auto ob = std::make_unique<OwnedBatch>();
  auto os = std::make_unique<OwnedSchema>();
  auto add_col = [&](const std::string& name, const std::string& fmt) -> OwnedColumn* {
    ob->cols.push_back(std::make_unique<OwnedColumn>());
    os->names.push_back(name);
    os->formats.push_back(fmt);
    return ob->cols.back().get();
  };
  const Labels& L = r.labels;
  std::vector<OwnedColumn*> c_tags(L.names.size());
  auto add_tag = [&](size_t t) {
    c_tags[t] = add_col(L.names[t], L.id_keyed ? "L" : "u");
    if (!L.id_keyed) c_tags[t]->offsets.push_back(0);
  };
  OwnedColumn* c_ts = nullptr;
  std::vector<OwnedColumn*> c_vals;  // [F]
  OwnedColumn* c_label = nullptr;    // count_values' counted value
  if (r.value_names.size() != r.F) throw PlanError(ErrorKind::Internal, "export: one value name per field expected");
  if (r.types.size() != r.F) throw PlanError(ErrorKind::Internal, "export: one type per field expected");
  if (r.columns == Columns::CountTagsTimeLabel && !r.counted)
    throw PlanError(ErrorKind::Internal, "export: the count_values layout without its counted column");
  // the Arrow format of a column of type t, and how a cell of it is stored
  auto format = [](ValueType t) { return t == ValueType::Float64 ? "g" : t == ValueType::Int32 ? "i" : "l"; };
  auto put = [](OwnedColumn* c, ValueType t, double v) {
    switch (t) {
      case ValueType::Float64: c->f64.push_back(v); break;
      case ValueType::Int64: c->i64.push_back(bits_i64(v)); break;
      case ValueType::Int32: c->i32.push_back((int32_t)v); break;
      case ValueType::Count: c->i64.push_back((int64_t)v); break;
    }
  };
  auto add_vals = [&] {
    for (uint32_t f = 0; f < r.F; ++f) c_vals.push_back(add_col(r.value_names[f], format(r.types[f])));
  };
  switch (r.columns) {
    case Columns::TimeValueTags:
      c_ts = add_col(r.time_index, "tsm:");
      add_vals();
      for (size_t t = 0; t < L.names.size(); ++t) add_tag(t);
      break;
    case Columns::TagsTimeValue:
      for (size_t t = 0; t < L.names.size(); ++t) add_tag(t);
      c_ts = add_col(r.time_index, "tsm:");
      add_vals();
      break;
    case Columns::ValueTagsTime:
      add_vals();
      for (size_t t = 0; t < L.names.size(); ++t) add_tag(t);
      c_ts = add_col(r.time_index, "tsm:");
      break;
    case Columns::CountTagsTimeLabel:
      add_vals();
      for (size_t t = 0; t < L.names.size(); ++t) add_tag(t);
      c_ts = add_col(r.time_index, "tsm:");
      c_label = add_col(r.counted->name, format(r.counted->type));
      break;
    case Columns::TimeSorted: {  // (`or`, one field)
      c_ts = add_col(r.time_index, "tsm:");
      std::vector<std::string> names = L.names;
      names.push_back(r.value_names[0]);
      std::sort(names.begin(), names.end());
      for (const std::string& name : names) {
        if (name == r.value_names[0] && c_vals.empty())
          c_vals.push_back(add_col(name, format(r.types[0])));
        else add_tag((size_t)L.column(name));
      }
      break;
    }
    case Columns::TimeValueLastTag:
      c_ts = add_col(r.time_index, "tsm:");
      add_vals();
      if (!L.names.empty()) add_tag(L.names.size() - 1);
      for (size_t t = 0; t + 1 < L.names.size(); ++t) add_tag(t);
      break;
    case Columns::None:  // (no rows either)
      break;
  }
  // a kept __tsid, after every other column (the reference's own position varies by node; its root projection drops it)
  OwnedColumn* c_tsid = L.tsid && r.columns != Columns::None ? add_col("__tsid", "L") : nullptr;
  int64_t n_out = 0;
  const bool ordered = !r.cell_order.empty();
  const uint64_t n_cells = ordered ? r.cell_order.size() : (uint64_t)r.rows * (uint64_t)r.T;
  for (uint64_t i = 0; i < n_cells; ++i) {
    const uint64_t cell = ordered ? r.cell_order[i] : i;
    const uint32_t row = (uint32_t)(cell / (uint64_t)r.T);
    const int64_t k = (int64_t)(cell % (uint64_t)r.T);
    if (!r.valid_at(row, k)) continue;
    c_ts->i64.push_back(r.eval_ts[(size_t)k]);
    const size_t at = (size_t)row * (size_t)r.T + (size_t)k;
    for (uint32_t f = 0; f < r.F; ++f) put(c_vals[f], r.types[f], r.field(f)[at]);
    if (c_label) put(c_label, r.counted->type, r.counted->values[at]);
    if (c_tsid) c_tsid->i64.push_back((int64_t)L.ids[row]);
    for (size_t t = 0; t < c_tags.size(); ++t) {
      if (L.id_keyed) {
        c_tags[t]->i64.push_back((int64_t)L.ids[row]);
      } else {
        OwnedColumn* c = c_tags[t];
        const Label& v = L.values[t][row];
        if (!v) {  // a real Arrow null
          if (c->validity.size() <= (size_t)(n_out >> 3)) c->validity.resize((size_t)(n_out >> 3) + 1, 0xFF);
          c->validity[(size_t)n_out >> 3] &= (uint8_t)~(1u << (n_out & 7));
          ++c->nulls;
        } else {
          c->chars += *v;
        }
        c->offsets.push_back((int32_t)c->chars.size());
      }
    }
    ++n_out;
  }

  // ---- wire up the Arrow C structs ------------------------------------------------------------------
  const size_t nc = ob->cols.size();
  ob->child_arrays.resize(nc);
  ob->child_ptrs.resize(nc);
  os->children.resize(nc);
  os->child_ptrs.resize(nc);
  for (size_t i = 0; i < nc; ++i) {
    OwnedColumn* c = ob->cols[i].get();
    ArrowArray& a = ob->child_arrays[i];
    std::memset(&a, 0, sizeof a);
    a.length = n_out;
    a.null_count = 0;
    a.offset = 0;
    const std::string& fmt = os->formats[i];
    if (fmt == "u") {
      if (c->offsets.empty()) c->offsets.push_back(0);
      c->buffers[0] = nullptr;
      if (c->nulls > 0) {
        c->validity.resize((size_t)(n_out + 7) / 8, 0xFF);
        c->buffers[0] = c->validity.data();
        a.null_count = c->nulls;
      }
      c->buffers[1] = c->offsets.data();
      c->buffers[2] = c->chars.data();
      a.n_buffers = 3;
    } else {
      c->buffers[0] = nullptr;
      c->buffers[1] = fmt == "g"   ? static_cast<const void*>(c->f64.data())
                      : fmt == "i" ? static_cast<const void*>(c->i32.data())
                                   : static_cast<const void*>(c->i64.data());
      a.n_buffers = 2;
    }
    a.buffers = c->buffers;
    a.release = release_child_array;
    ob->child_ptrs[i] = &a;
    ArrowSchema& sc = os->children[i];
    std::memset(&sc, 0, sizeof sc);
    sc.format = os->formats[i].c_str();
    sc.name = os->names[i].c_str();
    sc.flags = c->nulls > 0 ? kArrowFlagNullable : 0;
    sc.release = release_child_schema;
    os->child_ptrs[i] = &sc;
  }
  std::memset(out, 0, sizeof *out);
  out->length = n_out;
  out->n_buffers = 1;
  out->buffers = ob->buffers;
  out->n_children = (int64_t)nc;
  out->children = ob->child_ptrs.data();
  out->release = release_batch;
  out->private_data = ob.release();
  std::memset(out_schema, 0, sizeof *out_schema);
  out_schema->format = "+s";
  out_schema->name = "";
  out_schema->n_children = (int64_t)nc;
  out_schema->children = os->child_ptrs.data();
  out_schema->release = release_schema;
  out_schema->private_data = os.release();
}

}  // namespace

// ---- PlanNode ------------------------------------------------------------------------------------------
namespace {

struct FnName {
  const char* name;  // as the reference's projection shows it (ScalarFunctionExpr::name)
  int id;            // enum b2p_ifn
  int min_args, max_args;
};
// planner.rs:2368-2413: DataFusion math builtins under their own names, rad / deg / sgn as radians / degrees / signum,
// round as the prom_round UDF (a missing argument becomes 0.0), clamp* from GreptimeDB's scalar functions
const FnName kInstantFns[] = {
    {"abs", B2P_IFN_ABS, 0, 0},       {"ceil", B2P_IFN_CEIL, 0, 0},     {"floor", B2P_IFN_FLOOR, 0, 0},
    {"sqrt", B2P_IFN_SQRT, 0, 0},     {"exp", B2P_IFN_EXP, 0, 0},       {"ln", B2P_IFN_LN, 0, 0},
    {"log2", B2P_IFN_LOG2, 0, 0},     {"log10", B2P_IFN_LOG10, 0, 0},   {"sin", B2P_IFN_SIN, 0, 0},
    {"cos", B2P_IFN_COS, 0, 0},       {"tan", B2P_IFN_TAN, 0, 0},       {"asin", B2P_IFN_ASIN, 0, 0},
    {"acos", B2P_IFN_ACOS, 0, 0},     {"atan", B2P_IFN_ATAN, 0, 0},     {"sinh", B2P_IFN_SINH, 0, 0},
    {"cosh", B2P_IFN_COSH, 0, 0},     {"tanh", B2P_IFN_TANH, 0, 0},     {"asinh", B2P_IFN_ASINH, 0, 0},
    {"acosh", B2P_IFN_ACOSH, 0, 0},   {"atanh", B2P_IFN_ATANH, 0, 0},   {"prom_round", B2P_IFN_ROUND, 0, 1},
    {"degrees", B2P_IFN_DEG, 0, 0},   {"radians", B2P_IFN_RAD, 0, 0},   {"signum", B2P_IFN_SGN, 0, 0},
    {"clamp", B2P_IFN_CLAMP, 2, 2},   {"clamp_min", B2P_IFN_CLAMP_MIN, 1, 1}, {"clamp_max", B2P_IFN_CLAMP_MAX, 1, 1},
};

// the calendar functions: PromQL name, enum b2p_step_part and the date_part field DataFusion is asked for
// (planner.rs:2222-2300); days_in_month is named after its whole expression (date_part_name)
struct StepFnName {
  const char* name;
  int part;
  const char* field;
};
const StepFnName kStepFns[] = {
    {"minute", B2P_STEP_MINUTE, "minute"},     {"hour", B2P_STEP_HOUR, "hour"},
    {"month", B2P_STEP_MONTH, "month"},        {"year", B2P_STEP_YEAR, "year"},
    {"day_of_month", B2P_STEP_DAY_OF_MONTH, "day"}, {"day_of_week", B2P_STEP_DAY_OF_WEEK, "dow"},
    {"day_of_year", B2P_STEP_DAY_OF_YEAR, "doy"}, {"days_in_month", B2P_STEP_DAYS_IN_MONTH, nullptr},
};

// the value column of a calendar stage as the reference's projection names it over the time index
std::string date_part_name(const Stage& s, const std::string& ti) {
  if (s.part == B2P_STEP_DAYS_IN_MONTH)
    return "date_part(Utf8(\"day\"),date_trunc(Utf8(\"month\")," + ti +
           ") + IntervalYearMonth(\"1\") - IntervalDayTime(\"IntervalDayTime { days: 1, milliseconds: 0 }\"))";
  return "date_part(Utf8(\"" + s.fn_name + "\")," + ti + ")";
}

// an f64 as Rust's Display writes it: the shortest digits that round-trip, never an exponent ("12", "0.5", "inf")
std::string rust_display(double x) {
  if (std::isnan(x)) return "NaN";
  char buf[400];
  const auto res = std::to_chars(buf, buf + sizeof buf, x, std::chars_format::fixed);
  return std::string(buf, res.ptr);
}

}  // namespace

void PlanNode::add_scalar_op(int op, double scalar, bool scalar_on_left, bool return_bool) {
  check_op(op, return_bool);
  Stage s;
  s.op = op;
  s.scalar = scalar;
  s.scalar_on_left = scalar_on_left;
  s.return_bool = return_bool;
  stages_.push_back(s);
}

void PlanNode::add_function(const std::string& name, const std::vector<double>& args) {
  if (name == "negative" || std::any_of(std::begin(kStepFns), std::end(kStepFns), [&](const StepFnName& f) { return name == f.name; })) {
    if (!args.empty()) throw PlanError(ErrorKind::Plan, name + " takes 0 argument(s) after the vector, got " + std::to_string(args.size()));
    Stage s;
    s.is_fn = true;
    s.op = B2P_IFN_NEG;
    s.fn_name = name;
    for (const StepFnName& f : kStepFns)
      if (name == f.name) s.part = f.part, s.fn_name = f.field ? f.field : "";
    stages_.push_back(s);
    return;
  }
  for (const FnName& f : kInstantFns) {
    if (name != f.name) continue;
    const int n = (int)args.size();
    if (n < f.min_args || n > f.max_args)
      throw PlanError(ErrorKind::Plan, name + " takes " + std::to_string(f.min_args) +
                                           (f.max_args != f.min_args ? " or " + std::to_string(f.max_args) : "") +
                                           " argument(s) after the vector, got " + std::to_string(n));
    Stage s;
    s.is_fn = true;
    s.op = f.id;
    s.fn_name = name;
    s.args = args;
    if (f.id == B2P_IFN_ROUND && args.empty()) s.args.push_back(0.0);
    stages_.push_back(s);
    return;
  }
  throw PlanError(ErrorKind::Plan, "unsupported instant-vector function " + name);
}

void PlanNode::require(const char* node, std::initializer_list<const PlanNode*> children, bool device) const {
  if (device && !ctx_) throw PlanError(ErrorKind::Internal, std::string(node) + ": NULL context");
  for (const PlanNode* c : children)
    if (!c) throw PlanError(ErrorKind::Plan, std::string(node) + ": NULL child");
}

bool PlanNode::sharded_run(const char* node) const {
  if (b2p_comm_ranks(ctx_, nullptr) == 0) return false;
  std::vector<const PlanNode*> todo = children();
  while (!todo.empty()) {
    const PlanNode* n = todo.back();
    todo.pop_back();
    if (n->sharded_)
      throw PlanError(ErrorKind::Plan, std::string(node) + ": a sharded node below a sharded node: its result is "
                                                           "already on every rank, and merging it again would count every copy");
    if (const char* what = n->cross_row())
      throw PlanError(ErrorKind::Plan, std::string(node) + ": a sharded node over " + what + ", which computes over rows "
                                                           "other ranks hold: its result on one rank is not the query's");
    for (const PlanNode* c : n->children()) todo.push_back(c);
  }
  return true;
}

void PlanNode::run(NodeResult& r) {
  compute(r);
  for (const Stage& s : stages_) {
    const bool work = r.rows > 0 && r.T > 0;
    if (s.part >= 0) {
      // a calendar function: one date_part projection over the time index whatever the node's fields, typed Int32
      // (DataFusion's date_part width; not in the reference tree), labels and validity kept (K19)
      r.F = 1;
      r.val.resize(r.grid());
      if (work)
        check(b2p_step_fn(ctx_, s.part, r.eval_ts.data(), r.valid.data(), r.rows, (uint64_t)r.T, r.field(0)));
      r.types = {ValueType::Int32};
      r.value_names = {date_part_name(s, r.time_index)};
      r.labels.drop_tsid();  // a projection of time, value and tags (planner.rs:1055-1058)
      continue;
    }
    const bool filter = !s.is_fn && is_comparison(s.op) && !s.return_bool;
    if (s.is_fn && s.op == B2P_IFN_NEG && (r.has(ValueType::Int64) || r.has(ValueType::Int32)))  // integer negation and its overflow
      throw PlanError(ErrorKind::Plan, "unary minus over an integer value column is not supported by this node");
    // an Int64 value column under a stage: a filter would keep the Int64 column, which the reference tree does not
    // pin; a projection reads it as Float64 (DataFusion's coercion against the Float64 literal or function)
    if (filter && r.has(ValueType::Int64))
      throw PlanError(ErrorKind::Plan, "a filtering comparison over an Int64 value column is not supported by this node");
    // a filter keeps an Int32 (calendar) column; every other stage's result, and a filter's over a count, is Float64
    for (uint32_t f = 0; f < r.F; ++f)
      if (!(filter && r.types[f] == ValueType::Int32)) field_to_f64(ctx_, r, f);
    if (s.is_fn) {
      // as a calendar stage; unary minus, arithmetic, `bool` and filters keep it: projection_for_each_field_column
      // (planner.rs:543-553, 3926-3955)
      if (s.op != B2P_IFN_NEG) r.labels.drop_tsid();
      const double a0 = s.args.size() > 0 ? s.args[0] : 0.0, a1 = s.args.size() > 1 ? s.args[1] : 0.0;
      // clamp's bound check (clamp.rs:212-217); clamp_min / clamp_max meet the other bound at ±f64::MAX.  The reference
      // checks inside the function's invoke, once per input batch, so a node without rows gives no error
      const double lo = s.op == B2P_IFN_CLAMP_MAX ? -DBL_MAX : a0;
      const double hi = s.op == B2P_IFN_CLAMP ? a1 : s.op == B2P_IFN_CLAMP_MIN ? DBL_MAX : a0;
      const bool has_rows = std::any_of(r.valid.begin(), r.valid.end(), [](uint32_t w) { return w != 0; });
      if (s.op >= B2P_IFN_CLAMP && lo > hi && has_rows)
        throw PlanError(ErrorKind::Execution, "min '" + rust_display(lo) + "' > max '" + rust_display(hi) + "'");
      // once per field (planner.rs:2416); a function keeps every bit, so the fields share the bitmap
      for (uint32_t f = 0; f < r.F && work; ++f)
        check(b2p_instant_fn(ctx_, s.op, a0, a1, r.field(f), r.valid.data(), r.rows, (uint64_t)r.T, r.field(f),
                             r.valid.data()));
      for (std::string& value : r.value_names) {
        if (s.op == B2P_IFN_NEG) {
          value = "(- " + value + ")";
          continue;
        }
        std::string name = s.fn_name + "(" + value;
        for (double a : s.args) name += "," + float_literal(a);
        value = name + ")";
      }
      continue;
    }
    if (filter && r.F > 1)  // planner.rs:3976-3981
      throw PlanError(ErrorKind::Plan, "Unsupported expr type: filter on multi-value input");
    for (uint32_t f = 0; f < r.F && work; ++f)  // arithmetic and `bool` keep every bit (planner.rs:3930-3960)
      check(b2p_scalar_op(ctx_, s.op, s.return_bool ? 1 : 0, s.scalar_on_left ? 1 : 0, s.scalar, r.field(f),
                          r.valid.data(), r.rows, (uint64_t)r.T, r.field(f), r.valid.data()));
    if (!filter) {  // a projection names its expression; a filter keeps the column
      const std::string lit = float_literal(s.scalar), sym = kOpSymbols[s.op];
      for (std::string& value : r.value_names)
        value = s.scalar_on_left ? lit + " " + sym + " " + value : value + " " + sym + " " + lit;
    }
  }
}

void PlanNode::execute(ArrowArray* out, ArrowSchema* out_schema) {
  if (!out || !out_schema) throw PlanError(ErrorKind::Internal, "execute: NULL output structs");
  NodeResult r;
  run(r);
  export_result(r, out, out_schema);
}

// ---- BinaryPlan ----------------------------------------------------------------------------------------
BinaryPlan::BinaryPlan(b2p_ctx* ctx, int op, bool return_bool, std::shared_ptr<PlanNode> lhs,
                       std::shared_ptr<PlanNode> rhs, Matching matching, std::vector<std::string> labels,
                       bool labels_from_lhs)
    : PlanNode(ctx), op_(op), return_bool_(return_bool), lhs_(std::move(lhs)), rhs_(std::move(rhs)),
      matching_(matching), labels_(std::move(labels)), labels_from_lhs_(labels_from_lhs) {
  require("GpuPromBinaryExec", {lhs_.get(), rhs_.get()});
  check_op(op_, return_bool_);
}

void BinaryPlan::compute(NodeResult& r) {
  NodeResult L, R;
  lhs_->run(L);
  rhs_->run(R);
  if (L.T != R.T) throw PlanError(ErrorKind::Plan, "both sides of a binary operator must be evaluated on the same steps");
  // `scalar cmp vector`: the reference filters the vector and keeps its rows, labels, values and time index
  // (planner.rs:765-771, project_binary_join_side on the right).  time() is scalar-typed, so it is evaluated as
  // `vector cmp' scalar` with the mirrored comparison; an EmptyMetric literal may be vector(s), whose matching this
  // layer does not model there, so that shape is refused.
  int op = op_;
  if (is_comparison(op_) && !return_bool_ && !R.scalar_like && !R.literal_row) {
    if (L.literal_row)
      throw PlanError(ErrorKind::Plan, "GpuPromBinaryExec: a filtering comparison with a literal EmptyMetric lhs against a vector is not supported by this node");
    if (L.scalar_like) {
      std::swap(L, R);
      op = op_ == B2P_OP_GT ? B2P_OP_LT : op_ == B2P_OP_LT ? B2P_OP_GT : op_ == B2P_OP_GE ? B2P_OP_LE
           : op_ == B2P_OP_LE ? B2P_OP_GE : op_;  // (== and != are symmetric)
    }
  }
  // Int64 operands: against a Float64 side DataFusion coerces to Float64; between two Int64 sides it would run integer
  // arithmetic, division and overflow, which the reference tree does not pin, and a filter would keep the Int64 column
  for (uint32_t f = 0; f < std::min(L.F, R.F); ++f)
    if (L.is(f, ValueType::Int64) && R.is(f, ValueType::Int64))
      throw PlanError(ErrorKind::Plan, "GpuPromBinaryExec: a binary operator between two Int64 value columns is not supported by this node");
  // an Int32 (calendar) side meets a Float64 side only: DataFusion's integer result types are not pinned here
  if (L.has(ValueType::Int32) ? R.has(ValueType::Int32) || R.has(ValueType::Int64) : R.has(ValueType::Int32) && L.has(ValueType::Int64))
    throw PlanError(ErrorKind::Plan, "GpuPromBinaryExec: a binary operator between two integer value columns is not supported by this node");
  const bool filter = is_comparison(op) && !return_bool_;
  if (filter && L.has(ValueType::Int64))
    throw PlanError(ErrorKind::Plan, "a filtering comparison over an Int64 value column is not supported by this node");
  const std::vector<ValueType> lhs_types = L.types;  // a filter keeps the lhs column and its type
  to_f64(ctx_, L);
  to_f64(ctx_, R);
  // join keys (planner.rs:696-729, 3436-3468): the rhs context's tag columns, narrowed by on / ignoring; none when a
  // side has no tags (every row pairs with every row); two id-keyed sides, or two sides that carry __tsid, without a
  // modifier join on the id (binary_join_key_columns: without on / ignoring the match is one-to-one)
  std::vector<int> lcols, rcols;
  const bool by_tsid = L.labels.tsid && R.labels.tsid && matching_ == Matching::None;
  const bool by_id = by_tsid || (L.labels.id_keyed && R.labels.id_keyed && matching_ == Matching::None);
  auto row_key = [&](const Labels& labels, uint32_t q, const std::vector<int>& cols, std::string& key) {
    if (by_tsid) key.assign(reinterpret_cast<const char*>(&labels.ids[q]), sizeof(uint64_t));
    else labels.key(q, cols, key);
  };
  if (by_id) {
    lcols.push_back(0);
    rcols.push_back(0);
  } else if (!L.labels.names.empty() && !R.labels.names.empty()) {
    const std::vector<std::string> names = narrow_tags(R.labels.names, matching_, labels_);
    lcols = L.labels.columns(names);
    rcols = R.labels.columns(names);
    for (size_t i = 0; i < names.size(); ++i)
      if (lcols[i] < 0) throw PlanError(ErrorKind::Plan, "No field named " + names[i]);
  }
  // hash join of the series: rhs rows by key (in row order), then every lhs row in order against its key's rhs rows
  std::unordered_map<std::string, std::vector<uint32_t>> rhs_by_key;
  std::string key;
  rhs_by_key.reserve(R.rows);
  for (uint32_t q = 0; q < R.rows; ++q) {
    row_key(R.labels, q, rcols, key);
    rhs_by_key[key].push_back(q);
  }
  std::vector<uint32_t> lrow, rrow;
  for (uint32_t q = 0; q < L.rows; ++q) {
    row_key(L.labels, q, lcols, key);
    const auto it = rhs_by_key.find(key);
    if (it == rhs_by_key.end()) continue;
    for (uint32_t m : it->second) {
      lrow.push_back(q);
      rrow.push_back(m);
    }
  }
  const uint64_t n_pairs = lrow.size();
  if (n_pairs > UINT32_MAX) throw PlanError(ErrorKind::Plan, "GpuPromBinaryExec: more than 2^32 - 1 matched series pairs");
  // the fields zip pairwise, field i with field i (align_binary_field_columns, planner.rs:3401-3414); a filter decides
  // on its one pair and keeps every field of the lhs
  const uint32_t pairs = std::min(L.F, R.F);
  if (filter && pairs > 1) throw PlanError(ErrorKind::Plan, "Unsupported expr type: filter on multi-value input");
  r = NodeResult();
  r.T = L.T;
  r.Tw = L.Tw;
  r.rows = (uint32_t)n_pairs;
  r.F = filter ? L.F : pairs;
  r.types = filter ? lhs_types : std::vector<ValueType>(pairs, ValueType::Float64);
  r.eval_ts = L.eval_ts;
  r.val.assign((size_t)r.F * n_pairs * (size_t)r.T, 0.0);
  r.valid.assign((size_t)n_pairs * r.Tw, 0u);
  for (uint32_t f = 0; f < pairs && n_pairs > 0 && r.T > 0; ++f)  // arithmetic and `bool` keep the join's bits
    check(b2p_binary_op(ctx_, op, return_bool_ ? 1 : 0, L.field(f), L.valid.data(), lrow.data(), L.rows, R.field(f),
                        R.valid.data(), rrow.data(), R.rows, n_pairs, (uint64_t)r.T, r.field(f), r.valid.data()));
  // the lhs's other fields at the cells the comparison kept; a dropped cell holds 0.0, as the kernel writes it
  for (uint32_t f = 1; filter && f < r.F; ++f)
    for (uint64_t q = 0; q < n_pairs; ++q) {
      const double* src = L.field(f) + (size_t)lrow[q] * (size_t)r.T;
      double* dst = r.field(f) + (size_t)q * (size_t)r.T;
      for (int64_t k = 0; k < r.T; ++k)
        if (r.valid_at((uint32_t)q, k)) dst[k] = src[k];
    }
  // output labels: a filter passes the lhs rows through; a projection emits the tag columns of `label_side`; either
  // keeps that side's __tsid (project_binary_join_side, projection_for_each_field_column, planner.rs:779-838, 3926-3955)
  const bool from_lhs = filter || labels_from_lhs_;
  const NodeResult& side = from_lhs ? L : R;
  const std::vector<uint32_t>& srow = from_lhs ? lrow : rrow;
  r.time_index = side.time_index;
  r.labels = side.labels.gather(srow);
  if (filter) {
    r.columns = L.columns;
    r.value_names = L.value_names;
    if (L.counted) {  // the kept rows' counted values
      r.counted = CountedColumn{L.counted->name, L.counted->type, std::vector<double>((size_t)n_pairs * (size_t)r.T)};
      for (uint64_t p = 0; p < n_pairs; ++p)
        std::copy_n(L.counted->values.begin() + (size_t)lrow[p] * (size_t)r.T, (size_t)r.T,
                    r.counted->values.begin() + (size_t)p * (size_t)r.T);
    }
  } else {
    r.columns = Columns::TagsTimeValue;
    for (uint32_t f = 0; f < r.F; ++f)
      r.value_names.push_back(L.value_names[f] + " " + kOpSymbols[op] + " " + R.value_names[f]);
  }
}

// ---- SetOpPlan -----------------------------------------------------------------------------------------
namespace {

const char* const kSetNames[] = {"and", "or", "unless"};

// left.distinct() of `and` / `unless` (planner.rs:3549-3703): a cell whose labels, step and value bits (DataFusion's
// group equality on f64) equal those of a cell of an earlier row is dropped.  Only rows that share a label tuple can
// hold such cells, so only they are compared.  A counted value is a column of the row too.
void drop_duplicate_cells(NodeResult& n) {
  if (n.rows < 2 || n.T == 0) return;
  std::vector<int> all(n.labels.names.size());
  std::iota(all.begin(), all.end(), 0);
  std::unordered_map<std::string, std::vector<uint32_t>> by_labels;
  std::string key;
  for (uint32_t q = 0; q < n.rows; ++q) {
    n.labels.key(q, all, key);
    by_labels[key].push_back(q);
  }
  for (const auto& kv : by_labels) {
    const std::vector<uint32_t>& g = kv.second;
    for (size_t i = 1; i < g.size(); ++i)
      for (int64_t k = 0; k < n.T; ++k) {
        if (!n.valid_at(g[i], k)) continue;
        const double x = n.val[(size_t)g[i] * (size_t)n.T + (size_t)k];
        for (size_t j = 0; j < i; ++j) {
          const double y = n.val[(size_t)g[j] * (size_t)n.T + (size_t)k];
          const size_t a = (size_t)g[i] * (size_t)n.T + (size_t)k, b = (size_t)g[j] * (size_t)n.T + (size_t)k;
          if (n.valid_at(g[j], k) && std::memcmp(&x, &y, sizeof x) == 0 &&
              (!n.counted || std::memcmp(&n.counted->values[a], &n.counted->values[b], sizeof(double)) == 0)) {
            n.valid[(size_t)g[i] * n.Tw + (size_t)(k >> 5)] &= ~(1u << (k & 31));
            n.val[(size_t)g[i] * (size_t)n.T + (size_t)k] = 0.0;
            break;
          }
        }
      }
  }
}

}  // namespace

SetOpPlan::SetOpPlan(b2p_ctx* ctx, int op, std::shared_ptr<PlanNode> lhs, std::shared_ptr<PlanNode> rhs,
                     Matching matching, std::vector<std::string> labels)
    : PlanNode(ctx), op_(op), lhs_(std::move(lhs)), rhs_(std::move(rhs)), matching_(matching), labels_(std::move(labels)) {
  require("GpuPromSetOpExec", {lhs_.get(), rhs_.get()});
  if (op_ < B2P_SET_AND || op_ > B2P_SET_UNLESS) throw PlanError(ErrorKind::Plan, "unknown set operator " + std::to_string(op_));
}

void SetOpPlan::compute(NodeResult& r) {
  NodeResult L, R;
  lhs_->run(L);
  rhs_->run(R);
  const std::string what = std::string("set operator `") + kSetNames[op_] + "`: ";
  // planner.rs:3656-3661 (`and` and `unless` both name it the AND operator), 3718-3730
  if (op_ == B2P_SET_OR && L.F != R.F) {
    auto list = [](const std::vector<std::string>& v) {
      std::string out;
      for (const std::string& x : v) out += (out.empty() ? "\"" : ", \"") + x + "\"";
      return "[" + out + "]";
    };
    throw PlanError(ErrorKind::Plan, "Attempt to combine two tables with different column sets, left: " +
                                         list(L.value_names) + ", right: " + list(R.value_names));
  }
  // `and` / `unless` keep the lhs column and its type; `or` over an Int64 side is not pinned by the reference tree
  if (op_ == B2P_SET_OR && (L.has(ValueType::Int64) || R.has(ValueType::Int64)))
    throw PlanError(ErrorKind::Plan, what + "an Int64 value column is not supported by this node");
  if (op_ == B2P_SET_OR && L.has(ValueType::Int32) != R.has(ValueType::Int32))  // `or` of Int32 with Int32 stays Int32
    throw PlanError(ErrorKind::Plan, what + "an Int32 value column against another type is not supported by this node");
  if (L.F > 1)
    throw PlanError(ErrorKind::Plan, std::string("Multi fields calculation is not supported in ") +
                                         (op_ == B2P_SET_OR ? "OR operator" : "AND operator"));
  if (L.T != R.T || (L.rows > 0 && R.rows > 0 && L.eval_ts != R.eval_ts))
    throw PlanError(ErrorKind::Plan, what + "both sides must be evaluated on the same steps");
  // the reference matches set operators on label values (planner.rs:3626-3630), which an id-keyed node does not carry
  if (L.labels.id_keyed || R.labels.id_keyed) throw PlanError(ErrorKind::Plan, what + "an id-keyed (__tsid) side has no label values to match");
  const int64_t T = L.T;
  std::vector<std::string> names;  // match columns
  std::vector<std::string> all;    // `or`: the union of both sides' tags, sorted
  if (op_ != B2P_SET_OR) {
    // each side's tags narrowed by on / ignoring; the two key sets must be equal (CombineTableColumnMismatch)
    names = narrow_tags(L.labels.names, matching_, labels_);
    std::vector<std::string> rn = narrow_tags(R.labels.names, matching_, labels_);
    std::sort(names.begin(), names.end());
    std::sort(rn.begin(), rn.end());
    if (names != rn) {
      auto list = [](const std::vector<std::string>& v) {
        std::string s;
        for (const std::string& x : v) s += (s.empty() ? "" : ", ") + x;
        return "[" + s + "]";
      };
      throw PlanError(ErrorKind::Plan, what + "the key columns of the two sides differ: " + list(names) + " vs " + list(rn));
    }
  } else {
    all = L.labels.names;
    all.insert(all.end(), R.labels.names.begin(), R.labels.names.end());
    std::sort(all.begin(), all.end());
    all.erase(std::unique(all.begin(), all.end()), all.end());
    if (matching_ == Matching::On) {
      names = labels_;
      for (const std::string& l : names)
        if (!std::binary_search(all.begin(), all.end(), l)) throw PlanError(ErrorKind::Plan, what + "Column " + l + " not found");
    } else {
      names = narrow_tags(all, matching_, labels_);
    }
  }
  const std::vector<int> lcols = L.labels.columns(names), rcols = R.labels.columns(names);
  KeyIds keys;
  std::vector<uint32_t> lkey(L.rows), rkey(R.rows);
  std::string key;
  if (op_ == B2P_SET_OR) {
    for (uint32_t q = 0; q < L.rows; ++q) {
      L.labels.key(q, lcols, key);
      lkey[q] = keys.add(key);
    }
  }
  for (uint32_t q = 0; q < R.rows; ++q) {
    R.labels.key(q, rcols, key);
    rkey[q] = keys.add(key);
  }
  if (op_ != B2P_SET_OR) {
    for (uint32_t q = 0; q < L.rows; ++q) {
      L.labels.key(q, lcols, key);
      lkey[q] = keys.find(key);
    }
    drop_duplicate_cells(L);
    if (L.rows > 0 && T > 0)
      check(b2p_setop(ctx_, op_, L.val.data(), L.valid.data(), lkey.data(), L.rows, nullptr, R.valid.data(),
                            rkey.data(), R.rows, (uint32_t)keys.ids.size(), (uint64_t)T, L.val.data(), L.valid.data()));
    r = std::move(L);  // the lhs rows, columns and values
    return;
  }
  // or: the lhs rows, then the rhs rows, over the union of the tags (NULL where a side lacks one)
  const uint64_t n = (uint64_t)L.rows + R.rows;
  if (n > UINT32_MAX) throw PlanError(ErrorKind::Plan, what + "more than 2^32 - 1 rows");
  r = NodeResult();
  r.T = T;
  r.Tw = L.Tw;
  r.rows = (uint32_t)n;
  r.eval_ts = L.rows > 0 ? L.eval_ts : R.eval_ts;
  r.val.assign((size_t)n * (size_t)T, 0.0);
  r.valid.assign((size_t)n * r.Tw, 0u);
  if (n > 0 && T > 0)
    check(b2p_setop(ctx_, op_, L.val.data(), L.valid.data(), lkey.data(), L.rows, R.val.data(), R.valid.data(),
                          rkey.data(), R.rows, (uint32_t)keys.ids.size(), (uint64_t)T, r.val.data(), r.valid.data()));
  r.time_index = L.time_index;
  r.value_names = L.value_names;
  r.types = {L.has(ValueType::Int32) ? ValueType::Int32 : ValueType::Float64};  // (a count is Float64 here)
  r.columns = Columns::TimeSorted;
  r.labels.names = all;
  r.labels.values.resize(all.size());
  const std::vector<int> lall = L.labels.columns(all), rall = R.labels.columns(all);
  for (size_t t = 0; t < all.size(); ++t) {
    r.labels.values[t].reserve((size_t)n);
    for (uint32_t q = 0; q < L.rows; ++q) r.labels.values[t].push_back(L.labels.value(lall[t], q));
    for (uint32_t q = 0; q < R.rows; ++q) r.labels.values[t].push_back(R.labels.value(rall[t], q));
  }
  // __tsid only when both sides carry it (planner.rs:3776-3800, 3903); `and` / `unless` keep the lhs's (3632)
  if (L.labels.tsid && R.labels.tsid) {
    r.labels.tsid = true;
    r.labels.ids = L.labels.ids;
    r.labels.ids.insert(r.labels.ids.end(), R.labels.ids.begin(), R.labels.ids.end());
  }
}

// ---- ScalarPlan ----------------------------------------------------------------------------------------
ScalarPlan::ScalarPlan(b2p_ctx* ctx, std::shared_ptr<PlanNode> child) : PlanNode(ctx), child_(std::move(child)) {
  require("GpuPromScalarExec", {child_.get()});
}

void ScalarPlan::compute(NodeResult& r) {
  NodeResult C;
  child_->run(C);
  check_child(C, {{Shape::Int32, "GpuPromScalarExec: an Int32 value column is not supported by this node"},
                  {Shape::MultiField, "Multi fields calculation is not supported in scalar"}});  // planner.rs:3155-3160
  to_f64(ctx_, C);  // scalar() of an Int64 node is Float64
  // one dense key per label tuple over the child's tag columns (a tagless child is one series, an id-keyed one is keyed
  // by the id); a tuple with a NULL label gets B2P_NO_KEY (scalar_calculate.rs:543-569 compares NULL as None against
  // the "" it recorded)
  std::vector<uint32_t> key(C.rows, 0u);
  if (!C.labels.names.empty()) {
    KeyIds ids;
    std::vector<int> all(C.labels.names.size());
    std::iota(all.begin(), all.end(), 0);
    std::string k;
    for (uint32_t q = 0; q < C.rows; ++q) {
      const bool null_label = std::any_of(C.labels.values.begin(), C.labels.values.end(),
                                          [&](const std::vector<Label>& col) { return !col[q]; });
      C.labels.key(q, all, k);
      key[q] = null_label ? B2P_NO_KEY : ids.add(k);
    }
  }
  r = NodeResult();
  r.T = C.T;
  r.Tw = C.Tw;
  r.rows = 1;
  r.eval_ts = C.eval_ts;
  r.time_index = C.time_index;
  r.value_names = {"scalar(" + C.value_names[0] + ")"};
  r.val.assign((size_t)r.T, 0.0);
  r.valid.assign((size_t)r.Tw, 0u);
  if (r.T > 0)  // two rows of one series with a cell at the same step are bad data here, not a bad plan
    check(b2p_scalar_calculate(ctx_, C.val.data(), C.valid.data(), key.data(), C.rows, (uint64_t)r.T, r.val.data(),
                               r.valid.data()),
          ErrorKind::Execution);
}

// ---- TopkPlan ------------------------------------------------------------------------------------------
namespace {
int64_t total_key_host(double x) {  // f64::total_cmp's key
  int64_t b;
  std::memcpy(&b, &x, sizeof b);
  return b ^ (int64_t)((uint64_t)(b >> 63) >> 1);
}

// The columns of L an aggregation groups by (agg_modifier_to_col, planner.rs:1400-1480): `by` the listed labels L has,
// in the listed order; `without` L's tags that are not listed, in name order; none: no column (the time index alone)
std::vector<int> group_columns(const Labels& L, Modifier modifier, const std::vector<std::string>& labels) {
  std::vector<std::string> names;
  if (modifier == Modifier::By) {
    for (const std::string& l : labels)
      if (L.column(l) >= 0) names.push_back(l);
  } else if (modifier == Modifier::Without) {
    names = narrow_tags(L.names, Matching::Ignoring, labels);
    std::sort(names.begin(), names.end());
  }
  return L.columns(names);
}
}  // namespace

TopkPlan::TopkPlan(b2p_ctx* ctx, bool bottom, double k, std::shared_ptr<PlanNode> child, Modifier modifier,
                   std::vector<std::string> labels)
    : PlanNode(ctx), bottom_(bottom), k_(k), child_(std::move(child)), modifier_(modifier), labels_(std::move(labels)) {
  require("GpuPromTopkExec", {child_.get()});
}

void TopkPlan::compute(NodeResult& r) {
  child_->run(r);
  // planner.rs:2969-2974; the window orders ties by the label values (planner.rs:2980-2996), which an id-keyed node
  // does not carry
  check_child(r, {{Shape::MultiField, "Unsupported expr type: topk or bottomk on multi-value input"},
                  {Shape::IdKeyed, std::string(bottom_ ? "bottomk: " : "topk: ") +
                                       "an id-keyed (__tsid) child has no label values to order by"}});
  const Labels& L = r.labels;
  const std::vector<int> gcols = group_columns(L, modifier_, labels_);
  KeyIds groups;
  std::vector<uint32_t> gid(r.rows);
  std::string key;
  for (uint32_t q = 0; q < r.rows; ++q) {
    L.key(q, gcols, key);
    gid[q] = groups.add(key);
  }
  // the tie ordinal: rows ranked by their tuple as the window orders them after the value (every tag in column order,
  // descending for topk and ascending for bottomk, NULL first); identical tuples in row order.  Larger is better for
  // topk, smaller for bottomk, as b2p_topk compares (value, tie).
  auto tuple_before = [&](uint32_t a, uint32_t b) {  // a ranks before b
    for (const std::vector<Label>& col : L.values) {
      const Label &x = col[a], &y = col[b];
      if (x == y) continue;
      if (!x || !y) return !x;  // NULL first
      return bottom_ ? *x < *y : *x > *y;
    }
    return a < b;
  };
  std::vector<uint32_t> order(r.rows);
  std::iota(order.begin(), order.end(), 0u);
  std::sort(order.begin(), order.end(), tuple_before);
  std::vector<uint32_t> tie(r.rows);
  for (uint32_t p = 0; p < r.rows; ++p) tie[order[p]] = bottom_ ? p : r.rows - 1 - p;
  if (r.rows > 0 && r.T > 0)
    check(r.is(0, ValueType::Int64) ? b2p_topk_i64(ctx_, bottom_ ? 1 : 0, k_, reinterpret_cast<const int64_t*>(r.val.data()),
                                     r.valid.data(), gid.data(), r.rows, (uint32_t)groups.ids.size(), tie.data(),
                                     (uint64_t)r.T, r.valid.data())
                      : b2p_topk(ctx_, bottom_ ? 1 : 0, k_, r.val.data(), r.valid.data(), gid.data(), r.rows,
                                 (uint32_t)groups.ids.size(), tie.data(), (uint64_t)r.T, r.valid.data()));
  // export order (Sort(group labels, ts, rank)): group labels by Labels::less, then the step, then the rank
  r.cell_order.clear();
  for (uint32_t q = 0; q < r.rows; ++q)
    for (int64_t k = 0; k < r.T; ++k)
      if (r.valid_at(q, k)) r.cell_order.push_back((uint64_t)q * (uint64_t)r.T + (uint64_t)k);
  const uint64_t T = (uint64_t)r.T;
  std::sort(r.cell_order.begin(), r.cell_order.end(), [&](uint64_t a, uint64_t b) {
    const uint32_t ra = (uint32_t)(a / T), rb = (uint32_t)(b / T);
    for (int c : gcols) {
      const Label &x = L.values[(size_t)c][ra], &y = L.values[(size_t)c][rb];
      if (x != y) return Labels::less(x, y);
    }
    const uint64_t ka = a % T, kb = b % T;
    if (ka != kb) return ka < kb;
    const bool i64 = r.is(0, ValueType::Int64);  // (an Int64 value compares as the integer its bits are)
    const int64_t va = i64 ? bits_i64(r.val[a]) : total_key_host(r.val[a]);
    const int64_t vb = i64 ? bits_i64(r.val[b]) : total_key_host(r.val[b]);
    if (va != vb) return bottom_ ? va < vb : va > vb;
    return bottom_ ? tie[ra] < tie[rb] : tie[ra] > tie[rb];
  });
  // topk's layout: the rows, and a counted column, stay the child's; a count is exported as Float64
  r.columns = Columns::ValueTagsTime;
  if (r.is(0, ValueType::Count)) r.types[0] = ValueType::Float64;
}

// ---- AggregatePlan -------------------------------------------------------------------------------------
AggregatePlan::AggregatePlan(b2p_ctx* ctx, const std::string& op, double param, std::shared_ptr<PlanNode> child,
                             Modifier modifier, std::vector<std::string> labels)
    : PlanNode(ctx), param_(param), child_(std::move(child)), modifier_(modifier), labels_(std::move(labels)) {
  require("GpuPromAggregateExec", {child_.get()});
  // create_aggregate_exprs, planner.rs:2808-2897: the DataFusion function each aggregator becomes
  if (op == "count_values") throw PlanError(ErrorKind::Plan, "GpuPromAggregateExec: count_values is not supported by this node");
  if (op == "topk" || op == "bottomk")
    throw PlanError(ErrorKind::Plan, "GpuPromAggregateExec: " + op + " is a filter, not an aggregate: use b2p_plan_topk_create");
  op_ = op == "group" ? kAggGroup : op == "quantile" ? kAggQuantile : aggregate_id_from_name(op);
  if (op_ < 0) throw PlanError(ErrorKind::Plan, "GpuPromAggregateExec: unknown aggregator " + op);
  df_name_ = op == "stddev" ? "stddev_pop" : op == "stdvar" ? "var_pop" : op;
}

void AggregatePlan::compute(NodeResult& r) {
  const bool sharded = sharded_ && sharded_run("GpuPromAggregateExec");
  child_->run(r);
  // the reference would re-attach the tag columns of an id-keyed input (ensure_tag_columns_available); this layer has
  // only the id, so it can group such a node as a whole and nothing else.  group(): planner.rs:2815-2823
  check_child(r, {{Shape::Int32, "GpuPromAggregateExec: an Int32 value column is not supported by this node"},
                  {Shape::IdKeyed, modifier_ == Modifier::None ? "" : "GpuPromAggregateExec: an id-keyed (__tsid) child can only be aggregated without by / without"},
                  {Shape::MultiField, op_ == kAggGroup ? "Multi fields calculation is not supported in group()" : ""}});
  aggregate_rows(ctx_, op_, param_, group_columns(r.labels, modifier_, labels_), r, sharded);  // one aggregate per field
  for (std::string& value : r.value_names)
    value = op_ == kAggGroup      ? "max(" + float_literal(1.0) + ")"
            : op_ == kAggQuantile ? "quantile(" + float_literal(param_) + "," + value + ")"
                                  : df_name_ + "(" + value + ")";
}

// ---- CountValuesPlan -----------------------------------------------------------------------------------
CountValuesPlan::CountValuesPlan(b2p_ctx* ctx, std::string label, std::shared_ptr<PlanNode> child, Modifier modifier,
                                 std::vector<std::string> labels)
    : PlanNode(ctx), label_(std::move(label)), child_(std::move(child)), modifier_(modifier), labels_(std::move(labels)) {
  require("GpuPromCountValuesExec", {child_.get()});
}

void CountValuesPlan::compute(NodeResult& r) {
  const bool sharded = sharded_ && sharded_run("GpuPromCountValuesExec");
  child_->run(r);
  // planner.rs:2874-2879; keep_tsid is false for count_values (planner.rs:402): as for AggregatePlan, an id-keyed
  // child groups as a whole only
  check_child(r, {{Shape::Int32, "GpuPromCountValuesExec: an Int32 value column is not supported by this node"},
                  {Shape::MultiField, "Unsupported expr type: count_values on multi-value input"},
                  {Shape::IdKeyed, modifier_ == Modifier::None ? "" : "GpuPromCountValuesExec: an id-keyed (__tsid) child can only be counted without by / without"}});
  const std::vector<int> cols = group_columns(r.labels, modifier_, labels_);
  const std::string count_name = "count(" + r.value_names[0] + ")";
  // the projection would have two columns of one name (planner.rs:425-430)
  bool clash = label_ == r.time_index || label_ == count_name;
  for (int c : cols) clash = clash || r.labels.names[(size_t)c] == label_;
  if (clash) throw PlanError(ErrorKind::Plan, "GpuPromCountValuesExec: the label \"" + label_ + "\" names another column of the result");
  Groups groups = group_rows(r.labels, cols, r.rows);
  uint64_t cap = 0;  // sharded: the rows of every rank, which bound the merged rows
  if (sharded) {
    Agreement a = agree_groups(ctx_, groups, r);
    cap = a.n_rows;
    take_global(groups, a);
  }
  const uint32_t G = (uint32_t)groups.rank.size(), R = r.rows, Tw = r.Tw;
  const size_t T = (size_t)r.T;
  const bool i64 = r.is(0, ValueType::Int64);
  // b2p_count_values' rows: group g's members (rank rows) from goff[g]; sharded, the merged rows of group g from goff[g]
  std::vector<uint32_t> goff((size_t)G + 1, 0u), place(G);
  std::vector<double> cval((sharded ? cap : R) * T);
  std::vector<uint32_t> ccnt(cval.size());
  if (sharded) {
    check(i64 ? b2p_count_values_allgather_i64(ctx_, reinterpret_cast<const int64_t*>(r.val.data()), r.valid.data(),
                                               groups.id.data(), R, G, (uint64_t)T, cap, goff.data(),
                                               reinterpret_cast<int64_t*>(cval.data()), ccnt.data())
              : b2p_count_values_allgather(ctx_, r.val.data(), r.valid.data(), groups.id.data(), R, G, (uint64_t)T,
                                           cap, goff.data(), cval.data(), ccnt.data()),
          ErrorKind::Execution);
  } else {
    if (R > 0 && T > 0)
      check(i64 ? b2p_count_values_i64(ctx_, reinterpret_cast<const int64_t*>(r.val.data()), r.valid.data(),
                                       groups.id.data(), R, G, (uint64_t)T, reinterpret_cast<int64_t*>(cval.data()),
                                       ccnt.data())
                : b2p_count_values(ctx_, r.val.data(), r.valid.data(), groups.id.data(), R, G, (uint64_t)T, cval.data(),
                                   ccnt.data()),
            ErrorKind::Execution);
    for (uint32_t q = 0; q < R; ++q) ++goff[groups.id[q] + 1];
    std::partial_sum(goff.begin(), goff.end(), goff.begin());
  }
  // the counted values keep the child's type (count_values.result:31-62)
  r.counted = CountedColumn{label_, i64 ? ValueType::Int64 : ValueType::Float64, {}};
  r.types = {ValueType::Count};
  for (uint32_t g = 0; g < G; ++g) place[groups.rank[g]] = g;
  // output rows: the groups in label order, each with its rank rows that hold a value at some step
  std::vector<uint32_t> src, lab, first(1, 0u);
  for (uint32_t p = 0; p < G; ++p) {
    for (uint32_t q = goff[place[p]]; q < goff[place[p] + 1]; ++q) {
      if (!std::any_of(ccnt.begin() + (size_t)q * T, ccnt.begin() + (size_t)(q + 1) * T, [](uint32_t n) { return n != 0; }))
        break;  // ranks are dense: no later rank has a value either
      src.push_back(q);
      lab.push_back(p);
    }
    first.push_back((uint32_t)src.size());
  }
  const uint32_t n = (uint32_t)src.size();
  r.labels = groups.labels.gather(lab);
  r.val.assign((size_t)n * T, 0.0);
  r.valid.assign((size_t)n * Tw, 0u);
  r.counted->values.assign((size_t)n * T, 0.0);
  r.cell_order.clear();
  for (uint32_t o = 0; o < n; ++o)
    for (size_t k = 0; k < T; ++k) {
      const size_t c = (size_t)src[o] * T + k;
      if (ccnt[c] == 0) continue;
      r.val[(size_t)o * T + k] = (double)ccnt[c];
      r.counted->values[(size_t)o * T + k] = cval[c];
      r.valid[(size_t)o * Tw + (k >> 5)] |= 1u << (k & 31);
    }
  // export order Sort(group labels, ts, value): a group's rows by step, then rank (rank order is value order)
  for (uint32_t p = 0; p < G; ++p)
    for (size_t k = 0; k < T; ++k)
      for (uint32_t o = first[p]; o < first[p + 1]; ++o)
        if (r.valid_at(o, (int64_t)k)) r.cell_order.push_back((uint64_t)o * T + k);
  r.rows = n;
  r.columns = Columns::CountTagsTimeLabel;
  r.value_names = {count_name};
}

// ---- SubqueryPlan --------------------------------------------------------------------------------------
SubqueryPlan::SubqueryPlan(b2p_ctx* ctx, std::string function, const b2p_range_params& p, std::shared_ptr<PlanNode> child)
    : PlanNode(ctx), function_(std::move(function)), p_(p), child_(std::move(child)) {
  require("GpuPromSubqueryExec", {child_.get()});
  p_.fn_id = function_id_from_name(function_);
  if (p_.fn_id < 0) throw PlanError(ErrorKind::Plan, "GpuPromSubqueryExec: unknown range function " + function_);
  if (p_.interval <= 0) throw PlanError(ErrorKind::Plan, "GpuPromSubqueryExec: interval must be positive");
  if (p_.range <= 0) throw PlanError(ErrorKind::Plan, "GpuPromSubqueryExec: range must be positive (zero range selector)");
  if (p_.offset != 0 || p_.filter_nan != 0)
    throw PlanError(ErrorKind::Plan, "GpuPromSubqueryExec: offset and filter_nan must be 0 (RangeManipulate has neither)");
}

void SubqueryPlan::compute(NodeResult& r) {
  NodeResult C;
  child_->run(C);
  check_child(C, {{Shape::Int32, "GpuPromSubqueryExec: an Int32 value column is not supported by this node"},
                  {Shape::Int64, "GpuPromSubqueryExec: an Int64 value column is not supported by this node"}});
  const int64_t T_in = C.T;
  const int64_t step = T_in > 1 ? C.eval_ts[1] - C.eval_ts[0] : p_.interval;  // (one inner step: any positive step)
  bool regular = step > 0;
  for (int64_t k = 1; regular && k < T_in; ++k) regular = C.eval_ts[(size_t)k] == C.eval_ts[0] + k * step;
  if (!regular) throw PlanError(ErrorKind::Plan, "GpuPromSubqueryExec: the child's eval timestamps are not a regular grid");
  r = NodeResult();
  set_grid(r, p_.start, p_.end, p_.interval);
  r.rows = C.rows;
  r.F = C.F;
  r.types.assign(r.F, ValueType::Float64);
  r.val.assign((size_t)r.F * r.rows * (size_t)r.T, 0.0);
  r.valid.assign((size_t)r.rows * r.Tw, 0u);
  // the function once per field over the same windows (planner.rs:292-332), then the conjunction of the fields' IS NOT
  // NULL: a cell is kept where every field's result is
  std::vector<uint32_t> field_valid(r.F > 1 ? r.valid.size() : 0);
  for (uint32_t f = 0; f < r.F && r.rows > 0 && r.T > 0; ++f) {
    uint32_t* fv = f == 0 ? r.valid.data() : field_valid.data();
    check(b2p_subquery(ctx_, &p_, T_in > 0 ? C.eval_ts[0] : p_.start, step, C.field(f), C.valid.data(), C.rows,
                       (uint64_t)T_in, r.field(f), fv));
    if (f > 0)
      for (size_t w = 0; w < r.valid.size(); ++w) r.valid[w] &= fv[w];
  }
  r.time_index = C.time_index;
  r.labels = std::move(C.labels);
  r.labels.drop_tsid();  // a range function's projection (planner.rs:292-332)
  for (const std::string& value : C.value_names) {
    std::string name = function_ + "(" + C.time_index + "_range," + value;
    if (p_.fn_id == B2P_FN_RATE || p_.fn_id == B2P_FN_INCREASE || p_.fn_id == B2P_FN_DELTA) {
      name += "," + C.time_index + ",Int64(" + std::to_string(p_.range) + ")";
    } else if (p_.fn_id == B2P_FN_PREDICT_LINEAR || p_.fn_id == B2P_FN_QUANTILE_OVER_TIME) {
      name += "," + float_literal(p_.param0);
    } else if (p_.fn_id == B2P_FN_HOLT_WINTERS) {
      name += "," + float_literal(p_.param0) + "," + float_literal(p_.param1);
    }
    r.value_names.push_back(name + ")");
  }
}

// ---- HistogramQuantilePlan -----------------------------------------------------------------------------
HistogramQuantilePlan::HistogramQuantilePlan(b2p_ctx* ctx, std::string le_column, double phi,
                                             std::shared_ptr<PlanNode> child)
    : PlanNode(ctx), le_column_(std::move(le_column)), phi_(phi), child_(std::move(child)) {
  require("GpuPromHistogramFoldExec", {child_.get()});
}

void HistogramQuantilePlan::compute(NodeResult& r) {
  const bool sharded = sharded_ && sharded_run("GpuPromHistogramFoldExec");
  child_->run(r);
  // the reference folds the first field only (planner.rs:3084-3092, a FIXME); this node does not copy that
  const std::string int32 = "GpuPromHistogramFoldExec: an Int32 value column is not supported by this node";
  const std::string int64 = "GpuPromHistogramFoldExec: an Int64 value column is not supported by this node";
  // sharded, the value types a rank read from its batches are known only after the agreement (fold_sharded)
  check_child(r, {{Shape::Int32, sharded ? "" : int32},
                  {Shape::IdKeyed, "GpuPromHistogramFoldExec: an id-keyed (__tsid) child carries no " + le_column_ + " label"},
                  {Shape::Counted, "GpuPromHistogramFoldExec: a count_values child is not supported by this node"},
                  {Shape::MultiField, "GpuPromHistogramFoldExec: a multi-field child is not supported by this node"},
                  {Shape::Int64, sharded ? "" : int64}});
  r.cell_order.clear();
  r.counted.reset();  // (the folded rows are new rows)
  const int le = r.labels.column(le_column_);
  if (le < 0) {  // create_histogram_plan: no le tag -> EmptyRelation, no rows and no columns
    r.rows = 0;
    r.val.clear();
    r.valid.clear();
    r.labels = Labels();
    r.columns = Columns::None;
    return;
  }
  if (sharded) {
    fold_sharded(
        ctx_, le, r, [&](const NodeResult& c, uint32_t) { check_child(c, {{Shape::Int32, int32}, {Shape::Int64, int64}}); },
        [&](const uint32_t* row_hist, const double* row_le, uint32_t H, double* out, uint32_t* out_valid) {
          return b2p_histogram_fold_allgather(ctx_, phi_, r.val.data(), r.valid.data(), r.rows, (uint64_t)r.T, row_hist,
                                              row_le, H, out, out_valid);
        });
    return;
  }
  HistogramIndex ix = histogram_index(r.labels, le, r.rows);
  const uint32_t H = (uint32_t)ix.hist.rank.size();
  std::vector<double> out((size_t)H * (size_t)r.T, 0.0);
  std::vector<uint32_t> out_valid((size_t)H * r.Tw, 0u);
  if (H > 0 && r.T > 0)
    check(b2p_histogram_fold(ctx_, phi_, ix.hist_off.data(), ix.bucket_series.data(), ix.bucket_le.data(), H,
                             r.val.data(), r.valid.data(), r.rows, (uint64_t)r.T, out.data(), out_valid.data()),
          ErrorKind::Execution);
  r.val = std::move(out);
  r.valid = std::move(out_valid);
  r.labels = std::move(ix.hist.labels);
  r.rows = H;
}

// ---- SortPlan ------------------------------------------------------------------------------------------
SortPlan::SortPlan(b2p_ctx* ctx, const std::string& function, std::shared_ptr<PlanNode> child,
                   std::vector<std::string> labels)
    : PlanNode(ctx), child_(std::move(child)), labels_(std::move(labels)) {
  require("GpuPromSortExec", {child_.get()});
  if (function != "sort" && function != "sort_desc" && function != "sort_by_label" && function != "sort_by_label_desc")
    throw PlanError(ErrorKind::Plan, "GpuPromSortExec: unknown function " + function);
  by_label_ = function.compare(0, 13, "sort_by_label") == 0;
  desc_ = function == "sort_desc" || function == "sort_by_label_desc";
  // planner.rs:2743-2772: sort_by_label* needs at least one label (FunctionInvalidArgument)
  if (by_label_ && labels_.empty()) throw PlanError(ErrorKind::Plan, "GpuPromSortExec: " + function + " needs at least one label");
  if (!by_label_ && !labels_.empty()) throw PlanError(ErrorKind::Plan, "GpuPromSortExec: " + function + " takes no label");
}

void SortPlan::compute(NodeResult& r) {
  child_->run(r);
  // a multi-field child with an Int64 field is refused where sort has cells to order
  const bool int_keys = !by_label_ && r.rows > 0 && r.T > 0 && r.has(ValueType::Int64);
  check_child(r, {{Shape::Counted, "GpuPromSortExec: a count_values child is not supported by this node"},
                  {Shape::MultiField, int_keys ? "GpuPromSortExec: a multi-field child with an Int64 value column is not supported by this node" : ""},
                  {Shape::IdKeyed, by_label_ ? "GpuPromSortExec: an id-keyed (__tsid) child has no label values to sort by" : ""}});
  r.cell_order.clear();
  r.labels.drop_tsid();  // the function projection of time, value and tags (planner.rs:1055-1089)
  if (r.columns == Columns::None) return;  // no columns, no rows: the same empty batch
  r.columns = Columns::TimeValueTags;
  const uint64_t T = (uint64_t)r.T;
  if (!by_label_) {
    if (r.rows == 0 || T == 0) return;
    r.cell_order.resize((size_t)r.rows * (size_t)T);
    uint64_t n = 0;
    // by every field in turn (planner.rs:1066-1071): lexicographic over the fields
    std::vector<const double*> vals(r.F);
    for (uint32_t f = 0; f < r.F; ++f) vals[f] = r.field(f);
    check(r.is(0, ValueType::Int64) ? b2p_sort_cells_i64(ctx_, desc_ ? 1 : 0, reinterpret_cast<const int64_t*>(vals[0]), r.valid.data(),
                                           r.rows, T, r.cell_order.data(), &n)
                      : b2p_sort_cells_fields(ctx_, desc_ ? 1 : 0, vals.data(), (int32_t)r.F, r.valid.data(), r.rows, T,
                                              r.cell_order.data(), &n),
          ErrorKind::Execution);
    r.cell_order.resize((size_t)n);
    return;
  }
  std::vector<const std::vector<Label>*> cols;
  for (const std::string& l : labels_) {
    const int c = r.labels.column(l);
    if (c < 0) throw PlanError(ErrorKind::Plan, "GpuPromSortExec: No field named " + l);
    cols.push_back(&r.labels.values[(size_t)c]);
  }
  // arrow's Utf8 order: bytes (std::string compares chars as unsigned), "" first; NULL last in both directions
  auto before = [&](uint32_t a, uint32_t b) {
    for (const std::vector<Label>* col : cols) {
      const Label &x = (*col)[a], &y = (*col)[b];
      if (x == y) continue;
      if (!x || !y) return !y;
      return desc_ ? *y < *x : *x < *y;
    }
    return false;
  };
  std::vector<uint32_t> order(r.rows);
  std::iota(order.begin(), order.end(), 0u);
  std::stable_sort(order.begin(), order.end(), before);
  for (uint32_t q : order)
    for (uint64_t k = 0; k < T; ++k)
      if (r.valid_at(q, (int64_t)k)) r.cell_order.push_back((uint64_t)q * T + k);
}

// ---- AbsentPlan ----------------------------------------------------------------------------------------
AbsentPlan::AbsentPlan(b2p_ctx* ctx, Millisecond start, Millisecond end, Millisecond interval, std::string time_index,
                       std::string value_column, const std::vector<std::pair<std::string, std::string>>& labels,
                       std::shared_ptr<PlanNode> child)
    : PlanNode(ctx), start_(start), end_(end), interval_(interval), time_index_(std::move(time_index)),
      value_column_(std::move(value_column)), child_(std::move(child)) {
  require("GpuPromAbsentExec", {child_.get()});
  if (interval_ <= 0) throw PlanError(ErrorKind::Plan, "GpuPromAbsentExec: interval must be positive");
  // Absent::try_new: the fake labels collected into a HashMap (the last value of a name wins), sorted by name
  std::map<std::string, std::string> by_name;
  for (const auto& [name, value] : labels) {
    if (name == time_index_ || name == value_column_)
      throw PlanError(ErrorKind::Plan, "GpuPromAbsentExec: the label " + name + " is named like the time index or the value column");
    by_name[name] = value;
  }
  labels_.assign(by_name.begin(), by_name.end());
}

void AbsentPlan::compute(NodeResult& r) {
  NodeResult C;
  child_->run(C);
  r = NodeResult();
  set_grid(r, start_, end_, interval_);
  r.rows = 1;
  // the reference's cursor walks this grid and skips a step only when a child timestamp equals it
  if (C.rows > 0 && C.eval_ts != r.eval_ts)
    throw PlanError(ErrorKind::Plan, "GpuPromAbsentExec: the child's eval timestamps are not the grid (start, end, interval)");
  r.val.assign((size_t)r.T, 0.0);
  r.valid.assign((size_t)r.Tw, 0u);
  if (r.T > 0)
    check(b2p_absent(ctx_, C.rows > 0 ? C.valid.data() : nullptr, C.rows, (uint64_t)r.T, r.val.data(), r.valid.data()),
          ErrorKind::Execution);
  r.time_index = time_index_;
  r.value_names = {value_column_};
  for (const auto& [name, value] : labels_) {
    r.labels.names.push_back(name);
    r.labels.values.push_back({Label(value)});
  }
}

// ---- EmptyMetricPlan ---------------------------------------------------------------------------------
EmptyMetricPlan::EmptyMetricPlan(b2p_ctx* ctx, Millisecond start, Millisecond end, Millisecond interval,
                                 std::string time_index, std::string value_column, int kind, double literal)
    : PlanNode(ctx), start_(start), end_(end), interval_(interval), time_index_(std::move(time_index)),
      value_column_(std::move(value_column)), kind_(kind), literal_(literal) {
  require("GpuEmptyMetricExec", {});
  if (interval_ <= 0) throw PlanError(ErrorKind::Plan, "GpuEmptyMetricExec: interval must be positive");
  if (kind_ < B2P_EMPTY_NONE || kind_ > B2P_EMPTY_LITERAL)
    throw PlanError(ErrorKind::Plan, "GpuEmptyMetricExec: unknown kind " + std::to_string(kind_));
}

void EmptyMetricPlan::compute(NodeResult& r) {
  r = NodeResult();
  set_grid(r, start_, end_, interval_);
  r.rows = r.T > 0 ? 1 : 0;
  r.F = kind_ == B2P_EMPTY_NONE ? 0 : 1;
  r.types.assign(r.F, ValueType::Float64);
  r.time_index = time_index_;
  r.valid.assign((size_t)r.rows * r.Tw, ~0u);
  r.val.assign((size_t)r.F * r.grid(), kind_ == B2P_EMPTY_LITERAL ? literal_ : 0.0);
  if (kind_ == B2P_EMPTY_TIME) {  // time(): ts / 1000 (build_special_time_expr, empty_metric.rs:393-402), K19
    if (r.rows > 0) check(b2p_step_fn(ctx_, B2P_STEP_TIME, r.eval_ts.data(), r.valid.data(), 1, (uint64_t)r.T, r.field(0)));
    r.value_names = {time_index_ + " / " + float_literal(1000.0)};
    r.scalar_like = true;
  } else if (kind_ == B2P_EMPTY_LITERAL) {
    r.value_names = {value_column_};
    r.literal_row = true;
  }
}


// ---- LabelPlan -----------------------------------------------------------------------------------------
LabelPlan::LabelPlan(b2p_ctx* ctx, std::shared_ptr<PlanNode> child, std::string dst, std::string replacement,
                     std::string src, const std::string& regex)
    : PlanNode(ctx), child_(std::move(child)), join_(false), dst_(std::move(dst)), replacement_(std::move(replacement)),
      src_(std::move(src)) {
  // build_regexp_replace_label_expr's order: the destination name, then the raw regex (planner.rs:2531-2562); both
  // come before the child, so they can be checked without one
  if (!valid_label_name(dst_)) throw PlanError(ErrorKind::Plan, "Invalid destination label name in label_replace(): " + dst_);
  regex_ = std::make_unique<LabelRegex>(regex);
  if (regex_->verdict() == RegexVerdict::Invalid)
    throw PlanError(ErrorKind::Plan, "Invalid regular expression in label_replace(): " + regex);
  if (regex_->verdict() == RegexVerdict::Unsupported)
    throw PlanError(ErrorKind::Plan, "GpuPromLabelExec: the regular expression " + regex + " is not supported by this node: " +
                                         regex_->message());
  empty_regex_ = regex.empty();
  require("GpuPromLabelExec", {child_.get()}, false);
}

LabelPlan::LabelPlan(b2p_ctx* ctx, std::shared_ptr<PlanNode> child, std::string dst, std::string separator,
                     std::vector<std::string> srcs)
    : PlanNode(ctx), child_(std::move(child)), join_(true), dst_(std::move(dst)), replacement_(std::move(separator)),
      srcs_(std::move(srcs)) {
  require("GpuPromLabelExec", {child_.get()}, false);
  if (srcs_.empty()) throw PlanError(ErrorKind::Plan, "Invalid function argument for label_join");  // planner.rs:2687-2692
}

LabelPlan::~LabelPlan() = default;

void LabelPlan::compute(NodeResult& r) {
  child_->run(r);  // the child's result is this node's: grid, validity and the rest stay where they are
  check_child(r, {{Shape::IdKeyed, "GpuPromLabelExec: an id-keyed (__tsid) child has no label values to rewrite"},
                  {Shape::Counted, "GpuPromLabelExec: a count_values child is not supported by this node"}});
  r.labels.drop_tsid();  // its projection lists time, values and tags (create_tag_column_exprs, planner.rs:2714)
  if (r.columns == Columns::None) return;  // no columns and no rows: nothing to label
  Labels& L = r.labels;
  auto is_column = [&](const std::string& name) {
    return name == r.time_index || std::find(r.value_names.begin(), r.value_names.end(), name) != r.value_names.end();
  };
  const std::string fn = join_ ? "label_join" : "label_replace";
  const int src = join_ ? -1 : L.column(src_);
  if (!join_) {
    const bool noop = src >= 0 ? empty_regex_ : replacement_.empty();
    if (noop) {  // the projection {time index, values.., tags..} (planner.rs:2346-2351)
      r.columns = Columns::TimeValueTags;
      return;
    }
    if (L.column(dst_) >= 0) throw PlanError(ErrorKind::Plan, "vector cannot contain metrics with the same labelset");
  }
  if (is_column(dst_))
    throw PlanError(ErrorKind::Plan, "GpuPromLabelExec: " + fn + "() into " + dst_ + ", the name of the time index or a value column, is not supported by this node");
  std::vector<Label> out(r.rows);
  if (!join_ && src < 0) {  // the literal replacement on every row
    std::fill(out.begin(), out.end(), Label(replacement_));
  } else if (!join_) {  // regexp_replace over the source column, once per distinct value; NULL stays NULL
    std::unordered_map<std::string, std::string> done;
    const std::vector<Label>& in = L.values[(size_t)src];
    for (uint32_t q = 0; q < r.rows; ++q) {
      if (!in[q]) continue;
      auto it = done.find(*in[q]);
      if (it == done.end()) it = done.emplace(*in[q], regex_->replace(*in[q], replacement_)).first;
      out[q] = it->second;
    }
  } else {  // concat_ws(separator, src..): "" and absent sources are NULL literals, and NULLs are skipped
    std::vector<int> cols;
    for (const std::string& s : srcs_) {
      if (!s.empty() && is_column(s))
        throw PlanError(ErrorKind::Plan, "GpuPromLabelExec: label_join() over " + s + ", the time index or a value column, is not supported by this node");
      if (!s.empty() && L.column(s) >= 0) cols.push_back(L.column(s));
    }
    // (no cache: joining the parts costs less than hashing them)
    for (uint32_t q = 0; q < r.rows; ++q) {
      std::string v;
      bool first = true;
      for (int c : cols) {
        const Label& part = L.values[(size_t)c][q];
        if (!part) continue;
        if (!first) v += replacement_;
        v += *part;
        first = false;
      }
      out[q] = std::move(v);
    }
    const int old = L.column(dst_);  // dropped from the tags, then added as the new one (planner.rs:2318-2321)
    if (old >= 0) {
      L.names.erase(L.names.begin() + old);
      L.values.erase(L.values.begin() + old);
    }
  }
  L.names.push_back(dst_);
  L.values.push_back(std::move(out));
  r.columns = Columns::TimeValueLastTag;
  r.scalar_like = r.literal_row = false;
}

}  // namespace b2p

// ---- C entry points -----------------------------------------------------------------------------------
struct b2p_plan {
  std::shared_ptr<b2p::PlanNode> node;  // shared with the binary nodes built on top of it
  b2p::PromRangePlan* range() const { return dynamic_cast<b2p::PromRangePlan*>(node.get()); }
};

namespace {
thread_local std::string g_err;
int plan_fail(const b2p::PlanError& e) {
  g_err = e.what();
  switch (e.kind) {
    case b2p::ErrorKind::Plan: return B2P_E_INVALID;
    case b2p::ErrorKind::Internal: return B2P_E_UNSORTED;
    default: return B2P_E_CUDA;
  }
}
int not_a_range_node() {
  g_err = "this call needs a range / instant node (b2p_plan_range_create)";
  return B2P_E_INVALID;
}

// The body of a b2p_plan_*_create: a handle on the node make() returns, or NULL with the error for b2p_plan_last_error()
template <class Make>
b2p_plan* create(Make make) {
  try {
    return new b2p_plan{make()};
  } catch (const b2p::PlanError& e) {
    plan_fail(e);
  } catch (const std::exception& e) {
    g_err = e.what();
  }
  return nullptr;
}

// The body of an entry point that works on a node: B2P_OK, or the code of the error fn() throws
template <class Fn>
int guarded(Fn fn) {
  try {
    fn();
    return B2P_OK;
  } catch (const b2p::PlanError& e) {
    return plan_fail(e);
  } catch (const std::exception& e) {
    g_err = e.what();
    return B2P_E_NOMEM;
  }
}

// "on" / "ignoring"; NULL or "" is no modifier
b2p::Matching parse_matching(const char* m) {
  if (!m || !m[0]) return b2p::Matching::None;
  if (std::strcmp(m, "on") == 0) return b2p::Matching::On;
  if (std::strcmp(m, "ignoring") == 0) return b2p::Matching::Ignoring;
  throw b2p::PlanError(b2p::ErrorKind::Plan, std::string("unknown matching ") + m);
}

// "by" / "without"; NULL or "" is no modifier
b2p::Modifier parse_modifier(const char* m) {
  if (!m || !m[0]) return b2p::Modifier::None;
  if (std::strcmp(m, "by") == 0) return b2p::Modifier::By;
  if (std::strcmp(m, "without") == 0) return b2p::Modifier::Without;
  throw b2p::PlanError(b2p::ErrorKind::Plan, std::string("unknown modifier ") + m);
}

std::vector<std::string> strings(const char* const* v, int32_t n) {
  std::vector<std::string> out;
  for (int32_t i = 0; i < n; ++i) out.emplace_back(v[i]);
  return out;
}
}  // namespace

extern "C" {

const char* b2p_plan_last_error(void) { return g_err.c_str(); }

b2p_plan* b2p_plan_range_create_fields(b2p_ctx* ctx, const char* function, const b2p_range_params* p,
                                       const char* time_index, const char* const* field_columns, int32_t n_fields,
                                       const char* const* tag_columns, int32_t n_tags, const char* aggregate,
                                       const char* const* by_columns, int32_t n_by) {
  return create([&] {
    if (!function || !p || !time_index || !field_columns) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    if (n_fields < 1 || n_fields > B2P_MAX_FIELDS)
      throw b2p::PlanError(b2p::ErrorKind::Plan, "n_fields must be in [1, " + std::to_string(B2P_MAX_FIELDS) + "], got " +
                                                     std::to_string(n_fields));
    for (int32_t f = 0; f < n_fields; ++f)
      if (!field_columns[f]) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    b2p::PromRangePlanArgs a;
    a.function = function;
    a.start = p->start;
    a.end = p->end;
    a.interval = p->interval;
    a.range = p->range;
    a.offset = p->offset;
    a.need_filter_out_nan = p->filter_nan != 0;
    a.param0 = p->param0;
    a.param1 = p->param1;
    a.time_index = time_index;
    a.field_columns = strings(field_columns, n_fields);
    a.tag_columns = strings(tag_columns, n_tags);
    if (aggregate && aggregate[0]) a.aggregate = aggregate;
    a.by_columns = strings(by_columns, n_by);
    return std::make_shared<b2p::PromRangePlan>(ctx, std::move(a));
  });
}

b2p_plan* b2p_plan_range_create(b2p_ctx* ctx, const char* function, const b2p_range_params* p, const char* time_index,
                                const char* field_column, const char* const* tag_columns, int32_t n_tags,
                                const char* aggregate, const char* const* by_columns, int32_t n_by) {
  if (!field_column) {
    g_err = "NULL argument";
    return nullptr;
  }
  return b2p_plan_range_create_fields(ctx, function, p, time_index, &field_column, 1, tag_columns, n_tags, aggregate,
                                      by_columns, n_by);
}

b2p_plan* b2p_plan_binary_create(b2p_ctx* ctx, int32_t op, int32_t return_bool, b2p_plan* lhs, b2p_plan* rhs,
                                 const char* matching, const char* const* labels, int32_t n_labels,
                                 const char* label_side) {
  return create([&] {
    if (!lhs || !rhs || !label_side || (n_labels > 0 && !labels))
      throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    const b2p::Matching m = parse_matching(matching);
    const bool from_lhs = std::strcmp(label_side, "lhs") == 0;
    if (!from_lhs && std::strcmp(label_side, "rhs") != 0)
      throw b2p::PlanError(b2p::ErrorKind::Plan, std::string("label_side must be \"lhs\" or \"rhs\", got ") + label_side);
    return std::make_shared<b2p::BinaryPlan>(ctx, op, return_bool != 0, lhs->node, rhs->node, m,
                                             strings(labels, n_labels), from_lhs);
  });
}

b2p_plan* b2p_plan_setop_create(b2p_ctx* ctx, int32_t op, b2p_plan* lhs, b2p_plan* rhs, const char* matching,
                                const char* const* labels, int32_t n_labels) {
  return create([&] {
    if (!lhs || !rhs || (n_labels > 0 && !labels)) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    const b2p::Matching m = parse_matching(matching);
    return std::make_shared<b2p::SetOpPlan>(ctx, op, lhs->node, rhs->node, m, strings(labels, n_labels));
  });
}

b2p_plan* b2p_plan_scalar_create(b2p_ctx* ctx, b2p_plan* child) {
  return create([&] {
    if (!child) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::ScalarPlan>(ctx, child->node);
  });
}

b2p_plan* b2p_plan_topk_create(b2p_ctx* ctx, int32_t bottom, double k, b2p_plan* child, const char* modifier,
                               const char* const* labels, int32_t n_labels) {
  return create([&] {
    if (!child || (n_labels > 0 && !labels)) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::TopkPlan>(ctx, bottom != 0, k, child->node, parse_modifier(modifier),
                                           strings(labels, n_labels));
  });
}

b2p_plan* b2p_plan_aggregate_create(b2p_ctx* ctx, const char* op, double param, b2p_plan* child, const char* modifier,
                                    const char* const* labels, int32_t n_labels) {
  return create([&] {
    if (!op || !child || (n_labels > 0 && !labels)) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::AggregatePlan>(ctx, op, param, child->node, parse_modifier(modifier),
                                                strings(labels, n_labels));
  });
}

b2p_plan* b2p_plan_count_values_create(b2p_ctx* ctx, const char* label, b2p_plan* child, const char* modifier,
                                       const char* const* labels, int32_t n_labels) {
  return create([&] {
    if (!label || !child || (n_labels > 0 && !labels)) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::CountValuesPlan>(ctx, label, child->node, parse_modifier(modifier),
                                                  strings(labels, n_labels));
  });
}

b2p_plan* b2p_plan_subquery_create(b2p_ctx* ctx, const char* function, const b2p_range_params* p, b2p_plan* child) {
  return create([&] {
    if (!function || !p || !child) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::SubqueryPlan>(ctx, function, *p, child->node);
  });
}

b2p_plan* b2p_plan_histogram_quantile_create(b2p_ctx* ctx, const char* le_column, double phi, b2p_plan* child) {
  return create([&] {
    if (!child) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::HistogramQuantilePlan>(ctx, le_column ? le_column : "le", phi, child->node);
  });
}

b2p_plan* b2p_plan_sort_create(b2p_ctx* ctx, const char* function, b2p_plan* child, const char* const* labels,
                               int32_t n_labels) {
  return create([&] {
    if (!function || !child || n_labels < 0 || (n_labels > 0 && !labels))
      throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::SortPlan>(ctx, function, child->node, strings(labels, n_labels));
  });
}

b2p_plan* b2p_plan_absent_create(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval, const char* time_index,
                                 const char* value_column, const char* const* label_names,
                                 const char* const* label_values, int32_t n_labels, b2p_plan* child) {
  return create([&] {
    if (!time_index || !value_column || !child || (n_labels > 0 && (!label_names || !label_values)))
      throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    if (n_labels < 0) throw b2p::PlanError(b2p::ErrorKind::Plan, "n_labels < 0");
    std::vector<std::pair<std::string, std::string>> labels;
    for (int32_t i = 0; i < n_labels; ++i) {
      if (!label_names[i] || !label_values[i]) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL label name or value");
      labels.emplace_back(label_names[i], label_values[i]);
    }
    return std::make_shared<b2p::AbsentPlan>(ctx, start, end, interval, time_index, value_column, labels, child->node);
  });
}

b2p_plan* b2p_plan_empty_metric_create(b2p_ctx* ctx, int64_t start, int64_t end, int64_t interval,
                                       const char* time_index, const char* value_column, int32_t kind, double literal) {
  return create([&] {
    if (!time_index || !value_column) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::EmptyMetricPlan>(ctx, start, end, interval, time_index, value_column, kind, literal);
  });
}

b2p_plan* b2p_plan_label_replace_create(b2p_ctx* ctx, b2p_plan* child, const char* dst, const char* replacement,
                                        const char* src, const char* regex) {
  return create([&] {
    if (!dst || !replacement || !src || !regex) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::LabelPlan>(ctx, child ? child->node : nullptr, dst, replacement, src, regex);
  });
}

b2p_plan* b2p_plan_label_join_create(b2p_ctx* ctx, b2p_plan* child, const char* dst, const char* separator,
                                     const char* const* srcs, int32_t n_srcs) {
  return create([&] {
    if (!child || !dst || !separator || n_srcs < 0 || (n_srcs > 0 && !srcs))
      throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    for (int32_t i = 0; i < n_srcs; ++i)
      if (!srcs[i]) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    return std::make_shared<b2p::LabelPlan>(ctx, child->node, dst, separator, strings(srcs, n_srcs));
  });
}

int b2p_label_regex_check(const char* regex) {
  if (!regex) {
    g_err = "NULL argument";
    return B2P_E_INVALID;
  }
  const b2p::LabelRegex re(regex);
  g_err = re.message();
  return (int)re.verdict();
}

int b2p_label_regex_replace(const char* regex, const char* replacement, const char* input, char* out, uint64_t cap,
                            uint64_t* out_len) {
  if (!regex || !replacement || !input || (cap > 0 && !out)) {
    g_err = "NULL argument";
    return B2P_E_INVALID;
  }
  const b2p::LabelRegex re(regex);
  if (re.verdict() != b2p::RegexVerdict::Ok) {
    g_err = re.message();
    return B2P_E_INVALID;
  }
  const std::string v = re.replace(input, replacement);
  if (out_len) *out_len = v.size();
  if (v.size() + 1 > cap) {
    g_err = "the result needs " + std::to_string(v.size() + 1) + " bytes";
    return B2P_E_TOO_LARGE;
  }
  std::memcpy(out, v.c_str(), v.size() + 1);
  return B2P_OK;
}

int b2p_plan_set_timestamp(b2p_plan* plan, int64_t lookback_delta) {
  if (!plan) return B2P_E_INVALID;
  if (!plan->range()) return not_a_range_node();
  return plan->range()->set_timestamp(lookback_delta);
}

int b2p_plan_set_instant(b2p_plan* plan, int64_t lookback_delta) {
  if (!plan) return B2P_E_INVALID;
  if (!plan->range()) return not_a_range_node();
  return plan->range()->set_instant(lookback_delta);
}

int b2p_plan_set_label_columns(b2p_plan* plan, const char* const* names, int32_t n) {
  if (!plan) return B2P_E_INVALID;
  if (!plan->range()) return not_a_range_node();
  return guarded([&] {
    if (n < 0 || (n > 0 && !names)) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    for (int32_t i = 0; i < n; ++i)
      if (!names[i]) throw b2p::PlanError(b2p::ErrorKind::Plan, "NULL argument");
    plan->range()->set_label_columns(strings(names, n));
  });
}

int b2p_plan_set_histogram_quantile(b2p_plan* plan, const char* le_column, double quantile) {
  if (!plan || !le_column) return B2P_E_INVALID;
  if (!plan->range()) return not_a_range_node();
  return guarded([&] { plan->range()->set_histogram(le_column, quantile); });
}

int b2p_plan_set_scalar_op(b2p_plan* plan, int32_t op, double scalar, int32_t scalar_on_left, int32_t return_bool) {
  if (!plan) return B2P_E_INVALID;
  return guarded([&] { plan->node->add_scalar_op(op, scalar, scalar_on_left != 0, return_bool != 0); });
}

int b2p_plan_set_function(b2p_plan* plan, const char* name, const double* args, int32_t n_args) {
  if (!plan || !name || n_args < 0 || (n_args > 0 && !args)) return B2P_E_INVALID;
  return guarded([&] { plan->node->add_function(name, std::vector<double>(args, args + n_args)); });
}

int b2p_plan_push_batch(b2p_plan* plan, struct ArrowArray* batch, struct ArrowSchema* schema) {
  if (!plan) return B2P_E_INVALID;
  if (!plan->range()) return not_a_range_node();
  return guarded([&] { plan->range()->push(std::make_unique<b2p::RecordBatch>(batch, schema)); });
}

int b2p_plan_execute(b2p_plan* plan, struct ArrowArray* out, struct ArrowSchema* out_schema) {
  if (!plan) return B2P_E_INVALID;
  return guarded([&] { plan->node->execute(out, out_schema); });
}

int b2p_plan_set_sharded(b2p_plan* plan) {
  if (!plan) return B2P_E_INVALID;
  return guarded([&] {
    if (!plan->node->set_sharded())
      throw b2p::PlanError(b2p::ErrorKind::Plan, "b2p_plan_set_sharded: only an aggregate node, a count_values node, "
                                                 "a histogram_quantile node or a range / instant leaf with an aggregate "
                                                 "or HistogramFold stage has a sharded form");
  });
}

int b2p_group_keys_merge(const void* const* blocks, const uint64_t* sizes, int32_t n_ranks, int32_t rank,
                         void* out_table, uint64_t* out_table_bytes, uint32_t* n_groups, uint32_t* local_to_global) {
  return guarded([&] {
    if (!blocks || !sizes || n_ranks < 1 || rank < 0 || rank >= n_ranks || !out_table || !out_table_bytes || !n_groups)
      throw b2p::PlanError(b2p::ErrorKind::Plan, "b2p_group_keys_merge: bad arguments");
    std::vector<b2p::KeyBlock> parsed;
    uint64_t total = 0;
    for (int32_t r = 0; r < n_ranks; ++r) {
      if (!blocks[r] && sizes[r]) throw b2p::PlanError(b2p::ErrorKind::Plan, "b2p_group_keys_merge: NULL block");
      parsed.push_back(b2p::parse_keys(static_cast<const uint8_t*>(blocks[r]), sizes[r], r));
      total += sizes[r];
    }
    b2p::Agreement a = b2p::merge_keys(parsed, rank);
    const std::vector<uint32_t>& l2g = a.l2g;
    *n_groups = a.n_groups;
    if (!l2g.empty() && !local_to_global) throw b2p::PlanError(b2p::ErrorKind::Plan, "b2p_group_keys_merge: NULL local_to_global");
    const std::string bytes = b2p::serialize_keys(a.labels, a.n_groups, a.labels.tsid, a.n_rows, a.types);
    if (bytes.size() > total) throw b2p::PlanError(b2p::ErrorKind::Plan, "b2p_group_keys_merge: the table exceeds the blocks");
    std::memcpy(out_table, bytes.data(), bytes.size());
    *out_table_bytes = bytes.size();
    std::copy(l2g.begin(), l2g.end(), local_to_global);
  });
}

int64_t b2p_plan_num_series(b2p_plan* plan) { return plan && plan->range() ? plan->range()->num_series() : -1; }

void b2p_plan_destroy(b2p_plan* plan) { delete plan; }

}  // extern "C"
