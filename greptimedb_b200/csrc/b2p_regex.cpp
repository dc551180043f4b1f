// b2p_regex.cpp — the label_replace regex engine (see b2p_regex.hpp): a parser that returns Rust's verdict, a Thompson
// compiler and a Pike VM over code points.
#include "b2p_regex.hpp"

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace b2p {

namespace {

// UTF-8 -> code points and the byte offset of each (offsets has one more entry: the end); false on invalid UTF-8
bool decode(const std::string& s, std::vector<uint32_t>& cps, std::vector<uint32_t>* offsets) {
  cps.clear();
  if (offsets) offsets->clear();
  const auto* p = reinterpret_cast<const unsigned char*>(s.data());
  const size_t n = s.size();
  size_t i = 0;
  bool ok = true;
  while (i < n) {
    if (offsets) offsets->push_back((uint32_t)i);
    const unsigned char c = p[i];
    uint32_t cp = 0xFFFD;
    size_t len = 1;
    if (c < 0x80) {
      cp = c;
    } else {
      len = c >= 0xF0 && c < 0xF5 ? 4 : c >= 0xE0 ? 3 : c >= 0xC2 && c < 0xE0 ? 2 : 0;
      if (len == 0 || c >= 0xF5 || i + len > n) {
        ok = false;
        len = 1;
      } else {
        cp = c & (0x7F >> len);
        for (size_t k = 1; k < len; ++k) {
          if ((p[i + k] & 0xC0) != 0x80) ok = false;
          cp = (cp << 6) | (p[i + k] & 0x3F);
        }
        const uint32_t lo = len == 2 ? 0x80 : len == 3 ? 0x800 : 0x10000;
        if (!ok || cp < lo || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) {
          ok = false;
          cp = 0xFFFD;
          len = 1;
        }
      }
    }
    cps.push_back(cp);
    i += len;
  }
  if (offsets) offsets->push_back((uint32_t)n);
  return ok;
}

enum AssertKind : uint32_t { kTextStart, kTextEnd, kLineStart, kLineEnd };

struct Node {
  enum Kind { Empty, Lit, Dot, Class, Assert, Cat, Alt, Group, Repeat } k = Empty;
  uint32_t c = 0;       // Lit: code point; Class: index; Assert: kind
  bool dotall = false;  // Dot
  int cap = -1;         // Group: capture index, -1 for a non-capturing group
  uint32_t min = 0, max = 0;
  bool unbounded = false, greedy = true;
  std::vector<Node> kids;
};

struct Flags {
  bool s = false, m = false, U = false;
};

const char kMeta[] = ".+*?()|[]{}^$#&-~\\";

struct AsciiClass {
  const char* name;
  const char* ranges;  // pairs of inclusive bounds
};
const AsciiClass kAsciiClasses[] = {
    {"alnum", "09AZaz"}, {"alpha", "AZaz"}, {"ascii", "\x01\x7f"}, {"blank", "\t\t  "}, {"cntrl", "\x01\x1f\x7f\x7f"},
    {"digit", "09"}, {"graph", "!~"}, {"lower", "az"}, {"print", " ~"}, {"punct", "!/:@[`{~"},
    {"space", "\t\r  "}, {"upper", "AZ"}, {"word", "09AZ__az"}, {"xdigit", "09AFaf"},
};

int hexval(uint32_t c) {
  if (c >= '0' && c <= '9') return (int)(c - '0');
  if (c >= 'a' && c <= 'f') return (int)(c - 'a' + 10);
  if (c >= 'A' && c <= 'F') return (int)(c - 'A' + 10);
  return -1;
}

bool is_ascii_alpha(uint32_t c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'); }
bool is_ascii_digit(uint32_t c) { return c >= '0' && c <= '9'; }

}  // namespace

bool LabelRegex::CharClass::has(uint32_t c) const {
  bool in = false;
  for (const auto& r : ranges)
    if (c >= r.first && c <= r.second) {
      in = true;
      break;
    }
  return in != negated;
}

class RegexParser {
 public:
  RegexParser(LabelRegex& re, std::vector<uint32_t> p) : re_(re), p_(std::move(p)) {}

  Node parse() {
    Node n = alt(0);
    if (pos_ < p_.size()) fail(RegexVerdict::Invalid, "unopened group");  // (only `)` stops alt() early)
    return n;
  }

  struct Stop {};  // thrown once the verdict is known

 private:
  LabelRegex& re_;
  std::vector<uint32_t> p_;
  size_t pos_ = 0;
  Flags flags_{true, false, false};  // the pattern runs inside (?s:...)
  std::vector<std::string> names_;

  [[noreturn]] void fail(RegexVerdict v, const std::string& msg) {
    re_.verdict_ = v;
    re_.message_ = msg;
    throw Stop{};
  }
  bool more() const { return pos_ < p_.size(); }
  uint32_t peek(size_t ahead = 0) const { return pos_ + ahead < p_.size() ? p_[pos_ + ahead] : 0xFFFFFFFFu; }

  Node alt(int depth) {
    if (depth > 64) fail(RegexVerdict::Unsupported, "nesting deeper than 64");
    Node n;
    n.k = Node::Alt;
    n.kids.push_back(cat(depth));
    while (more() && peek() == '|') {
      ++pos_;
      n.kids.push_back(cat(depth));
    }
    return n.kids.size() == 1 ? std::move(n.kids[0]) : n;
  }

  Node cat(int depth) {
    Node n;
    n.k = Node::Cat;
    bool after_flags = false;  // the last item was a (?flags) group, which is no expression
    while (more() && peek() != '|' && peek() != ')') {
      const uint32_t c = peek();
      if (c == '*' || c == '+' || c == '?' || c == '{') {
        if (after_flags) fail(RegexVerdict::Unsupported, "a repetition after a flag group");
        if (n.kids.empty()) {
          if (c == '{') fail(RegexVerdict::Unsupported, "a `{` with nothing to repeat");
          fail(RegexVerdict::Invalid, "repetition operator missing expression");
        }
        Node& last = n.kids.back();
        if (last.k == Node::Repeat) fail(RegexVerdict::Unsupported, "a repetition of a repetition");
        if (last.k == Node::Assert) fail(RegexVerdict::Unsupported, "a repetition of an assertion");
        if (last.k == Node::Empty) fail(RegexVerdict::Invalid, "repetition operator missing expression");
        Node r;
        r.k = Node::Repeat;
        repetition(r);
        r.kids.push_back(std::move(last));
        last = std::move(r);
        continue;
      }
      Node a = atom(depth);
      after_flags = a.k == Node::Empty;
      if (!after_flags) n.kids.push_back(std::move(a));
    }
    if (n.kids.size() == 1) return std::move(n.kids[0]);
    if (n.kids.empty()) return Node();
    return n;
  }

  void repetition(Node& r) {
    const uint32_t c = p_[pos_++];
    if (c == '*') r.min = 0, r.unbounded = true;
    else if (c == '+') r.min = 1, r.unbounded = true;
    else if (c == '?') r.min = 0, r.max = 1;
    else {  // {n} {n,} {n,m}
      auto number = [&](uint32_t& out) {
        const size_t s = pos_;
        uint64_t v = 0;
        while (more() && is_ascii_digit(peek()) && v <= 100000) v = v * 10 + (p_[pos_++] - '0');
        if (pos_ == s) return false;
        if (v > 1000) fail(RegexVerdict::Unsupported, "a counted repetition above 1000");
        out = (uint32_t)v;
        return true;
      };
      if (!number(r.min)) fail(RegexVerdict::Unsupported, "a `{` that is not {n}, {n,} or {n,m}");
      if (more() && peek() == ',') {
        ++pos_;
        if (more() && peek() == '}') r.unbounded = true;
        else if (!number(r.max)) fail(RegexVerdict::Unsupported, "a `{` that is not {n}, {n,} or {n,m}");
      } else {
        r.max = r.min;
      }
      if (!more() || peek() != '}') fail(RegexVerdict::Unsupported, "a `{` that is not {n}, {n,} or {n,m}");
      ++pos_;
      if (!r.unbounded && r.max < r.min) fail(RegexVerdict::Invalid, "invalid repetition count range");
    }
    r.greedy = true;
    if (more() && peek() == '?') {
      ++pos_;
      r.greedy = false;
    }
    if (flags_.U) r.greedy = !r.greedy;
  }

  Node lit(uint32_t c) {
    Node n;
    n.k = Node::Lit;
    n.c = c;
    return n;
  }
  Node assertion(uint32_t kind) {
    Node n;
    n.k = Node::Assert;
    n.c = kind;
    return n;
  }

  Node atom(int depth) {
    const uint32_t c = p_[pos_++];
    switch (c) {
      case '(': return group(depth);
      case '[': return cls();
      case '.': {
        Node n;
        n.k = Node::Dot;
        n.dotall = flags_.s;
        return n;
      }
      case '^': return assertion(flags_.m ? kLineStart : kTextStart);
      case '$': return assertion(flags_.m ? kLineEnd : kTextEnd);
      case '\\': {
        if (more() && peek() == 'A') return ++pos_, assertion(kTextStart);
        if (more() && peek() == 'z') return ++pos_, assertion(kTextEnd);
        return lit(escape(false));
      }
      default: return lit(c);
    }
  }

  // an escape after the backslash, as one code point
  uint32_t escape(bool in_class) {
    if (!more()) fail(RegexVerdict::Invalid, "incomplete escape sequence");
    const uint32_t c = p_[pos_++];
    if (c < 0x80 && std::strchr(kMeta, (int)c)) return c;
    switch (c) {
      case 'n': return '\n';
      case 't': return '\t';
      case 'r': return '\r';
      case 'f': return 0x0C;
      case 'v': return 0x0B;
      case 'a': return 0x07;
      case 'x': {
        uint32_t v = 0;
        if (more() && peek() == '{') {
          ++pos_;
          int digits = 0;
          while (more() && peek() != '}') {
            const int h = hexval(p_[pos_++]);
            if (h < 0 || ++digits > 8) fail(RegexVerdict::Invalid, "invalid hexadecimal escape");
            v = v * 16 + (uint32_t)h;
          }
          if (!more() || digits == 0) fail(RegexVerdict::Invalid, "invalid hexadecimal escape");
          ++pos_;
        } else {
          for (int k = 0; k < 2; ++k) {
            const int h = more() ? hexval(p_[pos_++]) : -1;
            if (h < 0) fail(RegexVerdict::Invalid, "invalid hexadecimal escape");
            v = v * 16 + (uint32_t)h;
          }
        }
        if (v > 0x10FFFF || (v >= 0xD800 && v <= 0xDFFF)) fail(RegexVerdict::Invalid, "invalid hexadecimal escape");
        return v;
      }
      case 'd': case 'D': case 'w': case 'W': case 's': case 'S': case 'b': case 'B': case 'p': case 'P':
      case 'u': case 'U': case '<': case '>':
        fail(RegexVerdict::Unsupported, std::string("the escape \\") + (char)c);
      case 'A': case 'z':  // (outside a class, atom() takes them)
        if (in_class) fail(RegexVerdict::Unsupported, "an assertion escape inside a class");
        break;
      default: break;
    }
    if (is_ascii_digit(c)) fail(RegexVerdict::Invalid, "backreferences are not supported");
    if (is_ascii_alpha(c)) fail(RegexVerdict::Invalid, "unrecognized escape sequence");
    fail(RegexVerdict::Unsupported, "an escape of a character that is not a meta character");
  }

  Node group(int depth) {
    Node n;
    n.k = Node::Group;
    const Flags saved = flags_;
    if (more() && peek() == '?') {
      ++pos_;
      const uint32_t c = peek();
      if (c == '=' || c == '!') fail(RegexVerdict::Invalid, "look-around is not supported");
      if (c == '<' && (peek(1) == '=' || peek(1) == '!')) fail(RegexVerdict::Invalid, "look-around is not supported");
      if (c == '#') fail(RegexVerdict::Invalid, "unrecognized flag");
      if (c == 'P' || c == '<') {
        if (c == 'P') {
          ++pos_;
          if (peek() != '<') fail(RegexVerdict::Invalid, "unrecognized group syntax");
        }
        ++pos_;
        std::string name;
        bool ascii = true;
        while (more() && peek() != '>') {
          const uint32_t d = p_[pos_++];
          const bool ok = d == '_' || is_ascii_alpha(d) || (is_ascii_digit(d) && !name.empty());
          if (!ok) ascii = false;
          if (name.empty() && is_ascii_digit(d)) fail(RegexVerdict::Invalid, "invalid capture group name");
          name.push_back(d < 0x80 ? (char)d : '?');
        }
        if (!more()) fail(RegexVerdict::Invalid, "unclosed capture group name");
        ++pos_;
        if (name.empty()) fail(RegexVerdict::Invalid, "empty capture group name");
        if (!ascii) fail(RegexVerdict::Unsupported, "a capture group name outside [A-Za-z_][A-Za-z0-9_]*");
        if (std::find(names_.begin(), names_.end(), name) != names_.end())
          fail(RegexVerdict::Invalid, "duplicate capture group name");
        names_.push_back(name);
        n.cap = (int)re_.groups_++;
        re_.names_.emplace_back(name, (uint32_t)n.cap);
      } else {
        // flags: (?flags) for the rest of the enclosing group, (?flags:...) for the group
        bool negate = false, any = false, dangling = false;
        std::string seen;
        while (true) {
          if (!more()) fail(RegexVerdict::Invalid, "unclosed group");
          const uint32_t f = p_[pos_++];
          if (f == ':' || f == ')') {
            if (dangling) fail(RegexVerdict::Invalid, "dangling flag negation");
            if (f == ')') {
              if (!any && !negate) fail(RegexVerdict::Invalid, "empty flag group");
              n.k = Node::Empty;  // no group: the flags stay set after it
              return n;
            }
            break;
          }
          if (f == '-') {
            if (negate) fail(RegexVerdict::Invalid, "repeated flag negation");
            negate = dangling = true;
            continue;
          }
          if (f < 0x80 && seen.find((char)f) != std::string::npos) fail(RegexVerdict::Invalid, "duplicate flag");
          if (f < 0x80) seen.push_back((char)f);
          dangling = false;
          any = true;
          switch (f) {
            case 's': flags_.s = !negate; break;
            case 'm': flags_.m = !negate; break;
            case 'U': flags_.U = !negate; break;
            case 'i': case 'x': case 'u': case 'R':
              fail(RegexVerdict::Unsupported, std::string("the flag ") + (char)f);
            default: fail(RegexVerdict::Invalid, "unrecognized flag");
          }
        }
      }
    } else {
      n.cap = (int)re_.groups_++;
    }
    Node body = alt(depth + 1);
    if (!more() || peek() != ')') fail(RegexVerdict::Invalid, "unclosed group");
    ++pos_;
    flags_ = saved;
    n.kids.push_back(std::move(body));
    return n;
  }

  Node cls() {
    LabelRegex::CharClass cc;
    if (more() && peek() == '^') {
      ++pos_;
      cc.negated = true;
    }
    bool first = true;
    while (true) {
      if (!more()) fail(RegexVerdict::Invalid, "unclosed character class");
      uint32_t c = p_[pos_];
      if (c == ']' && !first) {
        ++pos_;
        break;
      }
      if (c == '[') {
        if (peek(1) == ':') {
          size_t e = pos_ + 2;
          while (e < p_.size() && p_[e] != ':' && p_[e] != ']') ++e;
          if (e + 1 < p_.size() && p_[e] == ':' && p_[e + 1] == ']') {
            bool neg = false;
            std::string name;
            for (size_t k = pos_ + 2; k < e; ++k) name.push_back(p_[k] < 0x80 ? (char)p_[k] : '?');
            if (!name.empty() && name[0] == '^') neg = true, name.erase(0, 1);
            const AsciiClass* found = nullptr;
            for (const AsciiClass& a : kAsciiClasses)
              if (name == a.name) found = &a;
            if (!found) fail(RegexVerdict::Invalid, "invalid ASCII class name");
            std::vector<std::pair<uint32_t, uint32_t>> rs;
            for (const char* r = found->ranges; *r; r += 2) rs.emplace_back((uint32_t)(unsigned char)r[0], (uint32_t)(unsigned char)r[1]);
            if (found == &kAsciiClasses[2]) rs = {{0, 0x7F}};
            if (found == &kAsciiClasses[4]) rs = {{0, 0x1F}, {0x7F, 0x7F}};
            if (neg) {  // the complement within all code points
              std::sort(rs.begin(), rs.end());
              std::vector<std::pair<uint32_t, uint32_t>> comp;
              uint32_t lo = 0;
              for (const auto& r : rs) {
                if (r.first > lo) comp.emplace_back(lo, r.first - 1);
                lo = std::max(lo, r.second + 1);
              }
              comp.emplace_back(lo, 0x10FFFF);
              rs = comp;
            }
            cc.ranges.insert(cc.ranges.end(), rs.begin(), rs.end());
            pos_ = e + 2;
            first = false;
            continue;
          }
        }
        fail(RegexVerdict::Unsupported, "a nested character class");
      }
      if ((c == '&' || c == '~' || c == '-') && peek(1) == c) fail(RegexVerdict::Unsupported, "a class set operation");
      if (c == '-' && !first && peek(1) != ']') fail(RegexVerdict::Unsupported, "a `-` inside a class that is not a range");
      ++pos_;
      if (c == '\\') c = escape(true);
      uint32_t hi = c;
      if (more() && peek() == '-' && peek(1) != ']' && pos_ + 1 < p_.size()) {
        ++pos_;
        hi = p_[pos_++];
        if (hi == '[' || hi == '-' || hi == '&' || hi == '~') fail(RegexVerdict::Unsupported, "a class range ending in an operator");
        if (hi == '\\') hi = escape(true);
        if (hi < c) fail(RegexVerdict::Invalid, "invalid character class range");
      }
      cc.ranges.emplace_back(c, hi);
      first = false;
    }
    Node n;
    n.k = Node::Class;
    n.c = (uint32_t)re_.classes_.size();
    re_.classes_.push_back(std::move(cc));
    return n;
  }
};

namespace {

using Inst = LabelRegex::Inst;

struct Compiler {
  std::vector<Inst>& prog;
  uint32_t emit(Inst::Op op, uint32_t a = 0, uint32_t b = 0) {
    if (prog.size() >= LabelRegex::kMaxProgram) throw std::length_error("program");
    prog.push_back(Inst{op, a, b});
    return (uint32_t)prog.size() - 1;
  }
  uint32_t here() const { return (uint32_t)prog.size(); }

  void node(const Node& n) {
    switch (n.k) {
      case Node::Empty: return;
      case Node::Lit: emit(Inst::Char, n.c); return;
      case Node::Dot: emit(n.dotall ? Inst::Any : Inst::AnyNoNL); return;
      case Node::Class: emit(Inst::Class, n.c); return;
      case Node::Assert: emit(Inst::Assert, n.c); return;
      case Node::Cat:
        for (const Node& k : n.kids) node(k);
        return;
      case Node::Group:
        if (n.cap >= 0) emit(Inst::Save, 2 * (uint32_t)n.cap);
        if (!n.kids.empty()) node(n.kids[0]);
        if (n.cap >= 0) emit(Inst::Save, 2 * (uint32_t)n.cap + 1);
        return;
      case Node::Alt: {
        std::vector<uint32_t> jumps;
        for (size_t i = 0; i < n.kids.size(); ++i) {
          if (i + 1 < n.kids.size()) {
            const uint32_t sp = emit(Inst::Split);
            prog[sp].a = here();
            node(n.kids[i]);
            jumps.push_back(emit(Inst::Jmp));
            prog[sp].b = here();
          } else {
            node(n.kids[i]);
          }
        }
        for (uint32_t j : jumps) prog[j].a = here();
        return;
      }
      case Node::Repeat: {
        const Node& e = n.kids[0];
        for (uint32_t i = 0; i < n.min; ++i) node(e);
        if (n.unbounded) {  // e*
          const uint32_t sp = emit(Inst::Split);
          node(e);
          emit(Inst::Jmp, sp);
          loop_split(sp, sp + 1, here(), n.greedy);
          return;
        }
        std::vector<uint32_t> splits;  // (e(e(e)?)?)?
        for (uint32_t i = n.min; i < n.max; ++i) {
          splits.push_back(emit(Inst::Split));
          node(e);
        }
        for (uint32_t sp : splits) loop_split(sp, sp + 1, here(), n.greedy);
        return;
      }
    }
  }
  void loop_split(uint32_t sp, uint32_t body, uint32_t out, bool greedy) {
    prog[sp].a = greedy ? body : out;
    prog[sp].b = greedy ? out : body;
  }
};

}  // namespace

LabelRegex::LabelRegex(const std::string& pattern) {
  std::vector<uint32_t> cps;
  if (!decode(pattern, cps, nullptr)) {
    verdict_ = RegexVerdict::Unsupported;
    message_ = "a pattern that is not valid UTF-8";
    return;
  }
  RegexParser parser(*this, std::move(cps));
  Node root;
  try {
    root = parser.parse();
  } catch (const RegexParser::Stop&) {
    prog_.clear();
    return;
  }
  // ^(?s:pattern)$ with the whole match as group 0
  Node wrapped;
  wrapped.k = Node::Cat;
  Node a;
  a.k = Node::Assert;
  a.c = kTextStart;
  wrapped.kids.push_back(a);
  wrapped.kids.push_back(std::move(root));
  a.c = kTextEnd;
  wrapped.kids.push_back(a);
  Compiler comp{prog_};
  try {
    comp.emit(Inst::Save, 0);
    comp.node(wrapped);
    comp.emit(Inst::Save, 1);
    comp.emit(Inst::Match);
  } catch (const std::length_error&) {
    prog_.clear();
    verdict_ = RegexVerdict::Unsupported;
    message_ = "a program above " + std::to_string(kMaxProgram) + " instructions";
  }
}

int LabelRegex::group_index(const std::string& name) const {
  for (const auto& [n, i] : names_)
    if (n == name) return (int)i;
  return -1;
}

bool LabelRegex::full_match(const std::string& input, std::vector<int64_t>& spans) const {
  std::vector<uint32_t> cps, offs;
  decode(input, cps, &offs);
  const size_t n = cps.size(), P = prog_.size(), S = 2 * (size_t)groups_;
  // a thread list: pcs in priority order, with their slots
  struct List {
    std::vector<uint32_t> pc;
    std::vector<int64_t> slots;
  };
  List cur, next;
  std::vector<uint64_t> seen(P, UINT64_MAX);
  std::vector<int64_t> work(S, -1), best;
  struct Frame {
    bool restore;
    uint32_t pc_or_slot;
    int64_t old;
  };
  std::vector<Frame> stack;
  uint64_t gen = 0;
  auto add = [&](List& list, uint32_t pc0, size_t pos) {
    stack.push_back({false, pc0, 0});
    while (!stack.empty()) {
      const Frame f = stack.back();
      stack.pop_back();
      if (f.restore) {
        work[f.pc_or_slot] = f.old;
        continue;
      }
      const uint32_t pc = f.pc_or_slot;
      if (seen[pc] == gen) continue;
      seen[pc] = gen;
      const Inst& in = prog_[pc];
      switch (in.op) {
        case Inst::Jmp: stack.push_back({false, in.a, 0}); break;
        case Inst::Split:
          stack.push_back({false, in.b, 0});
          stack.push_back({false, in.a, 0});
          break;
        case Inst::Save:
          stack.push_back({true, in.a, work[in.a]});
          work[in.a] = (int64_t)pos;
          stack.push_back({false, pc + 1, 0});
          break;
        case Inst::Assert: {
          bool ok = false;
          switch (in.a) {
            case kTextStart: ok = pos == 0; break;
            case kTextEnd: ok = pos == n; break;
            case kLineStart: ok = pos == 0 || cps[pos - 1] == '\n'; break;
            case kLineEnd: ok = pos == n || cps[pos] == '\n'; break;
          }
          if (ok) stack.push_back({false, pc + 1, 0});
          break;
        }
        default:
          list.pc.push_back(pc);
          list.slots.insert(list.slots.end(), work.begin(), work.end());
      }
    }
  };
  bool matched = false;
  add(cur, 0, 0);
  for (size_t pos = 0; pos <= n && !cur.pc.empty(); ++pos) {
    ++gen;
    next.pc.clear();
    next.slots.clear();
    for (size_t t = 0; t < cur.pc.size(); ++t) {
      const Inst& in = prog_[cur.pc[t]];
      const int64_t* sl = cur.slots.data() + t * S;
      if (in.op == Inst::Match) {  // (only at the end: the wrapped pattern ends in \z); lower priorities are cut
        best.assign(sl, sl + S);
        matched = true;
        break;
      }
      if (pos == n) continue;
      const uint32_t c = cps[pos];
      const bool step = in.op == Inst::Any || (in.op == Inst::AnyNoNL && c != '\n') || (in.op == Inst::Char && c == in.a) ||
                        (in.op == Inst::Class && classes_[in.a].has(c));
      if (!step) continue;
      std::copy(sl, sl + S, work.begin());
      add(next, cur.pc[t] + 1, pos + 1);
    }
    std::swap(cur, next);
  }
  if (!matched) return false;
  spans.assign(S, -1);
  for (size_t i = 0; i < S; i += 2)
    if (best[i] >= 0 && best[i + 1] >= 0) {
      spans[i] = offs[(size_t)best[i]];
      spans[i + 1] = offs[(size_t)best[i + 1]];
    }
  return true;
}

std::string LabelRegex::replace(const std::string& input, const std::string& replacement) const {
  std::vector<int64_t> spans;
  if (!full_match(input, spans)) return input;
  return expand_replacement(replacement, input, spans, names_);
}

bool valid_label_name(const std::string& name) {
  if (name.empty() || name.compare(0, 2, "__") == 0) return false;
  for (size_t i = 0; i < name.size(); ++i) {
    const unsigned char c = (unsigned char)name[i];
    const bool ok = c == '_' || is_ascii_alpha(c) || (i > 0 && is_ascii_digit(c));
    if (!ok) return false;
  }
  return true;
}

std::string expand_replacement(const std::string& replacement, const std::string& input, const std::vector<int64_t>& spans,
                               const std::vector<std::pair<std::string, uint32_t>>& names) {
  // DataFusion's regex_replace_posix_groups: `\` and the ASCII digits after it (possibly none) become ${digits}
  std::string rep;
  for (size_t i = 0; i < replacement.size(); ++i) {
    if (replacement[i] != '\\') {
      rep.push_back(replacement[i]);
      continue;
    }
    size_t j = i + 1;
    while (j < replacement.size() && is_ascii_digit((unsigned char)replacement[j])) ++j;
    rep += "${" + replacement.substr(i + 1, j - i - 1) + "}";
    i = j - 1;
  }
  auto append = [&](const std::string& ref, std::string& out) {
    // usize::from_str: an optional `+`, then one or more ASCII digits, no overflow
    size_t k = !ref.empty() && ref[0] == '+' ? 1 : 0;
    bool number = k < ref.size();
    uint64_t v = 0;
    for (size_t q = k; q < ref.size() && number; ++q) {
      if (!is_ascii_digit((unsigned char)ref[q]) || v > (UINT64_MAX - 9) / 10) number = false;
      else v = v * 10 + (uint64_t)(ref[q] - '0');
    }
    int64_t g = -1;
    if (number) {
      g = v < spans.size() / 2 ? (int64_t)v : -1;
    } else {
      for (const auto& [nm, idx] : names)
        if (nm == ref) g = idx;
    }
    if (g >= 0 && spans[2 * (size_t)g] >= 0)
      out.append(input, (size_t)spans[2 * (size_t)g], (size_t)(spans[2 * (size_t)g + 1] - spans[2 * (size_t)g]));
  };
  auto letter = [](unsigned char b) { return b == '_' || is_ascii_digit(b) || is_ascii_alpha(b); };
  std::string out;
  size_t i = 0;
  while (i < rep.size()) {
    const size_t d = rep.find('$', i);
    if (d == std::string::npos) break;
    out.append(rep, i, d - i);
    i = d;
    if (i + 1 < rep.size() && rep[i + 1] == '$') {
      out.push_back('$');
      i += 2;
      continue;
    }
    if (i + 1 < rep.size() && rep[i + 1] == '{') {
      const size_t close = rep.find('}', i + 2);
      if (close == std::string::npos) {
        out.push_back('$');
        ++i;
        continue;
      }
      append(rep.substr(i + 2, close - i - 2), out);
      i = close + 1;
      continue;
    }
    size_t e = i + 1;
    while (e < rep.size() && letter((unsigned char)rep[e])) ++e;
    if (e == i + 1) {
      out.push_back('$');
      ++i;
      continue;
    }
    append(rep.substr(i + 1, e - i - 1), out);
    i = e;
  }
  out.append(rep, i, std::string::npos);
  return out;
}

}  // namespace b2p
