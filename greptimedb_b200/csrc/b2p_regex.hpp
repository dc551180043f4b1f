// b2p_regex.hpp — host C++17: the regular expressions of label_replace, as the reference runs them.
//
// The reference checks the raw pattern with Rust's `regex::Regex::new` (planner.rs:2557-2562) and then evaluates
// DataFusion's `regexp_replace(src, "^(?s:" + pattern + ")$", replacement)` (planner.rs:2581-2609): at most one match,
// which is then the whole value; no match returns the value unchanged.  This file restates that over UTF-8 code points
// with a Pike VM (a Thompson NFA simulated with capture slots): leftmost-first priority, so the captures are the ones
// Rust's `regex` reports, in O(pattern x input) time whatever the pattern.
//
// A pattern gets one of three verdicts:
//   Ok           literals; the escapes \n \t \r \f \v \a \xHH \x{H..} and an escaped meta character (\.+*?()|[]{}^$#&-~);
//                `.`; bracket classes with ranges, negation and the ASCII classes [[:alnum:]] .. [[:xdigit:]] (and
//                [[:^name:]]); `|`; groups ( ), (?: ), (?P<name> ), (?<name> ) with ASCII names [A-Za-z_][A-Za-z0-9_]*;
//                * + ? {n} {n,} {n,m}, greedy and lazy; ^ $ \A \z; the flags s, m and U, set with (?flags) or scoped
//                with (?flags: ), `-` negating.
//   Invalid      what `Regex::new` rejects: an unbalanced group, a repetition with nothing to repeat, {n,m} with m < n,
//                look-around ((?= (?! (?<= (?<!), a backreference or octal (\0 .. \9), (?P= ), an unknown escape letter,
//                a malformed \x escape, an unknown or repeated flag, an empty or dangling flag group, an empty or
//                duplicate group name, an unclosed class, a reversed class range, an unknown [[:name:]].
//   Unsupported  valid in Rust, refused here (the plan node raises a Plan error, so the query stays on the CPU):
//                \d \D \w \W \s \S \b \B \p \P \u \U \< \> (Unicode-aware in Rust, or rare); the flags i, x, u, R; a
//                repetition of a repetition or of an assertion; a counted repetition above 1000 or a `{` that does not
//                read as {n}, {n,} or {n,m}; a program above kMaxProgram instructions; nesting deeper than 64;
//                nested classes and the class set operators && -- ~~; a `-` inside a class that is neither first, last
//                nor a range; a superfluous escape of other punctuation, a space or a non-ASCII character; a group name
//                outside ASCII [A-Za-z_][A-Za-z0-9_]*; a pattern that is not valid UTF-8.
// Widening the supported list is a change of its own: each construct needs Rust's exact semantics.
//
// The replacement is DataFusion's: `\N` (a backslash and ASCII digits, possibly none) is rewritten to `${N}`, then the
// regex crate's expansion: `$$` is `$`; `$name` takes the longest run of [_0-9A-Za-z]; `${name}` takes everything up to
// the next `}`; a name that parses as an unsigned integer is a group number; a group that does not exist or did not
// take part expands to nothing; a `$` that starts no reference stays a `$`.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace b2p {

enum class RegexVerdict { Ok = 0, Invalid = 1, Unsupported = 2 };

class LabelRegex {
 public:
  static constexpr size_t kMaxProgram = 20000;
  explicit LabelRegex(const std::string& pattern);
  RegexVerdict verdict() const { return verdict_; }
  const std::string& message() const { return message_; }  // why the verdict is not Ok
  // regexp_replace(input, "^(?s:" + pattern + ")$", replacement): the expanded replacement when the whole input
  // matches, else the input unchanged.  Needs verdict() == Ok.
  std::string replace(const std::string& input, const std::string& replacement) const;
  // the same, without the replacement: whether the whole input matches and each group's byte span ([2 * groups],
  // -1 for a group that did not take part; group 0 is the whole match)
  bool full_match(const std::string& input, std::vector<int64_t>& spans) const;

  struct Inst {
    enum Op : uint8_t { Char, Any, AnyNoNL, Class, Split, Jmp, Save, Assert, Match } op;
    uint32_t a = 0, b = 0;  // Char: code point; Class: class index; Split: x, y; Jmp: x; Save: slot; Assert: kind
  };
  struct CharClass {
    bool negated = false;
    std::vector<std::pair<uint32_t, uint32_t>> ranges;  // inclusive
    bool has(uint32_t c) const;
  };

 private:
  friend class RegexParser;
  RegexVerdict verdict_ = RegexVerdict::Ok;
  std::string message_;
  std::vector<Inst> prog_;
  std::vector<CharClass> classes_;
  uint32_t groups_ = 1;  // capture groups, the whole match included
  std::vector<std::pair<std::string, uint32_t>> names_;
  int group_index(const std::string& name) const;  // -1 when none
};

// Rust's check on a destination label name (planner.rs:2504-2515): not starting with "__" and ^[a-zA-Z_][a-zA-Z0-9_]*$
bool valid_label_name(const std::string& name);

// the regex crate's expansion of `replacement` (after DataFusion's \N rewrite) over `input` and the spans of full_match()
std::string expand_replacement(const std::string& replacement, const std::string& input, const std::vector<int64_t>& spans,
                               const std::vector<std::pair<std::string, uint32_t>>& names);

}  // namespace b2p
