// LIKE / NOT LIKE [INSENSITIVE] over a string dictionary, on the host.
//
// A restatement of the reference's LikeMatcher (expression/evaluation/like_matcher.{hpp,cpp}) as
// ColumnLikeTableScanImpl::_find_matches_in_dictionary applies it (column_like_table_scan_impl.cpp:75-140): the pattern
// is matched once per dictionary entry, and the device then scans value-IDs against the resulting bitmap. Strings never
// reach the GPU.
//
//   tokens      `_` = one character, `%` = any run of characters, everything else literal; no escape character.
//   forms       [str, %] starts-with; [%, str] ends-with; [%, str, %] contains; %str%str... (tokens alternate %, str,
//               starting with %) ordered multiple-contains, each string searched from the end of the previous match;
//               anything else an anchored ECMAScript std::regex with `.`, `^`, `$`, `+`, `?`, `(`, `)`, `{`, `}`, `|`,
//               `*` and `\` escaped, `%` -> `.*` and `_` -> `.`. The regex `.` does not match '\n' or '\r', the special
//               forms match any byte: `a%b` rejects "a\nb", `%a%b%` accepts it.
//   insensitive pattern and input are lowered byte by byte as std::tolower does in the C locale (A-Z only).
//   NOT         inverts the matcher.
#include <regex>
#include <string>
#include <string_view>
#include <vector>

#include "internal.hpp"

namespace hyb {
namespace {

enum class LikeForm { kStartsWith, kEndsWith, kContains, kMultipleContains, kRegex };

struct LikeMatcher {
  LikeForm form = LikeForm::kRegex;
  std::vector<std::string> strings;
  std::regex regex;
  bool insensitive = false;
  bool invert = false;
};

char lower_ascii(char c) { return c >= 'A' && c <= 'Z' ? static_cast<char>(c - 'A' + 'a') : c; }

struct Token {
  int wildcard;  // 0: literal `text`, 1: `_`, 2: `%`
  std::string text;
};

std::vector<Token> like_tokens(const std::string& pattern) {
  std::vector<Token> tokens;
  for (size_t at = 0; at < pattern.size();) {
    if (pattern[at] == '_' || pattern[at] == '%') {
      tokens.push_back({pattern[at] == '_' ? 1 : 2, {}});
      ++at;
    } else {
      const size_t next = pattern.find_first_of("_%", at);
      const size_t end = next == std::string::npos ? pattern.size() : next;
      tokens.push_back({0, pattern.substr(at, end - at)});
      at = end;
    }
  }
  return tokens;
}

std::string like_to_regex(const std::string& pattern) {
  std::string regex = "^";
  for (const char c : pattern) {
    switch (c) {
      case '\\':
      case '.':
      case '^':
      case '$':
      case '+':
      case '?':
      case '(':
      case ')':
      case '{':
      case '}':
      case '|':
      case '*':
        regex += '\\';
        regex += c;
        break;
      case '%':
        regex += ".*";
        break;
      case '_':
        regex += '.';
        break;
      default:
        regex += c;
        break;
    }
  }
  return regex + "$";
}

int compile_like(const std::string& raw_pattern, int32_t condition, LikeMatcher& matcher) {
  matcher.insensitive = condition == HYB_PRED_LIKE_INSENSITIVE || condition == HYB_PRED_NOT_LIKE_INSENSITIVE;
  matcher.invert = condition == HYB_PRED_NOT_LIKE || condition == HYB_PRED_NOT_LIKE_INSENSITIVE;
  std::string pattern = raw_pattern;
  if (matcher.insensitive) {
    for (char& c : pattern) c = lower_ascii(c);
  }
  const auto tokens = like_tokens(pattern);
  if (tokens.size() == 2 && tokens[0].wildcard == 0 && tokens[1].wildcard == 2) {
    matcher.form = LikeForm::kStartsWith;
    matcher.strings = {tokens[0].text};
    return HYB_OK;
  }
  if (tokens.size() == 2 && tokens[0].wildcard == 2 && tokens[1].wildcard == 0) {
    matcher.form = LikeForm::kEndsWith;
    matcher.strings = {tokens[1].text};
    return HYB_OK;
  }
  if (tokens.size() == 3 && tokens[0].wildcard == 2 && tokens[1].wildcard == 0 && tokens[2].wildcard == 2) {
    matcher.form = LikeForm::kContains;
    matcher.strings = {tokens[1].text};
    return HYB_OK;
  }
  // Multiple-contains: the tokens alternate `%`, literal, `%`, ... from the first one on. As in the reference, the
  // sequence need not end with `%` (`%a%b` is searched like `%a%b%`), and "" and "%" contain no literal: they match
  // every string.
  bool alternating = true;
  std::vector<std::string> strings;
  for (size_t i = 0; i < tokens.size() && alternating; ++i) {
    const bool expect_any = i % 2 == 0;
    if (expect_any ? tokens[i].wildcard != 2 : tokens[i].wildcard != 0) {
      alternating = false;
    } else if (!expect_any) {
      strings.push_back(tokens[i].text);
    }
  }
  if (alternating) {
    matcher.form = LikeForm::kMultipleContains;
    matcher.strings = std::move(strings);
    return HYB_OK;
  }
  matcher.form = LikeForm::kRegex;
  try {
    matcher.regex = std::regex(like_to_regex(pattern), std::regex::ECMAScript | std::regex::optimize);
  } catch (const std::regex_error& error) {  // e.g. an unbalanced `[`: the reference throws as well
    return fail(HYB_ERR_INVALID, std::string("LIKE pattern is not a valid regular expression: ") + error.what());
  }
  return HYB_OK;
}

bool like_match(const LikeMatcher& matcher, std::string_view input, std::string& lowered) {
  if (matcher.insensitive) {
    lowered.assign(input.begin(), input.end());
    for (char& c : lowered) c = lower_ascii(c);
    input = lowered;
  }
  bool match = false;
  switch (matcher.form) {
    case LikeForm::kStartsWith:
      match = input.substr(0, matcher.strings[0].size()) == matcher.strings[0];
      break;
    case LikeForm::kEndsWith:
      match = input.size() >= matcher.strings[0].size() &&
              input.substr(input.size() - matcher.strings[0].size()) == matcher.strings[0];
      break;
    case LikeForm::kContains:
      match = input.find(matcher.strings[0]) != std::string_view::npos;
      break;
    case LikeForm::kMultipleContains: {
      match = true;
      size_t at = 0;
      for (const auto& needle : matcher.strings) {
        const size_t found = input.find(needle, at);
        if (found == std::string_view::npos) {
          match = false;
          break;
        }
        at = found + needle.size();
      }
      break;
    }
    case LikeForm::kRegex:
      match = std::regex_match(input.begin(), input.end(), matcher.regex);
      break;
  }
  return match != matcher.invert;
}

}  // namespace

int like_match_dictionaries(const char* pattern, uint64_t pattern_length, int32_t condition,
                            const LikeDictionary* dictionaries, size_t dictionary_count, uint32_t* out_words,
                            uint64_t* out_match_count) {
  HYB_CHECK(pattern || pattern_length == 0, HYB_ERR_INVALID, "NULL pattern");
  HYB_CHECK(condition >= HYB_PRED_LIKE && condition <= HYB_PRED_NOT_LIKE_INSENSITIVE, HYB_ERR_INVALID,
            "not a LIKE condition: " + std::to_string(condition));
  for (size_t d = 0; d < dictionary_count; ++d) {
    const LikeDictionary& dictionary = dictionaries[d];
    HYB_CHECK(dictionary.count == 0 || (dictionary.offsets && out_words), HYB_ERR_INVALID, "NULL dictionary or output");
    // a dictionary of empty strings has no characters: its `chars` may legitimately be NULL
    HYB_CHECK(dictionary.count == 0 || dictionary.chars || dictionary.offsets[dictionary.count] == dictionary.offsets[0],
              HYB_ERR_INVALID, "NULL dictionary characters");
  }
  LikeMatcher matcher;
  HYB_TRY(compile_like(std::string(pattern ? pattern : "", pattern_length), condition, matcher));
  std::string lowered;
  uint64_t matches = 0;
  uint32_t* words = out_words;
  for (size_t d = 0; d < dictionary_count; ++d) {
    const LikeDictionary& dictionary = dictionaries[d];
    const char* chars = dictionary.chars ? dictionary.chars : "";
    for (uint32_t word = 0; word < (dictionary.count + 31) / 32; ++word) words[word] = 0;
    for (uint32_t entry = 0; entry < dictionary.count; ++entry) {
      const std::string_view value(chars + dictionary.offsets[entry],
                                   dictionary.offsets[entry + 1] - dictionary.offsets[entry]);
      if (like_match(matcher, value, lowered)) {
        words[entry >> 5] |= 1u << (entry & 31);
        ++matches;
      }
    }
    words += (dictionary.count + 31) / 32;
  }
  if (out_match_count) *out_match_count = matches;
  return HYB_OK;
}

}  // namespace hyb

using namespace hyb;

extern "C" {

int hyb_like_dictionary_matches(const char* pattern, uint64_t pattern_length, int32_t condition, const char* chars,
                                const uint64_t* offsets, uint32_t count, uint32_t* out_words, uint32_t* out_match_count) {
  const LikeDictionary dictionary{chars, offsets, count};
  uint64_t matches = 0;
  HYB_TRY(like_match_dictionaries(pattern, pattern_length, condition, &dictionary, 1, out_words, &matches));
  if (out_match_count) *out_match_count = static_cast<uint32_t>(matches);
  return HYB_OK;
}

}  // extern "C"
