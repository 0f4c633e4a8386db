// args.hpp -- the command-line parser of the tools of this package (`daccord`, `computeintrinsicqv`), in the style of libmaus2's
// ArgParser: short options carry their value attached (-w40), long options are matched by the longest name of `longs` they start with
// (--batchreads7, --batchreads=7); options precede the positional arguments.
#pragma once
#include <cctype>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace dhost {

struct Args { std::map<std::string, std::string> opt; std::vector<std::string> pos; };
// longs: the long option names the tool accepts, nullptr-terminated; false (message printed) on an unknown long option
inline bool parse_args(int argc, char** argv, const char* const* longs, Args& A) {
  int i = 1;
  for (; i < argc; ++i) {
    std::string s = argv[i];
    if (s.size() >= 2 && s[0] == '-' && s[1] == '-') {
      std::string body = s.substr(2), key, val; bool found = false;
      for (int j = 0; longs[j]; ++j) { size_t n = strlen(longs[j]); if (body.compare(0, n, longs[j]) == 0 && n > key.size()) { key = longs[j]; found = true; } }
      if (!found) { fprintf(stderr, "[E] unknown option %s\n", s.c_str()); return false; }
      val = body.substr(key.size());
      if (!val.empty() && val[0] == '=') val = val.substr(1);
      A.opt[key] = val;
    } else if (s.size() >= 2 && s[0] == '-' && !isdigit((unsigned char)s[1])) {
      A.opt[std::string(1, s[1])] = s.substr(2);          // libmaus2 ArgParser style: value attached (-w40)
    } else break;                                          // options must precede positionals (README.md:99)
  }
  for (; i < argc; ++i) A.pos.push_back(argv[i]);
  return true;
}

}  // namespace dhost
