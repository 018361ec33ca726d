// The formatter core of the matrix-file writer (marlin_b200/csrc/text.h) built as plain host C++: reads one input per
// line from stdin and prints its token on a line of its own.
//   text_driver d   inputs are 64-bit patterns of doubles in hex; tokens are Double.toString's (mt_utils._jdouble)
//   text_driver l   inputs are signed decimal int64; tokens are Long.toString's
#include "text.h"

#include <cinttypes>
#include <cstdio>
#include <cstring>

int main(int argc, char** argv) {
    using namespace mb::text;
    static const uint64_t pow5[] = MB_TEXT_POW5_TABLE;
    static const uint64_t pow5_inv[] = MB_TEXT_POW5_INV_TABLE;
    if (argc != 2 || (std::strcmp(argv[1], "d") != 0 && std::strcmp(argv[1], "l") != 0)) {
        std::fprintf(stderr, "usage: text_driver d|l < inputs\n");
        return 2;
    }
    const bool doubles = argv[1][0] == 'd';
    char line[64], tok[TEXT_TOKEN_MAX + 1];
    while (std::fgets(line, sizeof line, stdin)) {
        int n;
        if (doubles) {
            uint64_t bits = 0;
            if (std::sscanf(line, "%" SCNx64, &bits) != 1) return 2;
            const Token t = classify(bits, pow5, pow5_inv);
            n = write_token(t, tok);
            if (n != token_length(t)) {
                std::fprintf(stderr, "length mismatch at %016" PRIx64 "\n", bits);
                return 1;
            }
        } else {
            int64_t v = 0;
            if (std::sscanf(line, "%" SCNd64, &v) != 1) return 2;
            n = write_long(v, tok);
        }
        tok[n] = '\n';
        std::fwrite(tok, 1, (size_t)n + 1, stdout);
    }
    return 0;
}
