// What every C++ suite of the host mirror (tests/cpp/*_suite.cpp) shares: the failed-check counter and CHECK, throws, the
// GPU requirement and the closing line.  A suite exits 3 without a GPU (there is no CPU fallback), 1 on a failed check.
#pragma once

#include "marlin_b200.hpp"

#include <cstdio>
#include <exception>

inline int failed = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++failed; } } while (0)

// f() throws an Ex; any other exception, or none, is a no
template <class Ex = std::exception, class F>
bool throws(F f) {
    try { f(); } catch (const Ex&) { return true; } catch (...) { return false; }
    return false;
}

// if (!require_gpu()) return 3;  -- the first call into the library throws its "no CPU fallback" error without a GPU
inline bool require_gpu() {
    try {
        marlin::Context::get();
    } catch (const std::exception& e) {
        std::printf("cannot initialise marlin_b200: %s\n", e.what());
        return false;
    }
    return true;
}

// return finish("... suite");
inline int finish(const char* name) {
    std::printf("%s: %d failed checks\n", name, failed);
    return failed ? 1 : 0;
}
