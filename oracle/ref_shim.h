// TEST INFRASTRUCTURE ONLY.
//
// The one error path of every reference shim: an entry point that catches a reference exception stores its
// message with ref_set_last_error and returns -1 (or a null handle); oracle/ref.py reads the message back with
// ref_last_error.  Both live in ref_shim.cpp, so libfaiss_ref.so holds the only error slot and every shim
// library, linked against it, writes to that slot.
//
//   int ref_x(...) { REF_TRY ...; REF_CATCH }                       0, or -1 on an exception
//   void* ref_x_new(...) { REF_TRY ...; return h; REF_CATCH_RET(nullptr) }

#pragma once

#include <exception>

extern "C" void ref_set_last_error(const char* msg);

#define REF_TRY try {
#define REF_CATCH_RET(fail)           \
    }                                 \
    catch (const std::exception& e) { \
        ref_set_last_error(e.what()); \
        return fail;                  \
    }
#define REF_CATCH REF_CATCH_RET(-1) return 0;
