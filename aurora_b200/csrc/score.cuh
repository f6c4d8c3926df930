// Host-side argument checks shared by the score (score.cu) and spectrum (spectra.cu) entry points.
#pragma once

#include "common.h"

namespace ab {

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The checks every entry point makes on its descriptor array itself.
inline int check_array(const void* fields, int32_t n_fields, size_t field_bytes, size_t want, const char* type,
                       int max_fields, const char* who) {
  AB_CHECK_ARG(field_bytes == want, "%s: field_bytes %zu != sizeof(%s) %zu", who, field_bytes, type, want);
  AB_CHECK_ARG(n_fields >= 0, "%s: n_fields %d < 0", who, n_fields);
  if (n_fields > max_fields) {
    set_error("%s: %d fields in one call, at most %d are supported", who, n_fields, max_fields);
    return AB_ERR_UNSUPPORTED;
  }
  AB_CHECK_ARG(n_fields == 0 || fields, "%s: null argument", who);
  return AB_OK;
}

}  // namespace ab
