// The shim's logging.h plus FLARE_DCHECK, which flare/base/encoding/detail/hex_chars.h uses (oracle/keys.mk puts this
// directory in front of oracle/shim).
#pragma once
#include "../../../shim/flare/base/logging.h"
#define FLARE_DCHECK(expr, ...) FLARE_CHECK(expr)
