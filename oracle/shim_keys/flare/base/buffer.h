// Stand-in for flare's NoncontiguousBuffer: flare/base/crypto/blake3.cc only iterates one
// (Blake3(const NoncontiguousBuffer&)), and the harness never calls that overload.
#pragma once
#include <cstdint>
#include <string_view>
#include <vector>
namespace flare {
class NoncontiguousBuffer {
 public:
  std::vector<std::string_view>::const_iterator begin() const { return parts_.begin(); }
  std::vector<std::string_view>::const_iterator end() const { return parts_.end(); }

 private:
  std::vector<std::string_view> parts_;
};
}  // namespace flare
