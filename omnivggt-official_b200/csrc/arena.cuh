// Carving of a caller's workspace: nothing in libovg allocates device memory.  A component's layout function takes its buffers
// from an Arena in order; run over a null base (a size query) it forms no pointer and only measures.
#pragma once

namespace ovg {

struct Arena {
  char* base;
  long long off = 0;
  explicit Arena(void* b) : base(static_cast<char*>(b)) {}
  void* take(long long bytes) {          // each buffer starts on a 256-byte boundary
    const long long at = (off + 255) & ~255LL;
    off = at + bytes;
    return base ? base + at : nullptr;
  }
  template <typename T>
  T* get(long long n) { return static_cast<T*>(take(n * static_cast<long long>(sizeof(T)))); }
  long long bytes() const { return (off + 255) & ~255LL; }   // the layout's size in whole 256-byte blocks
};

}  // namespace ovg
