// Index samples drawn the way a std::mt19937(42) and std::uniform_int_distribution<std::mt19937::result_type> of the
// host's libstdc++ draw them, for the rotation RANSAC oracle's sample stream to be compared with.
//
//   uniform_int_host pin          the 10000th output of a default-seeded std::mt19937
//   uniform_int_host              reads lines "n size count" and prints, per line, count samples of size distinct
//                                 indices in [0, n) (a repeated index is drawn again), from a fresh mt19937(42)
#include <cstdio>
#include <cstring>
#include <random>
#include <vector>

int main(int argc, char** argv) {
  if (argc > 1 && !std::strcmp(argv[1], "pin")) {
    std::mt19937 g;
    for (int i = 0; i < 9999; ++i) g();
    std::printf("%u\n", (unsigned)g());
    return 0;
  }
  long long n;
  int size, count;
  while (std::scanf("%lld %d %d", &n, &size, &count) == 3) {
    std::mt19937 g(42);
    std::uniform_int_distribution<std::mt19937::result_type> d(0, (std::mt19937::result_type)(n - 1));
    for (int s = 0; s < count; ++s) {
      std::vector<unsigned long> idx;
      for (int k = 0; k < size; ++k) {
        unsigned long v;
        bool again;
        do {
          v = d(g);
          again = false;
          for (unsigned long u : idx) again |= u == v;
        } while (again);
        idx.push_back(v);
        std::printf("%lu ", v);
      }
    }
    std::printf("\n");
    std::fflush(stdout);
  }
  return 0;
}
