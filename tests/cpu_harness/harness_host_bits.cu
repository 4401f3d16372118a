// TEST INFRASTRUCTURE (CPU suite only): the CPU emulation of k_place_bits, the bitmap kernel of dfd_shuffle_host's
// compaction (csrc/dfd_exchange.cu), registered by name with the stand-in runtime's cudaLaunchKernel.  Linked with
// harness_exchange.cu (the push transport's kernels) by tests/test_host_shuffle_cpu_harness.py.
#include <cstdint>
#include <cstring>

namespace {
struct FakeDim3 { unsigned x, y, z; };
typedef int (*HarnessKernel)(FakeDim3 grid, FakeDim3 block, void** args);
extern "C" void harness_register_kernel(const char* name_fragment, HarnessKernel fn);

template <typename T>
T arg(void** args, int i) { T v; memcpy(&v, args[i], sizeof v); return v; }

// the run descriptor of k_place_bits — a COPY of the private struct in csrc/dfd_exchange.cu (same field order and types)
struct BitRun {
    const unsigned* src;
    unsigned* dst;
    long long dst_bit, n;
    int first_block;
};

// k_place_bits(const BitRun* runs, int n_runs): bit k of src -> bit dst_bit + k of dst, OR-ed in (the destination's other
// bits are left as they are: the library zeroes the destination before the launch)
int cpu_place_bits(FakeDim3, FakeDim3, void** a) {
    const BitRun* runs = arg<const BitRun*>(a, 0);
    const int n_runs = arg<int>(a, 1);
    for (int i = 0; i < n_runs; ++i) {
        const BitRun& r = runs[i];
        for (long long k = 0; k < r.n; ++k)
            if ((r.src[k >> 5] >> (k & 31)) & 1u) r.dst[(r.dst_bit + k) >> 5] |= 1u << ((r.dst_bit + k) & 31);
    }
    return 0;
}

__attribute__((constructor)) void register_host_bits_kernel() { harness_register_kernel("k_place_bits", cpu_place_bits); }
}  // namespace
