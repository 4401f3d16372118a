// TEST INFRASTRUCTURE (CPU suite only): the stand-in CUDA runtime of fake_cudart.cpp with its events accounted for, for the
// device-output harness that tests/test_exec_device_output_cpu_harness.py links in place of fake_cudart.cpp.  A device-output
// operator owns one event per device chunk, so that module checks that every event is destroyed (harness_live_events) and
// that a failing event creation is an error, never a crash or a leak (harness_fail_nth_event).  The stand-in's own event
// entry points are compiled under other names and wrapped here; everything else is fake_cudart.cpp as it stands.
#define cudaEventCreateWithFlags fake_cudart_event_create_with_flags
#define cudaEventCreate fake_cudart_event_create
#define cudaEventDestroy fake_cudart_event_destroy
#include "fake_cudart.cpp"
#undef cudaEventCreateWithFlags
#undef cudaEventCreate
#undef cudaEventDestroy

extern "C" {
static std::atomic<long> g_live_events{0};    // events created and not yet destroyed
static std::atomic<long> g_fail_event_in{0};  // > 0: fail the n-th cudaEventCreateWithFlags from now
long harness_live_events(void) { return g_live_events.load(); }
void harness_fail_nth_event(long n) { g_fail_event_in.store(n); }

cudaError_t_ cudaEventCreateWithFlags(void** e, unsigned flags) {
    *e = nullptr;
    long v = g_fail_event_in.load();
    while (v > 0)
        if (g_fail_event_in.compare_exchange_weak(v, v - 1)) {
            if (v == 1) return 2;  // cudaErrorMemoryAllocation
            break;
        }
    g_live_events.fetch_add(1);
    return fake_cudart_event_create_with_flags(e, flags);
}
cudaError_t_ cudaEventCreate(void** e) {
    g_live_events.fetch_add(1);
    return fake_cudart_event_create(e);
}
cudaError_t_ cudaEventDestroy(void* e) {
    if (e) g_live_events.fetch_sub(1);
    return fake_cudart_event_destroy(e);
}
}
