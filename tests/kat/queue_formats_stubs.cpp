// tests/kat/queue_formats_stubs.cpp — stand-in for urf_enqueue_cloud2_batch_mixed of liburf_b200.so, linked into the
// ThreadSanitizer builds of urf_queue.cpp (no CUDA): the real-context worker of a formats queue refers to it, the stress
// programs never reach it (their queues are created around stand-in batch functions).
#include "../../include/urf.h"

extern "C" int urf_enqueue_cloud2_batch_mixed(urf_ctx*, const void* const*, const int*, const urf_cloud2_format*, int, urf_result*,
                                              int8_t* const*) {
  return URF_ERR_NO_DEVICE;
}
