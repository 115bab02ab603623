// tests/kat/queue_async_stubs.cpp — stand-ins for the asynchronous batch entry points of liburf_b200.so, linked into the
// ThreadSanitizer builds of urf_queue.cpp (no CUDA): the real-context worker refers to them, the stress programs never
// reach them (their queues are created around stand-in batch functions).
#include "../../include/urf.h"

extern "C" int urf_enqueue_batch(urf_ctx*, const float* const*, const int*, int, urf_result*, int8_t* const*) { return URF_ERR_NO_DEVICE; }
extern "C" int urf_finish_batch(urf_ctx*) { return URF_ERR_INVALID; }
