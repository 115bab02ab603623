// tests/kat/queue_params_stubs.cpp — stand-in for urf_set_params_next of liburf_b200.so, linked into the ThreadSanitizer
// builds of urf_queue.cpp (no CUDA): the real-context worker refers to it, the stress programs never reach it (their queues
// are created around stand-in batch functions and apply parameter sets through urf_queue_set_params_hook).
#include "../../include/urf.h"

extern "C" int urf_set_params_next(urf_ctx*, const urf_params*) { return URF_ERR_NO_DEVICE; }
