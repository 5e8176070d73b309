// Unity translation unit of libovp.so (one TU: kernels defined in one file are launched from another).
#include "linalg.cu"
#include "cholfused.cu"
#include "cholpanel.cu"
#include "ekf.cu"
#include "features.cu"
#include "capi.cu"
#include "capi2.cu"
#include "planefit.cu"
#include "anchors.cu"
#ifdef OVP_DEBUG // libovp_debug.so only: micro-benchmarks and kernel-level test hooks (include/ovp_debug.h)
#include "debug_hooks.cu"
#endif
