// vb_debug_live_cuda_objects: the count the owning types of cuda_check.h keep, for leak checks of create / destroy paths.
#include "cuda_check.h"

extern "C" long long vb_debug_live_cuda_objects() { return vb::g_live_cuda_objects.load(); }
