#include "../../include/mi3d.h"
extern "C" const char* mi3d_version(void) { return "mi3d-b200 0.1 (sm_90a)"; }
