// migan_last_error(): the calling thread's last error (abi_error.h).
#include "abi_error.h"

extern "C" const char* migan_last_error(void) { return migan::g_last_error.c_str(); }
