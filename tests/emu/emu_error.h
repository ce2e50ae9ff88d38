// TEST HARNESS ONLY — the message of the last emu_* entry that failed on this thread; emu_last_error() (emu_capi.cu) returns it. The
// emulated mb2_* C-ABI keeps its own, mb2_last_error().
#pragma once
#include <string>

inline thread_local std::string g_emuErr;
