// tests/host_emul/ge_trace.h — the branch log of the group law (ge.cuh SV_GE_TRACE), shared by every host build that logs.
// One byte per addition, SV_GE_MIXED / SV_GE_FULL | SV_GE_ADD_*, kept per thread and only while a caller of
// emul_trace_begin / emul_trace_end (emul.cpp) has switched it on.  Include before the kernel headers.
#pragma once
#include <vector>
std::vector<unsigned char>*& emul_trace_log();  // emul.cpp: the calling thread's log, null while logging is off
#define SV_GE_TRACE(ev) do { if (std::vector<unsigned char>* t_ = emul_trace_log()) t_->push_back((unsigned char)(ev)); } while (0)
