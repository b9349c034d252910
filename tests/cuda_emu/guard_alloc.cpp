// TEST INFRASTRUCTURE — guarded device allocations for the emulated library (tests/emu_lib.py).  Linked into it with
// -Wl,--wrap=calloc,--wrap=free, so that the emulated cudaMalloc / cudaFree (calloc / free) come here.  While emu_guard_allocations(1) is in effect, every allocation is placed so
// that it ends exactly at an inaccessible page: a kernel that reads past the end of a context-owned buffer faults, the
// CPU counterpart of compute-sanitizer's memcheck.  Otherwise the calls go to the C library unchanged.
#include <stddef.h>
#include <string.h>
#include <sys/mman.h>
#include <unistd.h>

#include <map>
#include <utility>

extern "C" void* __real_calloc(size_t n, size_t size);
extern "C" void __real_free(void* p);

namespace
{
bool g_guard = false;
std::map<void*, std::pair<char*, size_t>>& guarded() // user pointer -> (mapping, mapping length)
{
	static std::map<void*, std::pair<char*, size_t>> m;
	return m;
}
} // namespace

extern "C" void emu_guard_allocations(int on)
{
	g_guard = on != 0;
}

// guarded allocations not yet freed
extern "C" int emu_guarded_live()
{
	return int(guarded().size());
}

extern "C" void* __wrap_calloc(size_t n, size_t size)
{
	if (!g_guard)
		return __real_calloc(n, size);
	const size_t bytes = n * size;
	const size_t page = size_t(sysconf(_SC_PAGESIZE));
	const size_t span = (bytes + page - 1) / page * page;
	void* m = mmap(nullptr, span + page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
	if (m == MAP_FAILED)
		return nullptr;
	char* base = static_cast<char*>(m);
	if (mprotect(base + span, page, PROT_NONE) != 0)
	{
		munmap(m, span + page);
		return nullptr;
	}
	void* p = base + span - bytes; // anonymous pages are zero-filled, like calloc
	guarded()[p] = { base, span + page };
	return p;
}

extern "C" void __wrap_free(void* p)
{
	auto it = guarded().find(p);
	if (it == guarded().end())
	{
		__real_free(p);
		return;
	}
	munmap(it->second.first, it->second.second);
	guarded().erase(it);
}
