// TEST INFRASTRUCTURE ONLY: built with the flags of libstitch_b200_emu_san.so and loaded the same way, so that
// tests/test_emu_memory.py can show the sanitizers are armed in its child processes: a float -> int conversion out of
// range (UBSan reports it and goes on) and a one-past-the-end read of a heap block (AddressSanitizer stops the process).
#include <cstdlib>

extern "C" __attribute__((visibility("default"))) int sb_probe_cast(float v)
{
    return (int)v;
}

extern "C" __attribute__((visibility("default"))) int sb_probe_overread(int n)
{
    volatile unsigned char *p = (volatile unsigned char *)std::malloc((size_t)n);
    for (int i = 0; i < n; ++i) p[i] = (unsigned char)i;
    const int v = p[n];
    std::free((void *)p);
    return v;
}
