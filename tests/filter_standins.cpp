// TEST INFRASTRUCTURE — the filter's CPU stand-ins for rcp.approx.ftz.f32 / sqrt.approx.ftz.f32 (nvc_filter.cuh under NVC_EMU,
// without the NVF_PERTURB jitter) as a plain host loop, so that tests/test_filter_approx.py can evaluate them on the billions of
// inputs it compares with the device.  Built by that test with g++ against tests/cuda_emu/include.
#include "cuda_runtime.h"

#include "nvc_filter.cuh"

extern "C" void nvf_standins(int op, const uint32_t* in, uint32_t* out, uint64_t n)
{
	for (uint64_t i = 0; i < n; ++i)
	{
		const float x = __uint_as_float(in[i]);
		out[i] = __float_as_uint(op == 0 ? nvc::nvf_rcp(x) : nvc::nvf_sqrt(x));
	}
}
