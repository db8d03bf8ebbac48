/* png_common.cuh -- what PNG load (png.cu) and PNG save (png_encode.cu) share. */
#pragma once

#include <cstdlib>

namespace vb200 {

/* PNG 2nd edition 9.2: Paeth's predictor */
__host__ __device__ __forceinline__ int
paeth(int a, int b, int c)
{
	const int p = a + b - c;
	const int pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
	return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

} // namespace vb200
