// lancir_types_shim.cpp -- upstream CLancIR (lancir.h, unmodified, from REF) behind a C entry point for
// every element type upstream lists (lancir.h:373-381): TEST INFRASTRUCTURE, the reference of
// tests/test_lancir_types.py and tests/test_gpu_lancir_types.py.  Built by oracle/types.mk with the
// pinned flags into _ref/liblancir_types_ref.so.

#include <cstdint>

#include "lancir.h"

namespace {

template< typename TI >
int resize_out( const int tout, const void* src, int sw, int sh, void* dst,
	int nw, int nh, int C, const avir::CLancIRParams& p )
{
	avir::CLancIR r;

	switch( tout )
	{
		case 0: return r.resizeImage( (const TI*) src, sw, sh, (uint8_t*) dst, nw, nh, C, &p );
		case 1: return r.resizeImage( (const TI*) src, sw, sh, (uint16_t*) dst, nw, nh, C, &p );
		case 2: return r.resizeImage( (const TI*) src, sw, sh, (float*) dst, nw, nh, C, &p );
		case 3: return r.resizeImage( (const TI*) src, sw, sh, (double*) dst, nw, nh, C, &p );
		case 4: return r.resizeImage( (const TI*) src, sw, sh, (uint32_t*) dst, nw, nh, C, &p );
	}

	return -1;
}

} // namespace

extern "C" {

// CLancIR::resizeImage (lancir.h:386).  tin / tout: avirb200_dtype codes, 0 = uint8_t, 1 = uint16_t,
// 2 = float, 3 = double, 4 = uint32_t.  Returns upstream's return value, -1 for a code outside 0..4.
int lancir_types_ref_resize( int tin, int tout, const void* src, int sw, int sh,
	void* dst, int nw, int nh, int C, int srcssize, int newssize,
	double kx, double ky, double ox, double oy, double la )
{
	avir::CLancIRParams p( srcssize, newssize, kx, ky, ox, oy );
	p.la = la;

	switch( tin )
	{
		case 0: return resize_out< uint8_t >( tout, src, sw, sh, dst, nw, nh, C, p );
		case 1: return resize_out< uint16_t >( tout, src, sw, sh, dst, nw, nh, C, p );
		case 2: return resize_out< float >( tout, src, sw, sh, dst, nw, nh, C, p );
		case 3: return resize_out< double >( tout, src, sw, sh, dst, nw, nh, C, p );
		case 4: return resize_out< uint32_t >( tout, src, sw, sh, dst, nw, nh, C, p );
	}

	return -1;
}

} // extern "C"
