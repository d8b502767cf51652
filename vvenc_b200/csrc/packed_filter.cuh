// packed_filter.cuh -- the packed pel-pair interpolation filter of the MCTF kernels (mctf_affine_kernels.cuh) and of the fractional refinement
// (frac_kernels.cuh).
//
// A reference window is staged as 32-bit words that hold pel pairs, starting at the even pel at or below the window's first pel.  The horizontal
// pass runs along those words; the callers store its results as row pairs (row 2r in the low half, row 2r + 1 in the high half), so the vertical
// pass runs on words of the same layout.  An N-tap output whose first pel is the low half of a word ("E") takes N/2 IDP.2A over the words
// that cover it; one whose first pel is the high half ("O") takes N/2 + 1 with the taps shifted by one byte and zero-padded at both ends.
// Taps fit int8, pels and intermediates fit int16, the sums are int32.  Rounding, clipping and the row-pair store belong to each caller.
#pragma once
#include "common.cuh"

namespace vvb {

// four signed taps as the int8x4 word IDP.2A reads: byte k = the low byte of d_k (the inner permutes put d0, d1 and d2, d3 into bytes 0 and 1,
// the outer one joins those halves)
__device__ __forceinline__ int pack_taps4( int d0, int d1, int d2, int d3 )
{
  return (int) __byte_perm( __byte_perm( d0, d1, 0x0040 ), __byte_perm( d2, d3, 0x0040 ), 0x5410 );
}

// The packed taps of an N-tap filter f[0..N-1]: E words FA = (f0 f1 f2 f3), FB = (f4 f5 f6 f7); O words GA = (0 f0 f1 f2), GB = (f3 f4 f5 f6),
// GC = (f7 0 0 0); taps past N are 0, so for 6 taps FB = (f4 f5 0 0), GB = (f3 f4 f5 0) and there is no GC.  The 6-tap record is one 16-byte
// shared-memory load.
template<int N> struct PackedTaps;
template<> struct __align__( 16 ) PackedTaps<6> { int FA, FB, GA, GB; };
template<> struct PackedTaps<8> { int FA, FB, GA, GB, GC; };

template<int N>
__device__ __forceinline__ PackedTaps<N> pack_taps( const int ( &f )[N] )
{
  static_assert( N == 6 || N == 8, "6- or 8-tap filters" );
  PackedTaps<N> t;
  if constexpr( N == 6 )
  {
    t.FA = pack_taps4( f[0], f[1], f[2], f[3] ); t.FB = pack_taps4( f[4], f[5], 0, 0 );
    t.GA = pack_taps4( 0, f[0], f[1], f[2] );    t.GB = pack_taps4( f[3], f[4], f[5], 0 );
  }
  else
  {
    t.FA = pack_taps4( f[0], f[1], f[2], f[3] ); t.FB = pack_taps4( f[4], f[5], f[6], f[7] );
    t.GA = pack_taps4( 0, f[0], f[1], f[2] );    t.GB = pack_taps4( f[3], f[4], f[5], f[6] ); t.GC = pack_taps4( f[7], 0, 0, 0 );
  }
  return t;
}

// E: the output's first pel is the low half of w[0]; reads w[0 .. N/2 - 1]
template<int N>
__device__ __forceinline__ int filter_e( const uint32_t* w, const PackedTaps<N>& t )
{
  int s = __dp2a_hi( (int) w[1], t.FA, __dp2a_lo( (int) w[0], t.FA, 0 ) );
  s = __dp2a_lo( (int) w[2], t.FB, s );
  if constexpr( N == 8 ) s = __dp2a_hi( (int) w[3], t.FB, s );
  return s;
}

// O: the output's first pel is the high half of w[0]; reads w[0 .. N/2]
template<int N>
__device__ __forceinline__ int filter_o( const uint32_t* w, const PackedTaps<N>& t )
{
  int s = __dp2a_hi( (int) w[1], t.GA, __dp2a_lo( (int) w[0], t.GA, 0 ) );
  s = __dp2a_hi( (int) w[3], t.GB, __dp2a_lo( (int) w[2], t.GB, s ) );
  if constexpr( N == 8 ) s = __dp2a_lo( (int) w[4], t.GC, s );
  return s;
}

// The raw sums of two adjacent outputs from the N/2 + 1 words w[0 .. N/2] that cover both: consecutive words of a window row (horizontal
// pass) or row-pair words of one column (vertical pass).  odd: the first output starts in the high half of w[0].
template<int N>
__device__ __forceinline__ int2 filter_pair( const uint32_t* w, bool odd, const PackedTaps<N>& t )
{
  int2 s;
  if( !odd ) { s.x = filter_e<N>( w, t ); s.y = filter_o<N>( w, t ); }
  else       { s.x = filter_o<N>( w, t ); s.y = filter_e<N>( w + 1, t ); }
  return s;
}

// The horizontal pass of one row-pair item: outputs x, x + 1 of the rows at ra and rb (rows 2r and 2r + 1 of a staged window), raw sums.
// Both rows share one branch on odd (as filter_pair's, written out once for the pair: two filter_pair calls compile to longer code).
template<int N>
__device__ __forceinline__ void filter_row_pair( const uint32_t* ra, const uint32_t* rb, bool odd, const PackedTaps<N>& t, int2& a, int2& b )
{
  uint32_t wa[N / 2 + 1], wb[N / 2 + 1];
#pragma unroll
  for( int k = 0; k <= N / 2; k++ ) wa[k] = ra[k];
#pragma unroll
  for( int k = 0; k <= N / 2; k++ ) wb[k] = rb[k];
  if( !odd ) { a = make_int2( filter_e<N>( wa, t ), filter_o<N>( wa, t ) ); b = make_int2( filter_e<N>( wb, t ), filter_o<N>( wb, t ) ); }
  else       { a = make_int2( filter_o<N>( wa, t ), filter_e<N>( wa + 1, t ) ); b = make_int2( filter_o<N>( wb, t ), filter_e<N>( wb + 1, t ) ); }
}

// Stages `rows` rows of the words that cover the `pels` pels from src on (row stride `stride` pels) into dst (pitch `pitch` words), starting at
// the even pel at or below src; thread t of T copies words t, t + T, ...  Returns the parity o of src: pel src[x] is half (x + o) & 1 of word
// dst[(x + o) >> 1].  Plane rows are 16-byte aligned, so every row has the parity of the first.  The caller provides the barriers.
__device__ __forceinline__ int stage_pel_pairs( uint32_t* dst, int pitch, const int16_t* src, int stride, int pels, int rows, int t, int T )
{
  const int o = (int)( ( reinterpret_cast<uintptr_t>( src ) >> 1 ) & 1 );
  const uint32_t* srcW = reinterpret_cast<const uint32_t*>( src - o );
  const int nW = ( pels + o + 1 ) >> 1;
  const float invNw = 1.0f / (float) nW;
  const int strideW = stride >> 1;
  for( int i = t; i < rows * nW; i += T )
  {
    const int r = div_rcp( i, invNw ), k = i - r * nW;
    dst[r * pitch + k] = __ldg( srcW + (ptrdiff_t) r * strideW + k );
  }
  return o;
}

} // namespace vvb
