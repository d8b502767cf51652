/*
 * oracle/rdoq_oracle.cpp -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU build of the RDOQ restatement (QuantRDOQ2::xRateDistOptQuantFast).  The algorithm text is vvenc_b200/csrc/rdoq_core.h (each block there cites the lines of
 * CommonLib/QuantRDOQ2.cpp / ContextModelling.h it follows) and the constant set-up is rdoq_host.h; this file compiles both with g++ so that
 *   - tests/test_oracle_vs_reference.py can pin the restatement against the reference's own QuantRDOQ2::xRateDistOptQuant (oracle/_ref probe) and against the
 *     golden vectors the reference generated (tests/golden/golden_v6_rdoq.npz), here, without a GPU;
 *   - the GPU tests compare the device kernel (the same text compiled by nvcc for sm_90a) with this build on the same inputs.
 * The product library never loads this file.
 */
#include "../vvenc_b200/csrc/rdoq_core.h"
#include "../vvenc_b200/csrc/rdoq_host.h"
#include <vector>
#include <cstring>

using namespace vvbrq;

extern "C" {

// rates: the 190 int32 of vvb_rdoq_rates; coef [n][h][w]; q [n][h][w]; absSum / lastPos [n].  qp: CU QP (the bit-depth offset is added here, as the library does)
int orc_rdoq( int w, int h, int bitDepth, int qp, int isChroma, int lfnst, int sbtZeroOut, int signHiding, double lambda, int thrVal, const int32_t* rates,
              const int32_t* coef, int n, int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  if( !rq_shape_ok( w, h ) ) return -1;
  int qpInternal = qp + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > 63 + 6 * ( bitDepth - 8 ) ? 63 + 6 * ( bitDepth - 8 ) : qpInternal;
  const RqPar p = rq_init_par( w, h, bitDepth, qpInternal, lfnst, sbtZeroOut, signHiding, isChroma, lambda, thrVal );
  RqRates r; memcpy( &r, rates, sizeof( r ) );
  std::vector<int32_t> scan( 1024 );
  rq_build_scan( w, h, scan.data() );
  for( int i = 0; i < n; i++ ) rq_quant_tu( p, r, scan.data(), coef + (size_t) i * w * h, q + (size_t) i * w * h, absSum + i, lastPos + i );
  return 0;
}

// the second engine of the same routine (accumulated templates, cost tables): same arguments, same results
int orc_rdoq_v2( int w, int h, int bitDepth, int qp, int isChroma, int lfnst, int sbtZeroOut, int signHiding, double lambda, int thrVal, const int32_t* rates,
                 const int32_t* coef, int n, int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  if( !rq_shape_ok( w, h ) ) return -1;
  int qpInternal = qp + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > 63 + 6 * ( bitDepth - 8 ) ? 63 + 6 * ( bitDepth - 8 ) : qpInternal;
  const RqPar p = rq_init_par( w, h, bitDepth, qpInternal, lfnst, sbtZeroOut, signHiding, isChroma, lambda, thrVal );
  RqRates r; memcpy( &r, rates, sizeof( r ) );
  const RqCost c = rq_init_cost( p, r );
  std::vector<int32_t> scan( 1024 );
  rq_build_scan( w, h, scan.data() );
  uint8_t cgIdx[64];
  rq_build_cg_index( scan.data(), w, h, cgIdx );
  for( int i = 0; i < n; i++ ) rq_quant_tu_v2( p, r, c, scan.data(), cgIdx, coef + (size_t) i * w * h, q + (size_t) i * w * h, absSum + i, lastPos + i );
  return 0;
}

// transform-skipped TUs (QuantRDOQ::rateDistOptQuantTS): rates = the 44 int32 of vvb_rdoq_ts_rates; qp: CU QP (luma) or mapped chroma QP minus qpBdOffset; inputDelta =
// sps.internalMinusInputBitDepth (the QP floor of skipped transforms)
int orc_rdoq_ts( int w, int h, int bitDepth, int qp, int inputDelta, double lambda, const int32_t* rates, const int32_t* coef, int n, int16_t* q, int32_t* absSum )
{
  if( !rq_ts_shape_ok( w, h ) ) return -1;
  int qpInternal = qp + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > 63 + 6 * ( bitDepth - 8 ) ? 63 + 6 * ( bitDepth - 8 ) : qpInternal;
  if( qpInternal < 4 + 6 * inputDelta ) qpInternal = 4 + 6 * inputDelta;
  const RqTsPar p = rq_ts_init_par( w, h, bitDepth, qpInternal, lambda );
  RqTsRates r; memcpy( &r, rates, sizeof( r ) );
  std::vector<int32_t> scan( 1024 );
  rq_build_scan( w, h, scan.data() );
  for( int i = 0; i < n; i++ ) rq_ts_quant_tu( p, r, scan.data(), coef + (size_t) i * w * h, q + (size_t) i * w * h, absSum + i );
  return 0;
}
// BDPCM TUs (QuantRDOQ::forwardRDPCM): dirMode 1 horizontal, 2 vertical; everything else as orc_rdoq_ts
int orc_rdoq_bdpcm( int w, int h, int bitDepth, int qp, int inputDelta, int dirMode, double lambda, const int32_t* rates, const int32_t* coef, int n, int16_t* q, int32_t* absSum )
{
  if( !rq_ts_shape_ok( w, h ) || dirMode < 1 || dirMode > 2 ) return -1;
  int qpInternal = qp + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > 63 + 6 * ( bitDepth - 8 ) ? 63 + 6 * ( bitDepth - 8 ) : qpInternal;
  if( qpInternal < 4 + 6 * inputDelta ) qpInternal = 4 + 6 * inputDelta;
  const RqTsPar p = rq_ts_init_par( w, h, bitDepth, qpInternal, lambda );
  const RqBdpcmPar b = rq_bdpcm_init_par( dirMode, qpInternal );
  RqTsRates r; memcpy( &r, rates, sizeof( r ) );
  std::vector<int32_t> scan( 1024 ), full( (size_t) w * h );
  rq_build_scan( w, h, scan.data() );
  for( int i = 0; i < n; i++ ) rq_bdpcm_quant_tu( p, b, r, scan.data(), coef + (size_t) i * w * h, q + (size_t) i * w * h, full.data(), absSum + i );
  return 0;
}

// quantScale, qBits, maxCtxBins and the error scale (double)
int orc_rdoq_ts_constants( int w, int h, int bitDepth, int qp, int inputDelta, int32_t outInt[3], double* errorScale )
{
  if( !rq_ts_shape_ok( w, h ) ) return -1;
  int qpInternal = qp + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > 63 + 6 * ( bitDepth - 8 ) ? 63 + 6 * ( bitDepth - 8 ) : qpInternal;
  if( qpInternal < 4 + 6 * inputDelta ) qpInternal = 4 + 6 * inputDelta;
  const RqTsPar p = rq_ts_init_par( w, h, bitDepth, qpInternal, 1.0 );
  outInt[0] = p.quantScale; outInt[1] = p.qBits; outInt[2] = p.maxCtxBins; *errorScale = p.errorScale;
  return 0;
}

// the constants of one call: quantScale, errScale, qBits, useThres, remRegBins, numCG, firstScanPos
int orc_rdoq_constants( int w, int h, int bitDepth, int qp, int isChroma, int lfnst, int sbtZeroOut, int thrVal, int32_t out[7] )
{
  if( !rq_shape_ok( w, h ) ) return -1;
  int qpInternal = qp + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > 63 + 6 * ( bitDepth - 8 ) ? 63 + 6 * ( bitDepth - 8 ) : qpInternal;
  const RqPar p = rq_init_par( w, h, bitDepth, qpInternal, lfnst, sbtZeroOut, 0, isChroma, 1.0, thrVal );
  out[0] = p.quantScale; out[1] = p.errScale; out[2] = p.qBits; out[3] = p.useThres; out[4] = p.remRegBins; out[5] = p.numCG; out[6] = p.firstScanPos;
  return 0;
}

}
