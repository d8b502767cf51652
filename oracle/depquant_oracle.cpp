/*
 * oracle/depquant_oracle.cpp -- TEST INFRASTRUCTURE, not product code.
 *
 * CPU build of the dependent-quantisation restatement.  The algorithm text is vvenc_b200/csrc/depquant_core.h (each function there cites the lines of
 * CommonLib/DepQuant.cpp it follows) and the table / constant set-up is depquant_host.h; this file compiles both with g++ so that
 *   - tests/test_oracle_vs_reference.py can pin the restatement against the reference's own DepQuant::quant (oracle/_ref probe, scalar and AVX2 members) and
 *     against the golden vectors the reference generated (tests/golden/depquant_*.npz), here, without a GPU;
 *   - the GPU tests compare the device kernel (the same text compiled by nvcc for sm_90a) with this build on the same inputs.
 * The product library never loads this file.
 */
#include "../vvenc_b200/csrc/depquant_core.h"
#include "../vvenc_b200/csrc/depquant_host.h"
#include <vector>
#include <cstdlib>

using namespace vvbdq;

namespace {
struct Tables { std::vector<DqScanInfo> si; std::vector<DqNbOut> nb; DqShapeTables shapes[25]; explicit Tables( bool chroma ) { dq_build_tables( si, nb, shapes, chroma ); } };
const Tables& tables( int chroma = 0 ) { static Tables l( false ), c( true ); return chroma ? c : l; }
}

extern "C" {

// rates: the 266 int32 of vvb_dq_rates; coef [n][h][w]; q [n][h][w]; absSum / lastPos [n]
static int dep_quant_any( int chroma, int w, int h, int bitDepth, int qp, double lambda, int dqThrVal, int zeroOut, int lfnst, int scalarMembers, const int32_t* rates, const int32_t* coef, int n,
                          int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  const int idx = dq_shape_index( w, h );
  if( idx < 0 ) return -1;
  const Tables& t = tables( chroma );
  DqShape sh; sh.width = w; sh.height = h; sh.numCoeff = t.shapes[idx].numCoeff; sh.numSbb = t.shapes[idx].numSbb;
  sh.scanInfo = t.si.data() + t.shapes[idx].offset; sh.nbOut = t.nb.data() + t.shapes[idx].offset;
  const DqQuant qu = dq_init_quant( w, h, bitDepth, qp + 6 * ( bitDepth - 8 ), lambda, dqThrVal );
  DqRates r; memcpy( &r, rates, sizeof( r ) );
  std::vector<uint8_t> ctxMem( 8 * ( sh.numSbb + sh.numCoeff ) );
  std::vector<DqTrellis> trellis( 2 * sh.numCoeff );
  DqWork wk; wk.ctxMem = ctxMem.data(); wk.trellis = trellis.data();
  for( int i = 0; i < n; i++ )
    dq_quant_tu( sh, qu, r, zeroOut != 0, lfnst != 0, scalarMembers == 0, coef + (size_t) i * w * h, q + (size_t) i * w * h, wk, absSum + i, lastPos + i );
  return 0;
}

int orc_dep_quant( int w, int h, int bitDepth, int qp, double lambda, int dqThrVal, int zeroOut, int lfnst, int scalarMembers, const int32_t* rates, const int32_t* coef, int n,
                   int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  return dep_quant_any( 0, w, h, bitDepth, qp, lambda, dqThrVal, zeroOut, lfnst, scalarMembers, rates, coef, n, q, absSum, lastPos );
}
// chroma component: the chroma context offsets in the scan tables; qp is the mapped chroma QP minus qpBdOffset, rates come from the chroma context sets
int orc_dep_quant_chroma( int w, int h, int bitDepth, int qp, double lambda, int dqThrVal, int lfnst, int scalarMembers, const int32_t* rates, const int32_t* coef, int n,
                          int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  return dep_quant_any( 1, w, h, bitDepth, qp, lambda, dqThrVal, 0, lfnst, scalarMembers, rates, coef, n, q, absSum, lastPos );
}

int orc_dep_quant_constants( int w, int h, int bitDepth, int qp, double lambda, int dqThrVal, int64_t out[9] )
{
  if( dq_shape_index( w, h ) < 0 ) return -1;
  const DqQuant q = dq_init_quant( w, h, bitDepth, qp + 6 * ( bitDepth - 8 ), lambda, dqThrVal );
  out[0] = q.qShift; out[1] = q.maxQIdx; out[2] = q.thresLast; out[3] = q.distShift; out[4] = q.qAdd; out[5] = q.qScale; out[6] = q.distAdd; out[7] = q.distStepAdd; out[8] = q.distOrgFact;
  return 0;
}

// scan geometry of one shape, for table-level pins: scanInfo as 24-byte records, nbOut as 16-byte records
int orc_dep_quant_tables_ex( int chroma, int w, int h, void* scanInfoOut, void* nbOutOut );
int orc_dep_quant_tables( int w, int h, void* scanInfoOut, void* nbOutOut ) { return orc_dep_quant_tables_ex( 0, w, h, scanInfoOut, nbOutOut ); }
int orc_dep_quant_tables_ex( int chroma, int w, int h, void* scanInfoOut, void* nbOutOut )
{
  const int idx = dq_shape_index( w, h );
  if( idx < 0 ) return -1;
  const Tables& t = tables( chroma );
  const int nc = t.shapes[idx].numCoeff;
  if( scanInfoOut ) memcpy( scanInfoOut, t.si.data() + t.shapes[idx].offset, sizeof( DqScanInfo ) * nc );
  if( nbOutOut ) memcpy( nbOutOut, t.nb.data() + t.shapes[idx].offset, sizeof( DqNbOut ) * nc );
  return nc;
}

}
