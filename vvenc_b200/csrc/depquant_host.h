// depquant_host.h -- host-side set-up of the dependent-quantisation kernel (plain C++, no CUDA): the per-shape scan tables of
// DQIntern::Rom::xInitScanArrays / TUParameters::xSetScanInfo (CommonLib/DepQuant.cpp:75-342) and the quantiser constants of
// Quantizer::initQuantBlock (:533-572).  Built once per context (tables) / once per call (constants).
#pragma once
#include "depquant_core.h"
#include <vector>
#include <cmath>
#include <cstring>

namespace vvbdq {

struct DqShapeTables { int width, height, numCoeff, numSbb; size_t offset; };     // offset: first entry of the shape in the two table arrays

inline int dq_shape_index( int w, int h )
{
  int lw = 0, lh = 0;
  while( ( 1 << lw ) < w ) lw++;
  while( ( 1 << lh ) < h ) lh++;
  if( ( 1 << lw ) != w || ( 1 << lh ) != h || lw < 2 || lw > 6 || lh < 2 || lh > 6 ) return -1;
  return ( lw - 2 ) * 5 + ( lh - 2 );
}

// up-right diagonal scan of a bw x bh grid (Rom.cpp:1098-1136)
inline void dq_diag( int bw, int bh, std::vector<int>& xs, std::vector<int>& ys )
{
  xs.resize( bw * bh ); ys.resize( bw * bh );
  int line = 0, col = 0;
  for( int i = 0; i < bw * bh; i++ )
  {
    xs[i] = col; ys[i] = line;
    if( col == bw - 1 || line == 0 ) { line += col + 1; col = 0; if( line >= bh ) { col += line - ( bh - 1 ); line = bh - 1; } }
    else { col++; line--; }
  }
}

// all 25 shapes (sides 4..64) of one channel type; scanInfo / nbOut are concatenated, shapes[] says where each one starts.  chroma: the context offsets of
// xSetScanInfo's CH_C branch (:326-330) -- the only thing in the tables that depends on the channel type
inline void dq_build_tables( std::vector<DqScanInfo>& scanInfo, std::vector<DqNbOut>& nbOut, DqShapeTables shapes[25], bool chroma = false )
{
  scanInfo.clear(); nbOut.clear();
  std::vector<int> cx, cy, gx, gy;
  dq_diag( 4, 4, cx, cy );
  for( int lw = 2; lw <= 6; lw++ )
    for( int lh = 2; lh <= 6; lh++ )
    {
      const int W = 1 << lw, H = 1 << lh, rw = W < 32 ? W : 32, rh = H < 32 ? H : 32;        // JVET_C0024_ZERO_OUT_TH: only the 32x32 region is scanned
      const int wSbb = rw >> 2, hSbb = rh >> 2, numCoeff = rw * rh, numSbb = wSbb * hSbb;
      DqShapeTables& st = shapes[( lw - 2 ) * 5 + ( lh - 2 )];
      st.width = W; st.height = H; st.numCoeff = numCoeff; st.numSbb = numSbb; st.offset = scanInfo.size();
      dq_diag( wSbb, hSbb, gx, gy );
      std::vector<int> px( numCoeff ), py( numCoeff ), raster( numCoeff ), raster2id( (size_t) W * H, 0 );
      for( int g = 0; g < numSbb; g++ )
        for( int c = 0; c < 16; c++ )
        {
          const int id = g * 16 + c;
          px[id] = gx[g] * 4 + cx[c]; py[id] = gy[g] * 4 + cy[c]; raster[id] = py[id] * W + px[id];
          raster2id[raster[id]] = id;
        }
      std::vector<DqScanInfo> si( numCoeff );
      std::vector<DqNbOut>    no( numCoeff );
      memset( si.data(), 0, sizeof( DqScanInfo ) * numCoeff );
      memset( no.data(), 0, sizeof( DqNbOut ) * numCoeff );
      for( int id = 0; id < numCoeff; id++ )
      {
        const int x = px[id], y = py[id], rpos = raster[id], begSbb = id & ~15;
        // the five template neighbours (right, right+1, diagonal, below, below+1), split into "same group" and "later group" (DepQuant.cpp:127-209)
        int nb[5];
        nb[0] = x + 1 < rw               ? raster2id[rpos + 1]         : -1;
        nb[1] = x + 2 < rw               ? raster2id[rpos + 2]         : -1;
        nb[2] = x + 1 < rw && y + 1 < rh ? raster2id[rpos + 1 + W]     : -1;
        nb[3] = y + 1 < rh               ? raster2id[rpos + W]         : -1;
        nb[4] = y + 2 < rh               ? raster2id[rpos + 2 * W]     : -1;
        int in[5], nin = 0, out[5], nout = 0;
        for( int k = 0; k < 5; k++ )
        {
          if( nb[k] < 0 ) continue;
          if( nb[k] < begSbb + 16 ) { if( nb[k] - begSbb != 0 ) in[nin++] = nb[k] - begSbb; }        // a relative position of 0 counts as "none" there (cpos != 0 test)
          else if( nb[k] != 0 ) out[nout++] = nb[k];
        }
        for( int a = 1; a < nin; a++ )  for( int b = a; b > 0 && in[b] < in[b - 1]; b-- )  { const int t = in[b]; in[b] = in[b - 1]; in[b - 1] = t; }
        for( int a = 1; a < nout; a++ ) for( int b = a; b > 0 && out[b] < out[b - 1]; b-- ) { const int t = out[b]; out[b] = out[b - 1]; out[b - 1] = t; }
        for( int k = 0; k < nin; k++ ) { DqScanInfo& t = si[begSbb + in[k]]; if( t.numInv < 5 ) t.invInPos[t.numInv++] = (uint8_t)( id & 15 ); }
        DqNbOut& o = no[id];
        o.num = (uint16_t) nout;
        for( int k = 0; k < nout; k++ ) o.outPos[k] = (uint16_t) out[k];
        int maxDist = id == 0 ? 0 : (int) no[id - 1].maxDist;                 // still absolute here
        for( int k = 0; k < nout; k++ ) if( out[k] > maxDist ) maxDist = out[k];
        o.maxDist = (uint16_t) maxDist;
      }
      for( int id = 0; id < numCoeff; id++ )                                  // "make it relative" (:212-223)
      {
        const int begSbb = id & ~15;
        for( int k = 0; k < no[id].num; k++ ) no[id].outPos[k] = (uint16_t)( no[id].outPos[k] - begSbb );
        no[id].maxDist = (uint16_t)( no[id].maxDist - id );
      }
      for( int id = 0; id < numCoeff; id++ )                                  // xSetScanInfo (:302-342)
      {
        DqScanInfo& t = si[id];
        t.rasterPos = (int16_t) raster[id];
        t.sbbPos    = (int16_t)( gy[id >> 4] * wSbb + gx[id >> 4] );
        t.insidePos = (int8_t)( id & 15 );
        t.spt = SCAN_ISCSBB;
        if( t.insidePos == 15 && id > 16 && id < numCoeff - 1 ) t.spt = SCAN_SOCSBB;
        else if( t.insidePos == 0 && id > 0 && id < numCoeff - 16 ) t.spt = SCAN_EOCSBB;
        t.posX = (int8_t) px[id]; t.posY = (int8_t) py[id];
        if( id )
        {
          const int nx = id - 1, diag = px[nx] + py[nx];
          if( !chroma )
          {
            t.sigCtxOffsetNext = (int8_t)( diag < 2 ? 8 : diag < 5 ? 4 : 0 );
            t.gtxCtxOffsetNext = (int8_t)( diag < 1 ? 16 : diag < 3 ? 11 : diag < 10 ? 6 : 1 );
          }
          else
          {
            t.sigCtxOffsetNext = (int8_t)( diag < 2 ? 4 : 0 );
            t.gtxCtxOffsetNext = (int8_t)( diag < 1 ? 6 : 1 );
          }
          t.nextInsidePos = (int8_t)( nx & 15 );
          if( t.insidePos == 0 )
          {
            const int nsp = gy[nx >> 4] * wSbb + gx[nx >> 4], nsy = nsp / wSbb, nsx = nsp - nsy * wSbb;
            t.nextSbbRight = (int16_t)( nsx < wSbb - 1 ? nsp + 1 : 0 );
            t.nextSbbBelow = (int16_t)( nsy < hSbb - 1 ? nsp + wSbb : 0 );
          }
        }
      }
      scanInfo.insert( scanInfo.end(), si.begin(), si.end() );
      nbOut.insert( nbOut.end(), no.begin(), no.end() );
    }
}

// Quantizer::initQuantBlock (:533-572) for a luma, non-transform-skip TU without scaling lists.  qpInternal = CU QP + 6 * (bitDepth - 8), clipped here to
// 0..63 + 6 * (bitDepth - 8) as QpParam clips cQP.Qp( false ) (Quant.cpp:109): below 0 the scale index qpRem would be negative.
// Same double-precision operation order as the reference (the library is built with -ffp-contract=off; this file must be, too).
inline DqQuant dq_init_quant( int w, int h, int bitDepth, int qpInternal, double lambda, int dqThrVal )
{
  static const int quantScales[2][6] = { { 26214, 23302, 20560, 18396, 16384, 14564 }, { 18396, 16384, 14564, 13107, 11651, 10280 } };      // g_quantScales, Rom.cpp:1390-1394
  const int maxQp = 63 + 6 * ( bitDepth - 8 );
  qpInternal = qpInternal < 0 ? 0 : qpInternal > maxQp ? maxQp : qpInternal;
  int lw = 0, lh = 0;
  while( ( 1 << lw ) < w ) lw++;
  while( ( 1 << lh ) < h ) lh++;
  const int qpDQ = qpInternal + 1, qpPer = qpDQ / 6, qpRem = qpDQ - 6 * qpPer;
  const int maxLog2TrDynamicRange = 15;
  const int nomTransformShift = maxLog2TrDynamicRange - bitDepth - ( ( lw + lh ) >> 1 );       // getTransformShift
  const bool sqrt2 = ( ( lw + lh ) & 1 ) != 0;                                                  // TU::needsSqrt2Scale
  const int transformShift = nomTransformShift + ( sqrt2 ? -1 : 0 );
  DqQuant q;
  q.qShift = 14 - 1 + qpPer + transformShift;                                                   // QUANT_SHIFT = 14
  q.qAdd   = -( ( (int64_t) 3 << q.qShift ) >> 1 );
  const int invShift = 6 + 1 - qpPer - transformShift;                                          // IQUANT_SHIFT = 6
  q.qScale = quantScales[sqrt2 ? 1 : 0][qpRem];
  const unsigned a = maxLog2TrDynamicRange + 1, b = (unsigned)( 8 * sizeof( int ) + invShift - 6 - 1 );
  const unsigned qIdxBD = a < b ? a : b;
  q.maxQIdx = ( 1 << ( qIdxBD - 1 ) ) - 4;
  if( q.qShift ) q.thresLast = (int32_t)( (int64_t) dqThrVal << ( q.qShift - 1 ) );
  else           q.thresLast = (int32_t)( (int64_t)( dqThrVal >> 1 ) << q.qShift );
  const int64_t qScale = q.qScale;
  const int nomDShift = 15 - 2 * nomTransformShift + q.qShift + ( sqrt2 ? 1 : 0 );              // SCALE_BITS = 15, DISTORTION_PRECISION_ADJUSTMENT = 0
  const double qScale2 = double( qScale * qScale );
  const double nomDistFactor = ( nomDShift < 0 ? 1.0 / ( double( int64_t( 1 ) << ( -nomDShift ) ) * qScale2 * lambda ) : double( int64_t( 1 ) << nomDShift ) / ( qScale2 * lambda ) );
  const uint32_t pow2dfShift = (uint32_t)( nomDistFactor * qScale2 ) + 1;
  int dfShift = 0;                                                                              // ceilLog2( x ) = x > 1 ? floorLog2( x - 1 ) + 1 : 0 (CommonDef.h)
  if( pow2dfShift > 1 ) { uint32_t v = pow2dfShift - 1; while( v ) { dfShift++; v >>= 1; } }
  q.distShift   = 62 + q.qShift - 2 * maxLog2TrDynamicRange - dfShift;
  q.distAdd     = ( int64_t( 1 ) << q.distShift ) >> 1;
  q.distStepAdd = ( ( q.distShift + q.qShift ) >= 64 ? (int64_t)( nomDistFactor * pow( 2, q.distShift + q.qShift ) + .5 ) : (int64_t)( nomDistFactor * double( int64_t( 1 ) << ( q.distShift + q.qShift ) ) + .5 ) );
  q.distOrgFact = (int64_t)( nomDistFactor * double( int64_t( 1 ) << ( q.distShift + 1 ) ) + .5 );
  return q;
}

} // namespace vvbdq
