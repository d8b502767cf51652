// integration/InterSearchB200.h -- reference-side binding of libvvenc_b200.so for the motion-search loops of EncoderLib/InterSearch.cpp.
//
// Companion of RdCostB200.h (which patches the per-call function-pointer tables): here whole loops of the reference are handed to one batched call and
// their selection logic is replayed on the returned numbers (INTEGRATION.md section 3):
//
//   xPatternSearchB200         <->  InterSearch::xPatternSearch        (InterSearch.cpp:2209-2251)   one vvb_sad_search
//   xPatternSearchFracDIFB200  <->  InterSearch::xPatternSearchFracDIF (InterSearch.cpp:2677-2725)   one vvb_frac_cost_grid + the two xPatternRefinement rounds
//                                                                      (:760-972, m_fastSubPel == 0) as table look-ups
//   xTZSearchB200              <->  InterSearch::xTZSearch             (InterSearch.cpp:2297-2573)   one vvb_sad_search with its SAD table, then the UNMODIFIED
//                                                                      member runs on that table (its SAD function-pointer slot answers by look-up)
//   B200RowSearch                   the production shape: all PUs of a CTU row against resident pictures, one launch per block size
//
// The member-shaped functions take the InterSearch object and the TZSearchStruct the reference already fills (piRefY, iRefStride, pcPatternKey, searchRange,
// imvShift, subShiftMode, useAltHpelIf) and read the predictor / lambda / cost scale from its RdCost exactly as the members do, so a maintainer can
// swap the call inside xMotionEstimation (:2441-2497) without touching the callers.  They upload the pattern key and the reference window per call:
// that is the correctness-first form (it is what tests compare with the members themselves); B200RowSearch is the form that performs.
//
// Include after RdCostB200.h, EncoderLib/InterSearch.h and CommonLib/RdCost.h.  Private members are used (m_pcRdCost, m_pcEncCfg, m_lumaClpRng):
// inside the encoder these would be member functions of InterSearch; oracle/ref_shim.cpp compiles this file against the unmodified reference.
#pragma once
#include <cmath>
#include <vector>
#include "RdCostB200.h"

struct B200SearchApi
{
  bool bound = false;
  decltype( &vvb_plane_upload )    planeUpload = nullptr;
  decltype( &vvb_sad_search )      sadSearch = nullptr;
  decltype( &vvb_frac_cost_grid )  fracCostGrid = nullptr;
  decltype( &vvb_set_tma_staging ) setTmaStaging = nullptr;
} ;
static B200SearchApi g_b200s;

// binds the search entry points of the library RdCostB200.h has opened; returns 0, -1 (library not loaded) or -2 (symbol missing)
inline int b200LoadSearch( const char* libPath )
{
  if( g_b200s.bound ) return 0;
  int rc = b200Load( libPath );
  if( rc ) return rc;
  void* h = g_b200.handle;
#define VVB_RESOLVE( member, name ) g_b200s.member = (decltype( g_b200s.member )) dlsym( h, #name ); if( !g_b200s.member ) { g_b200.error = "missing " #name; return -2; }
  VVB_RESOLVE( planeUpload, vvb_plane_upload )  VVB_RESOLVE( sadSearch, vvb_sad_search )  VVB_RESOLVE( fracCostGrid, vvb_frac_cost_grid )
  VVB_RESOLVE( setTmaStaging, vvb_set_tma_staging )
#undef VVB_RESOLVE
  g_b200s.bound = true;
  return 0;
}

// vvb_me_par of an RdCost in its current state: the library derives the motion lambda as sqrt( lambda ) like RdCost::setLambda (RdCost.cpp:73-78)
inline vvb_me_par b200MePar( RdCost& rc, int costScale, unsigned imvShift, int subShift )
{
  if( rc.m_motionLambda != std::sqrt( rc.m_dLambda ) ) THROW( "motion lambda is not sqrt( lambda ): call selectMotionLambda() after setLambda()" );
  vvb_me_par me = {};
  me.lambda = rc.m_dLambda; me.cost_scale = costScale; me.imv_shift = (int) imvShift; me.sub_shift = subShift;
  return me;
}

// RdCost::setDistParam's sub-sampling rule (RdCost.cpp:187-200)
inline int b200SubShift( int subShiftMode, int w, int h )
{
  if( subShiftMode == 1 && h > 8 && w <= 128 ) return 1;
  if( subShiftMode == 2 && h > 8 ) return 1;
  return 0;
}

// plane ids the per-call forms use for their uploads
enum { B200_PLANE_KEY = 14, B200_PLANE_WINDOW = 15 };

// The per-PU forms search a window that was uploaded for this one call: nothing for the TMA staging of the dense kernel to win (it pays on resident pictures, where the
// aligned boxes of neighbouring blocks hit in L2), so they run with the load/store staging and put the context's default back afterwards.
struct B200NoTmaScope
{
  B200NoTmaScope()  { g_b200s.setTmaStaging( b200CtxOfThread(), 0 ); }
  ~B200NoTmaScope() { g_b200s.setTmaStaging( b200CtxOfThread(), 2 ); }
};

// uploads the pattern key (margin 0) and the reference window around piRefY (margin `reach` on every side: the reference pictures are padded, Picture.cpp:461-501)
inline void b200UploadKeyAndWindow( const CPelBuf& key, const Pel* piRefY, int refStride, int reach, int bitDepth )
{
  vvb_ctx* ctx = b200CtxOfThread();
  b200Check( g_b200s.planeUpload( ctx, B200_PLANE_KEY, key.buf, key.stride, key.width, key.height, 0, bitDepth ) );
  b200Check( g_b200s.planeUpload( ctx, B200_PLANE_WINDOW, piRefY, refStride, key.width, key.height, reach, bitDepth ) );
}

// ---------------------------------------------------------------------------------------------------------------------------------------------
// InterSearch::xPatternSearch (InterSearch.cpp:2209-2251): full search over cStruct.searchRange, raster order, first strictly smaller SAD + MV cost wins
inline void xPatternSearchB200( InterSearch& is, InterSearch::TZSearchStruct& cStruct, Mv& rcMv, Distortion& ruiSAD )
{
  RdCost& rc = *is.m_pcRdCost;
  const CPelBuf& key = *cStruct.pcPatternKey;
  const InterSearch::SearchRange& sr = cStruct.searchRange;
  const int subShift = b200SubShift( cStruct.subShiftMode, key.width, key.height );
  const int reach = std::max( std::max( -sr.left, sr.right ), std::max( -sr.top, sr.bottom ) );
  b200UploadKeyAndWindow( key, cStruct.piRefY, cStruct.iRefStride, std::max( reach, 0 ), is.m_lumaClpRng.bd );

  vvb_block blk = {};
  blk.left = (int16_t) sr.left; blk.right = (int16_t) sr.right; blk.top = (int16_t) sr.top; blk.bottom = (int16_t) sr.bottom;
  blk.pred_hor = (int16_t) rc.m_mvPredictor.hor; blk.pred_ver = (int16_t) rc.m_mvPredictor.ver;
  if( blk.pred_hor != rc.m_mvPredictor.hor || blk.pred_ver != rc.m_mvPredictor.ver ) THROW( "predictor outside the 16-bit range of vvb_block" );
  const vvb_me_par me = b200MePar( rc, rc.m_iCostScale, cStruct.imvShift, subShift );
  vvb_best best = {};
  { B200NoTmaScope noTma; b200Check( g_b200s.sadSearch( b200CtxOfThread(), B200_PLANE_KEY, B200_PLANE_WINDOW, &blk, 1, key.width, key.height, &me, nullptr, 0, &best ) ); }

  rcMv.set( best.dx, best.dy );
  cStruct.uiBestSad = best.cost;                                                          // :2248
  ruiSAD = best.cost - rc.getCostOfVectorWithPredictor( best.dx, best.dy, cStruct.imvShift );
}

// ---------------------------------------------------------------------------------------------------------------------------------------------
// InterSearch::xPatternSearchFracDIF (InterSearch.cpp:2677-2725): the interpolation of xExtDIFUpSamplingH / Q (and, for m_fastSubPel == 1, the half-pel blocks
// xPatternRefinement filters itself, :812-848) and every distortion call of xPatternRefinement come back as ONE 7x7 table t[j+3][i+3] (quarter-pel offset (i, j)
// from rcMvInt; vvb_frac_cost_grid: SAD, SATD or fast SATD, square and rectangular PUs); the two rounds are replayed on it.
//   m_fastSubPel == 0 (slower): both rounds visit all nine positions, each round starts from MAX_DISTORTION.
//   m_fastSubPel == 1 (faster ... slow): the half-pel round stops early (:808-811) and classifies the cost surface into a pattern id (:886-969); the quarter-pel round
//     visits only what s_skipQpelPosition allows for that pattern (:93-137 -- file-static in the reference, restated here as one 9-bit mask per pattern, bit i =
//     position i skipped) and keeps the half-pel best as its threshold (:769); pattern 0 ends the search after the half-pel round (:2710) with rcMvQter untouched.
//   m_fastSubPel == 2 (the first pass of a two-pass encode, vvencCfg.cpp:2661): xMotionEstimation does not call the function (:2113).
inline void xPatternSearchFracDIFB200( InterSearch& is, InterSearch::TZSearchStruct& cStruct, const Mv& rcMvInt, Mv& rcMvHalf, Mv& rcMvQter, Distortion& ruiCost )
{
  const VVEncCfg& cfg = *is.m_pcEncCfg;
  if( cfg.m_fastSubPel != 0 && cfg.m_fastSubPel != 1 ) THROW( "m_fastSubPel == 2 never reaches the fractional search (InterSearch.cpp:2113)" );
  RdCost& rc = *is.m_pcRdCost;
  const CPelBuf& key = *cStruct.pcPatternKey;
  const int reach = std::max( std::abs( rcMvInt.hor ), std::abs( rcMvInt.ver ) ) + 5;        // integer vector + one pel of refinement + 4 pels of filter
  b200UploadKeyAndWindow( key, cStruct.piRefY, cStruct.iRefStride, reach, is.m_lumaClpRng.bd );

  vvb_block blk = {};
  blk.start_x = (int16_t) rcMvInt.hor; blk.start_y = (int16_t) rcMvInt.ver;
  uint32_t t[7][7];
  const int dfunc = cfg.m_bUseHADME ? ( cfg.m_fastHad ? VVB_DF_HAD_FAST : VVB_DF_HAD ) : VVB_DF_SAD;     // setDistParam( ..., m_bUseHADME ? ( m_fastHad ? 2 : 1 ) : 0 ), :775
  b200Check( g_b200s.fracCostGrid( b200CtxOfThread(), dfunc, B200_PLANE_KEY, B200_PLANE_WINDOW, &blk, 1, key.width, key.height,
                                   cfg.m_meReduceTap, cStruct.useAltHpelIf ? 1 : 0, &t[0][0] ) );

  static const int8_t orderH[9][2] = { { 0, 0 }, { 0, -1 }, { 0, 1 }, { -1, 0 }, { 1, 0 }, { -1, -1 }, { 1, -1 }, { -1, 1 }, { 1, 1 } };     // s_acMvRefineH
  static const int8_t orderQ[9][2] = { { 0, 0 }, { 0, -1 }, { 0, 1 }, { -1, -1 }, { 1, -1 }, { -1, 0 }, { 1, 0 }, { -1, 1 }, { 1, 1 } };     // s_acMvRefineQ
  static const uint16_t skipMask[42] = { 510, 479, 447, 509, 469, 429, 507, 347, 187, 123, 479, 347, 447, 187, 485, 479, 469, 447, 429, 175, 509, 429, 507, 187, 343, 509, 469,
                                         507, 347, 447, 507, 187, 479, 507, 347, 447, 509, 429, 479, 509, 469, 0 };
  const bool fast = cfg.m_fastSubPel == 1;
  Distortion uiDistBest = MAX_DISTORTION;
  int patternId = 41;
  // one round of xPatternRefinement (:760-972)
  auto round = [&]( const int8_t ( *order )[2], int iFrac, const Mv& baseRefMv, Mv& rcMvFrac ) -> Distortion
  {
    if( !fast ) uiDistBest = MAX_DISTORTION;                                                                         // :769
    uint32_t dir = 0;
    Distortion distH[9] = { uiDistBest, uiDistBest, uiDistBest, uiDistBest, uiDistBest, uiDistBest, uiDistBest, uiDistBest, uiDistBest };
    for( uint32_t i = 0; i < 9; i++ )
    {
      if( fast )
      {
        if( ( skipMask[patternId] >> i ) & 1 ) continue;                                                             // :802
        if( iFrac == 2 && ( ( i == 5 && dir == 0 ) || ( i == 7 && dir == 1 ) || ( i == 8 && ( dir == 1 || dir == 3 || dir == 5 ) ) ) ) break;   // :808-811
      }
      const int hor = ( order[i][0] + baseRefMv.hor ) * iFrac, ver = ( order[i][1] + baseRefMv.ver ) * iFrac;      // quarter-pel offset from rcMvInt (:852-856)
      Distortion d = t[ver + 3][hor + 3];
      d += rc.getCostOfVectorWithPredictor( order[i][0] + rcMvFrac.hor, order[i][1] + rcMvFrac.ver, 0 );           // :875 (imvShift 0 inside the refinement)
      distH[i] = d;
      if( d < uiDistBest ) { uiDistBest = d; dir = i; }
    }
    rcMvFrac.set( order[dir][0], order[dir][1] );
    if( fast && iFrac == 2 )                                                                                          // :886-969, Distortion arithmetic wraps as there
    {
      const Distortion TH = 17, TL = 15; const int shift = 4;
      auto ratio = [&]( int a, int b, int hi, int lo ) { distH[a] <<= shift; return distH[a] > TH * distH[b] ? hi : ( distH[a] < TL * distH[b] ? lo : 0 ); };
      auto slope = [&]( int a, int c, int b ) { return distH[a] - distH[c] > distH[c] - distH[b]; };
      switch( dir )
      {
      case 0: patternId += ratio( 3, 4, 2, 1 ); patternId += ratio( 1, 2, 6, 3 ); break;
      case 1: patternId += ratio( 5, 6, 4, 2 ); patternId += slope( 2, 0, 1 ) ? 1 : 0; patternId += ( 41 == patternId ? 0 : 8 );  break;
      case 2: patternId += ratio( 7, 8, 4, 2 ); patternId += slope( 1, 0, 2 ) ? 1 : 0; patternId += ( 41 == patternId ? 0 : 13 ); break;
      case 3: patternId += slope( 4, 0, 3 ) ? 1 : 0; patternId += ratio( 5, 7, 4, 2 ); patternId += ( 41 == patternId ? 0 : 18 ); break;
      case 4: patternId += slope( 3, 0, 4 ) ? 1 : 0; patternId += ratio( 6, 8, 4, 2 ); patternId += ( 41 == patternId ? 0 : 23 ); break;
      case 5: patternId += slope( 6, 1, 5 ) ? 1 : 0; patternId += slope( 7, 3, 5 ) ? 2 : 0; patternId += ( 41 == patternId ? 0 : 28 ); break;
      case 6: patternId += slope( 5, 1, 6 ) ? 1 : 0; patternId += slope( 8, 4, 6 ) ? 2 : 0; patternId += ( 41 == patternId ? 0 : 31 ); break;
      case 7: patternId += slope( 8, 2, 7 ) ? 1 : 0; patternId += slope( 5, 3, 7 ) ? 2 : 0; patternId += ( 41 == patternId ? 0 : 34 ); break;
      case 8: patternId += slope( 7, 2, 8 ) ? 1 : 0; patternId += slope( 6, 4, 8 ) ? 2 : 0; patternId += ( 41 == patternId ? 0 : 37 ); break;
      default: break;
      }
    }
    return uiDistBest;
  };

  rc.setCostScale( 1 );                                                                       // :2695
  rcMvHalf = rcMvInt; rcMvHalf <<= 1;
  ruiCost = round( orderH, 2, Mv( 0, 0 ), rcMvHalf );
  patternId -= fast ? 41 : 0;                                                                 // :2707
  if( cStruct.imvShift == IMV_OFF && 0 != patternId )                                         // :2711
  {
    rc.setCostScale( 0 );
    Mv baseRefMv = rcMvHalf; baseRefMv <<= 1;
    rcMvQter = rcMvInt; rcMvQter <<= 1; rcMvQter += rcMvHalf; rcMvQter <<= 1;
    ruiCost = round( orderQ, 1, baseRefMv, rcMvQter );
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------------------
// InterSearch::xTZSearch (InterSearch.cpp:2297-2573).  The TZ search is a data-dependent walk (start candidates, log-spaced diamonds, raster, star refinement,
// xTZ2PointSearch) whose every step is `SAD of one position + MV rate, keep if smaller` (xTZSearchHelp :410-438).  Instead of re-implementing the walk, the SADs
// of the whole window it can visit are produced by ONE dense launch (vvb_sad_search with its SAD table -- pels are visited once, the headline kernel), the
// RdCost slot the walk calls through (m_afpDistortFunc[.][DF_SAD + log2 w], selected by RdCost::setDistParam :158-200) is pointed at a table look-up for the
// duration of the call, and the reference's own xTZSearch runs unchanged.  Positions outside the table (a start candidate far from the predictor) are answered by
// the per-block entry point, so the result never depends on the window guess -- only the number of launches does.
struct B200TzTable
{
  const Pel* corner = nullptr;                                                                // address of the window's top-left position: piRefY + top * stride + left
  uint32_t   stride = 0, nx = 0, ny = 0, span = 0;                                            // span = ny * stride
  uint64_t   invStride = 0;                                                                   // ceil( 2^40 / stride ): off / stride without a divide (exact for off < 2^20)
  int        subShift = 0;
  const uint32_t* sad = nullptr;                                                              // [ny][nx], row-major over the window
  uint64_t hits = 0, misses = 0;
  void set( const Pel* piRefY, ptrdiff_t refStride, int left, int top, int nx_, int ny_, int subShift_, const uint32_t* sad_ )
  {
    corner = piRefY + (ptrdiff_t) top * refStride + left; stride = (uint32_t) refStride; nx = (uint32_t) nx_; ny = (uint32_t) ny_;
    span = ( ny && (uint64_t) ny * stride < ( 1u << 20 ) ) ? ny * stride : 0;                 // a window beyond the exact range of the reciprocal is treated as empty
    invStride = ( ( 1ull << 40 ) + stride - 1 ) / ( stride ? stride : 1 );
    subShift = subShift_; sad = sad_; hits = misses = 0;
  }
};
static thread_local B200TzTable t_b200tz;

inline Distortion tzTableSadB200( const DistParam& dp )
{
  B200TzTable& t = t_b200tz;
  const uint64_t off = (uint64_t)( dp.cur.buf - t.corner );                                   // positions before the corner wrap to huge values and miss
  if( off < t.span && dp.subShift == t.subShift )
  {
    const uint32_t dy = (uint32_t)( ( off * t.invStride ) >> 40 ), dx = (uint32_t) off - dy * t.stride;
    if( dx < t.nx ) { t.hits++; return t.sad[dy * t.nx + dx]; }
  }
  t.misses++;
  return distB200<VVB_DF_SAD>( dp );
}

// window guess for the walk: the search range (+1 for xTZ2PointSearch) around the integer start vector and around the zero vector -- the two start candidates of
// :2338-2346 --, kept inside the readable reach.  rcMv: the start vector in internal (1/16 pel) units, as xTZSearch receives it.
inline void b200TzWindow( const Mv& rcMv, int searchRange, bool bFastSettings, int refReach, int& left, int& right, int& top, int& bottom )
{
  const int R = ( searchRange >> ( bFastSettings ? 1 : 0 ) ) + 1;
  const int px = rcMv.hor >> MV_FRACTIONAL_BITS_INTERNAL, py = rcMv.ver >> MV_FRACTIONAL_BITS_INTERNAL;
  auto clampR = [&]( int v ) { return std::max( -refReach, std::min( refReach, v ) ); };
  left = clampR( std::min( px, 0 ) - R ); right = clampR( std::max( px, 0 ) + R ); top = clampR( std::min( py, 0 ) - R ); bottom = clampR( std::max( py, 0 ) + R );
}

// the unmodified member on a prepared table: the SAD slot RdCost::setDistParam will select (:172-176) answers by look-up for the duration of the call
inline void b200TzWalk( InterSearch& is, const CodingUnit& cu, RefPicList refPicList, int iRefIdxPred, InterSearch::TZSearchStruct& cStruct, Mv& rcMv, Distortion& ruiSAD,
                        const bool bExtendedSettings, const bool bFastSettings, const uint32_t* sad, int left, int top, int nx, int ny, int subShift )
{
  RdCost& rc = *is.m_pcRdCost;
  B200TzTable& t = t_b200tz;
  t.set( cStruct.piRefY, cStruct.iRefStride, left, top, nx, ny, subShift, sad );
  const int base = is.m_lumaClpRng.bd > 10 ? 1 : 0, slot = DF_SAD + Log2( cStruct.pcPatternKey->width );
  const FpDistFunc saved = rc.m_afpDistortFunc[base][slot];
  rc.m_afpDistortFunc[base][slot] = tzTableSadB200;
  try { is.xTZSearch( cu, refPicList, iRefIdxPred, cStruct, rcMv, ruiSAD, bExtendedSettings, bFastSettings ); }
  catch( ... ) { rc.m_afpDistortFunc[base][slot] = saved; t.sad = nullptr; t.span = 0; throw; }
  rc.m_afpDistortFunc[base][slot] = saved; t.sad = nullptr; t.span = 0;
}

// refReach: how far (in pels, every direction) the reference picture is readable around the block -- the picture margin the encoder pads (Picture.cpp:461-501)
inline void xTZSearchB200( InterSearch& is, const CodingUnit& cu, RefPicList refPicList, int iRefIdxPred, InterSearch::TZSearchStruct& cStruct, Mv& rcMv, Distortion& ruiSAD,
                           const bool bExtendedSettings, const bool bFastSettings, const int refReach )
{
  RdCost& rc = *is.m_pcRdCost;
  const CPelBuf& key = *cStruct.pcPatternKey;
  const int subShift = b200SubShift( cStruct.subShiftMode, key.width, key.height );
  int left, right, top, bottom;
  b200TzWindow( rcMv, is.m_iSearchRange, bFastSettings, refReach, left, right, top, bottom );
  b200UploadKeyAndWindow( key, cStruct.piRefY, cStruct.iRefStride, refReach, is.m_lumaClpRng.bd );

  const int nx = right - left + 1, ny = bottom - top + 1;
  std::vector<uint32_t> sad( (size_t) nx * ny );
  vvb_block blk = {};
  blk.left = (int16_t) left; blk.right = (int16_t) right; blk.top = (int16_t) top; blk.bottom = (int16_t) bottom;
  blk.pred_hor = (int16_t) rc.m_mvPredictor.hor; blk.pred_ver = (int16_t) rc.m_mvPredictor.ver;
  const vvb_me_par me = b200MePar( rc, rc.m_iCostScale, cStruct.imvShift, subShift );
  vvb_best best = {};
  int rcSearch;
  { B200NoTmaScope noTma; rcSearch = g_b200s.sadSearch( b200CtxOfThread(), B200_PLANE_KEY, B200_PLANE_WINDOW, &blk, 1, key.width, key.height, &me, sad.data(), nx * ny, &best ); }
  if( rcSearch != VVB_OK && rcSearch != VVB_ERR_UNSUPPORTED ) b200Check( rcSearch );
  // a window the dense kernel cannot stage (block + range beyond its shared-memory budget) leaves the table empty: every position then takes the per-block path
  const bool haveTable = rcSearch == VVB_OK;
  b200TzWalk( is, cu, refPicList, iRefIdxPred, cStruct, rcMv, ruiSAD, bExtendedSettings, bFastSettings, sad.data(), left, top, haveTable ? nx : 0, haveTable ? ny : 0, subShift );
}

// ---------------------------------------------------------------------------------------------------------------------------------------------
// Production shape (INTEGRATION.md section 3): the pictures are uploaded once, the PUs of a CTU row are queued with the search range and predictor the
// reference computed for them (xSetSearchRange :2178-2206, setPredictor), and run() issues one vvb_sad_search per block size.  Results equal
// xPatternSearch per PU, including the raster tie-break.
class B200RowSearch
{
public:
  struct Result { Mv mv; Distortion sad; Distortion cost; };

  void setPictures( const CPelBuf& org, const CPelBuf& ref, int margin, int bitDepth )
  {
    b200Check( g_b200s.planeUpload( b200CtxOfThread(), 0, org.buf, org.stride, org.width, org.height, 0, bitDepth ) );
    b200Check( g_b200s.planeUpload( b200CtxOfThread(), 1, ref.buf, ref.stride, ref.width, ref.height, margin, bitDepth ) );
    m_margin = margin;
  }
  // returns the index under which results() reports this PU
  int add( int x, int y, int w, int h, const InterSearch::SearchRange& sr, const Mv& predictor )
  {
    Group* g = nullptr;
    for( auto& c : m_groups ) if( c.w == w && c.h == h ) g = &c;
    if( !g ) { m_groups.push_back( Group() ); g = &m_groups.back(); g->w = w; g->h = h; }
    vvb_block b = {};
    b.x = x; b.y = y; b.left = (int16_t) sr.left; b.right = (int16_t) sr.right; b.top = (int16_t) sr.top; b.bottom = (int16_t) sr.bottom;
    b.pred_hor = (int16_t) predictor.hor; b.pred_ver = (int16_t) predictor.ver;
    g->blocks.push_back( b ); g->index.push_back( (int) m_results.size() );
    m_results.push_back( Result() );
    return (int) m_results.size() - 1;
  }
  void run( RdCost& rc, unsigned imvShift, int subShiftMode )
  {
    for( auto& g : m_groups )
    {
      const int subShift = b200SubShift( subShiftMode, g.w, g.h );
      const vvb_me_par me = b200MePar( rc, rc.m_iCostScale, imvShift, subShift );
      std::vector<vvb_best> best( g.blocks.size() );
      const bool tma = boxesInside( g.blocks );
      if( !tma ) g_b200s.setTmaStaging( b200CtxOfThread(), 0 );
      const int rcS = g_b200s.sadSearch( b200CtxOfThread(), 0, 1, g.blocks.data(), (int) g.blocks.size(), g.w, g.h, &me, nullptr, 0, best.data() );
      if( !tma ) g_b200s.setTmaStaging( b200CtxOfThread(), 2 );
      b200Check( rcS );
      for( size_t i = 0; i < best.size(); i++ )
      {
        Result& r = m_results[g.index[i]];
        r.mv.set( best[i].dx, best[i].dy ); r.cost = best[i].cost; r.sad = best[i].sad;
      }
    }
    m_groups.clear();
  }
  // the TMA boxes of the dense kernel are whole windows rounded up to 8 pels: keep them inside the uploaded margin, else stage with loads
  bool boxesInside( const std::vector<vvb_block>& blocks ) const
  {
    for( const vvb_block& b : blocks ) if( std::max( std::max( -b.left, (int) b.right ), std::max( -b.top, (int) b.bottom ) ) + 8 > m_margin ) return false;
    return true;
  }
  const std::vector<Result>& results() const { return m_results; }
  void clear() { m_groups.clear(); m_results.clear(); m_tables.clear(); }

  // ---- TZ search for the row: one dense launch per block size fills every PU's SAD table, then the reference's own xTZSearch walks each table on the host.
  // addTz queues a PU with the window b200TzWindow derives from its start vector; runTables launches; tzSearch( i, ... ) is xTZSearch for PU i (same
  // arguments as the member: the TZSearchStruct still names the PU's pattern key and its position in the reference picture).
  int addTz( int x, int y, int w, int h, const Mv& startMvInternal, const Mv& predictor, int searchRange, bool bFastSettings, int refReach )
  {
    InterSearch::SearchRange sr;
    b200TzWindow( startMvInternal, searchRange, bFastSettings, refReach, sr.left, sr.right, sr.top, sr.bottom );
    return add( x, y, w, h, sr, predictor );
  }
  void runTables( RdCost& rc, unsigned imvShift, int subShiftMode )
  {
    m_tables.assign( m_results.size(), Table() );
    for( auto& g : m_groups )
    {
      const int subShift = b200SubShift( subShiftMode, g.w, g.h );
      const vvb_me_par me = b200MePar( rc, rc.m_iCostScale, imvShift, subShift );
      int tableStride = 0;
      for( const vvb_block& b : g.blocks ) tableStride = std::max( tableStride, ( b.right - b.left + 1 ) * ( b.bottom - b.top + 1 ) );
      std::vector<uint32_t> tabs( (size_t) tableStride * g.blocks.size() );
      std::vector<vvb_best> best( g.blocks.size() );
      const bool tma = boxesInside( g.blocks );
      if( !tma ) g_b200s.setTmaStaging( b200CtxOfThread(), 0 );
      const int rcS = g_b200s.sadSearch( b200CtxOfThread(), 0, 1, g.blocks.data(), (int) g.blocks.size(), g.w, g.h, &me, tabs.data(), tableStride, best.data() );
      if( !tma ) g_b200s.setTmaStaging( b200CtxOfThread(), 2 );
      b200Check( rcS );
      for( size_t i = 0; i < g.blocks.size(); i++ )
      {
        const vvb_block& b = g.blocks[i];
        Table& t = m_tables[g.index[i]];
        t.left = b.left; t.top = b.top; t.nx = b.right - b.left + 1; t.ny = b.bottom - b.top + 1; t.subShift = subShift;
        t.sad.assign( tabs.begin() + (ptrdiff_t)( i * tableStride ), tabs.begin() + (ptrdiff_t)( i * tableStride + (size_t) t.nx * t.ny ) );
      }
    }
    m_groups.clear();
  }
  void tzSearch( int i, InterSearch& is, const CodingUnit& cu, RefPicList refPicList, int iRefIdxPred, InterSearch::TZSearchStruct& cStruct, Mv& rcMv, Distortion& ruiSAD,
                 const bool bExtendedSettings, const bool bFastSettings ) const
  {
    const Table& t = m_tables[i];
    b200TzWalk( is, cu, refPicList, iRefIdxPred, cStruct, rcMv, ruiSAD, bExtendedSettings, bFastSettings, t.sad.data(), t.left, t.top, t.nx, t.ny, t.subShift );
  }

private:
  struct Group { int w, h; std::vector<vvb_block> blocks; std::vector<int> index; };
  struct Table { int left = 0, top = 0, nx = 0, ny = 0, subShift = 0; std::vector<uint32_t> sad; };
  std::vector<Group>  m_groups;
  std::vector<Result> m_results;
  std::vector<Table>  m_tables;
  int                 m_margin = 0;
};
