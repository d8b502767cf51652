// rdoq_core.h -- the fast rate-distortion optimised quantiser of one TU: QuantRDOQ2::xRateDistOptQuantFast<bSBH, false> (CommonLib/QuantRDOQ2.cpp:475-1281) with
// its helpers xiGetICRateCost (:320-401), xiGetCostLast (:445-461), _dist (:468-473) and the CoeffCodingContext members it drives (ContextModelling.h:158-269,
// ContextModelling.cpp:113-133), restated for one thread per TU.  This is what Quant::m_RDOQ == 2 selects (the presets faster and fast, vvencCfg.cpp:2675, 2737)
// for every TU that is not transform skipped, and what DepQuant::quant falls back to in slices without dependent quantisation (DepQuant.cpp:1486-1489).
//
// What stays on the host: everything that depends on the encoder's entropy-coding state.  The fractional bits of the contexts the routine reads (significance
// set 0, parity, greater-1, greater-2, significant-group, the last-position tables of xInitLastPosBitsTab :408-434, the coded-block-flag context of :1185-1226)
// arrive as `RqRates`; the per-call constants (quantiser scale and shift, the error scale of xSetErrScaleCoeffNoScalingList :203-219, thresholds) as `RqPar`
// (rdoq_host.h).  No scaling lists, no transform skip (rateDistOptQuantTS), sides 4..64 (coefficient groups are always 4x4 there, g_log2SbbSize).
//
// The template bookkeeping of the reference (m_tplBuf: per position the sum of min( 4 + ( l & 1 ), l ) and the count of the five already-coded neighbours,
// kept in step with the level buffer by absVal1stPass / remAbsVal1stPass at every change) is a pure function of the level buffer, so it is read from the
// levels directly (the form sigCtxIdAbs, ContextModelling.h:115-156, uses).
//
// Plain C++ without CUDA syntax outside VVB_HD: the test suite compiles the very same text for the CPU (g++), where it is pinned against the reference's member.
#pragma once
#include <stdint.h>

#ifndef VVB_HD
#ifdef __CUDACC__
#define VVB_HD __host__ __device__ __forceinline__
#else
#define VVB_HD inline
#endif
#endif

namespace vvbrq {

enum { RQ_SCALE_BITS = 15, RQ_ERR_SCALE_SHIFT = 20 /* COEFF_ERR_SCALE_PRECISION_BITS, QuantRDOQ2.cpp:84 */, RQ_SBH_THRESHOLD = 4, RQ_REMAIN_BIN_REDUCTION = 5 };

typedef int64_t cost_t;              // QuantRDOQ2.h:59

struct RqRates                       // BinFracBits::intBits of the contexts, as FracBitsAccess::getFracBitsArray returns them at the point of the call
{
  int32_t sigBits[12][2];            // Ctx::SigFlag[chType]( ctxOfs ): set 0 (state 0), ctxOfs 0..11 (luma) / 0..7 (chroma)
  int32_t parBits[21][2];            // Ctx::ParFlag[chType]( ctxOffsetAbs )
  int32_t gt1Bits[21][2];            // Ctx::GtxFlag[chType + 2]( ctxOffsetAbs )  (greater1CtxIdAbs, ContextModelling.h:239)
  int32_t gt2Bits[21][2];            // Ctx::GtxFlag[chType]( ctxOffsetAbs )      (greater2CtxIdAbs, :240)
  int32_t sigGroupBits[2][2];        // Ctx::SigCoeffGroup[chType]( sigRight | sigLower )
  int32_t lastBitsX[16], lastBitsY[16];   // m_lastBitsX / m_lastBitsY[chType][ctxId] after xInitLastPosBitsTab
  int32_t cbfBits[2];                // the coded-block-flag context of :1185-1226 (QtRootCbf for inter luma, QtCbf otherwise); zeros when the flag is inferred
  int32_t pad[2];
};

struct RqPar
{
  int32_t width, height, log2W;      // TU size
  int32_t regionW;                   // min( 32, width ): row pitch of the scan table entries
  int32_t numCG;                     // iCGNum, :553
  int32_t firstScanPos;              // the position the search for the first non-zero coefficient starts from, :554-559
  int32_t quantScale;                // g_quantScales[needsSqrt2][rem], :518
  int32_t errScale;                  // xGetErrScaleCoeffNoScalingList, :519
  int32_t qBits;                     // qShift, :522
  int32_t useThres;                  // thres / ( quantScale << 2 ), :573-583
  int32_t remRegBins;                // ( tbAreaAfterCoefZeroOut * 28 ) >> 4, :539
  int32_t signHiding;                // bSBH
  int32_t isChroma;                  // channel type of the component (context offsets)
  int32_t pad;
  double  lambda;                    // Quant::m_dLambda
};

#ifdef __CUDACC__
#define VVB_RQ_TAB __device__ __constant__
#else
#define VVB_RQ_TAB static const
#endif
VVB_RQ_TAB uint8_t c_rqGoRicePars[32] = { 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 3, 3, 3 };      // g_auiGoRiceParsCoeff, Rom.cpp:1464-1467
VVB_RQ_TAB uint8_t c_rqGroupIdx[32]   = { 0, 1, 2, 3, 4, 4, 5, 5, 6, 6, 6, 6, 7, 7, 7, 7, 8, 8, 8, 8, 8, 8, 8, 8, 9, 9, 9, 9, 9, 9, 9, 9 };      // g_uiGroupIdx, Rom.cpp:1463 (positions < 32)

VVB_HD int rq_min( int a, int b ) { return a < b ? a : b; }
VVB_HD int rq_max( int a, int b ) { return a > b ? a : b; }
VVB_HD int rq_abs( int a ) { return a < 0 ? -a : a; }

VVB_HD cost_t rq_icost( const RqPar& P, int rate ) { return (cost_t)( P.lambda * rate ); }                   // xiGetICost, :303-306

// xiGetICRateCost, :320-401
VVB_HD cost_t rq_level_rate_cost( const RqPar& P, uint32_t lv, const int32_t* par, const int32_t* gt1, const int32_t* gt2, int remRegBins, uint32_t riceZero, uint32_t goRice )
{
  cost_t rate = (cost_t) 1 << RQ_SCALE_BITS;                    // xGetIEPRate: the sign bin
  if( remRegBins < 4 )
  {
    uint32_t symbol = ( lv == 0 ? riceZero : lv <= riceZero ? lv - 1 : lv );
    uint32_t length;
    const int threshold = RQ_REMAIN_BIN_REDUCTION;
    if( symbol < ( (uint32_t) threshold << goRice ) )
    {
      length = symbol >> goRice;
      rate += (cost_t)( length + 1 + goRice ) << RQ_SCALE_BITS;
    }
    else
    {
      length = goRice;
      symbol = symbol - ( (uint32_t) threshold << goRice );
      while( symbol >= ( 1u << length ) ) symbol -= ( 1u << ( length++ ) );
      rate += (cost_t)( threshold + length + 1 - goRice + length ) << RQ_SCALE_BITS;
    }
  }
  else
  {
    const uint32_t cthres = 4;
    if( lv >= cthres )
    {
      uint32_t symbol = ( lv - cthres ) >> 1;
      uint32_t length;
      const int threshold = RQ_REMAIN_BIN_REDUCTION;
      if( symbol < ( (uint32_t) threshold << goRice ) )
      {
        length = symbol >> goRice;
        rate += (cost_t)( length + 1 + goRice ) << RQ_SCALE_BITS;
      }
      else
      {
        length = goRice;
        symbol = symbol - ( (uint32_t) threshold << goRice );
        while( symbol >= ( 1u << length ) ) symbol -= ( 1u << ( length++ ) );
        rate += (cost_t)( threshold + length + 1 - goRice + length ) << RQ_SCALE_BITS;
      }
      rate += gt1[1];
      rate += par[( lv - 2 ) & 1];
      rate += gt2[1];
    }
    else if( lv == 1 ) { rate += gt1[0]; }
    else if( lv == 2 ) { rate += gt1[1]; rate += par[0]; rate += gt2[0]; }
    else if( lv == 3 ) { rate += gt1[1]; rate += par[1]; rate += gt2[0]; }
    else rate = 0;
  }
  return rq_icost( P, (int) rate );
}

VVB_HD cost_t rq_dist( cost_t err, cost_t errScale )              // _dist, :468-473
{
  const int64_t s = ( err * errScale ) >> RQ_ERR_SCALE_SHIFT;
  return s * s;
}

// the five already-coded neighbours of (x, y) in the level buffer (levels are kept as magnitudes until the sign pass at the end)
#define VVB_RQ_TEMPLATE( q, W, H, x, y, OP ) { const int16_t* pd_ = ( q ) + ( y ) * ( W ) + ( x ); \
  if( ( x ) < ( W ) - 1 ) { OP( pd_[1] ); if( ( x ) < ( W ) - 2 ) OP( pd_[2] ); if( ( y ) < ( H ) - 1 ) OP( pd_[( W ) + 1] ); } \
  if( ( y ) < ( H ) - 1 ) { OP( pd_[( W )] ); if( ( y ) < ( H ) - 2 ) OP( pd_[2 * ( W )] ); } }

// one TU.  scan: scan position -> raster index inside the scanned region (row pitch P.regionW), grouped 4x4 diagonal scan; coef [h][w] TCoeff; q [h][w] levels (written);
// absSum / lastPos as the reference leaves uiAbsSum / tu.lastPos (lastPos -1 where the reference does not write it: nothing coded)
VVB_HD void rq_quant_tu( const RqPar& P, const RqRates& R, const int32_t* scan, const int32_t* coef, int16_t* q, int32_t* absSumOut, int32_t* lastPosOut )
{
  const int W = P.width, H = P.height, lw = P.log2W;
  const int lrw = ( P.regionW == 32 ? 5 : P.regionW == 16 ? 4 : P.regionW == 8 ? 3 : 2 );
  const bool bSBH = P.signHiding != 0, luma = P.isChroma == 0;
  const int qShift = P.qBits, quantScale = P.quantScale;
  const int qHalf = 1 << ( qShift - 1 );
  const cost_t errScl = P.errScale;
  const int widthInGroups = rq_min( 32, W ) >> 2, heightInGroups = rq_min( 32, H ) >> 2;
#define RQ_BLKPOS( sp ) ( ( ( scan[sp] >> lrw ) << lw ) + ( scan[sp] & ( P.regionW - 1 ) ) )

  for( int i = 0; i < W * H; i++ ) q[i] = 0;                      // :513

  cost_t keepCost[16], sigCost[16], zeroCost[16], flipDelta[16];
  int    flipStep[16];
  for( int i = 0; i < 16; i++ ) { keepCost[i] = 0; sigCost[i] = 0; zeroCost[i] = 0; flipDelta[i] = 0; flipStep[i] = 0; }

  cost_t codedTu = 0, uncodedTu = 0;
  int    lastPosNow = -1, lastGrp = -1;
  bool   lastSearchDone = false;
  cost_t bestTuCost = INT64_MAX / 2;
  int    remRegBins = P.remRegBins;
  uint32_t rice = 0;
  int    sumTu = 0;
  const int grpLen = 16, grpMask = 15, lgGrpLen = 4;
  uint64_t grpFlags = 0;                                     // m_sigCoeffGroupFlag, indexed by the raster position of the group
  int    tplDiag = -1, tplSum1 = -1;                        // CoeffCodingContext::m_tmplCpDiag / m_tmplCpSum1 (persist from position to position)

  int spos = P.firstScanPos;
  for( ; spos > 0; spos-- ) if( coef[RQ_BLKPOS( spos )] ) break;        // :561-567

  int grp = spos >> lgGrpLen;
  for( ; grp >= 0; grp-- )
  {
    int    nzWeight = 0, sumGrp = 0;
    cost_t codedGrp = 0, uncodedGrp = 0;
    int    inGrp = spos & ( grpLen - 1 );

    if( lastPosNow < 0 && spos >= 16 )                      // :599-656 (the SIMD and the scalar form test the same positions: everything above spos is zero)
    {
      bool allBelow = true;
      for( int xp = inGrp, xs = spos; allBelow && xp >= 0; xp--, xs-- ) allBelow &= rq_abs( coef[RQ_BLKPOS( xs )] ) <= P.useThres;
      if( allBelow ) { spos -= inGrp + 1; continue; }
    }

    // group position and the context of its significant-group flag (initSubblock, ContextModelling.cpp:113-133)
    const int cgRaster = scan[grp << 4], cgX = ( cgRaster & ( P.regionW - 1 ) ) >> 2, cgY = ( cgRaster >> lrw ) >> 2;
    const int grpRaster = cgY * widthInGroups + cgX;
    const uint64_t cgBit = (uint64_t) 1 << grpRaster;
    int binsAtGrpStart = remRegBins;
    int grpCtx = 0;

    bool seekLast = lastPosNow < 0;
    for( ;; )
    {
      if( seekLast )                                              // findlast2, :658-686
      {
        for( ; inGrp >= 0; inGrp--, spos-- )
        {
          const uint32_t maxAbsLevel = (uint32_t)( ( rq_abs( coef[RQ_BLKPOS( spos )] ) * quantScale + qHalf ) >> qShift );
          if( maxAbsLevel ) { lastPosNow = spos; lastGrp = grp; break; }
        }
        seekLast = false;
      }
      {
        const unsigned sigRight = ( cgX + 1 ) < widthInGroups  ? (unsigned)( ( grpFlags >> ( grpRaster + 1 ) ) & 1 ) : 0u;
        const unsigned sigLower = ( cgY + 1 ) < heightInGroups ? (unsigned)( ( grpFlags >> ( grpRaster + widthInGroups ) ) & 1 ) : 0u;
        grpCtx = (int)( sigRight | sigLower );
      }
      binsAtGrpStart = remRegBins;

      bool again = false;
      for( ; inGrp >= 0; inGrp--, spos-- )      // :697-969
      {
        const int raster = scan[spos], posX = raster & ( P.regionW - 1 ), posY = raster >> lrw;
        const int cpos = ( posY << lw ) + posX;
        const int scaledMag = rq_abs( coef[cpos] ) * quantScale;
        const int roundedLvl = ( scaledMag + qHalf ) >> qShift;

        int sigCtx = 0;
        if( spos != lastPosNow )                            // sigCtxIdAbsWithAcc( iScanPos, 0 ), ContextModelling.h:158-178
        {
          int numPos = 0, sumAbs = 0;
          // the member accumulates min( 4 + ( level & 1 ), level ) of the full level (:950); a level above 32767 is kept here as its low 16 bits (TCoeffSig,
          // :942), which read as uint16 give the same term for every level below 65533 (levels reach 104858 at the lowest QP of a 64-sided TU; the header states the rest)
#define RQ_UPD( v ) { const int a_ = (uint16_t)( v ); sumAbs += rq_min( 4 + ( a_ & 1 ), a_ ); numPos += a_ != 0; }
          VVB_RQ_TEMPLATE( q, W, H, posX, posY, RQ_UPD )
#undef RQ_UPD
          const int diag = posX + posY;
          sigCtx = rq_min( ( sumAbs + 1 ) >> 1, 3 ) + ( diag < 2 ? 4 : 0 );
          if( luma ) sigCtx += diag < 5 ? 4 : 0;
          tplDiag = diag; tplSum1 = sumAbs - numPos;
        }
        int ctxOffset = 0;                                        // ctxOffsetAbs, ContextModelling.h:227-236
        if( tplDiag != -1 )
        {
          ctxOffset  = rq_min( tplSum1, 4 ) + 1;
          ctxOffset += ( !tplDiag ? ( luma ? 15 : 5 ) : luma ? ( tplDiag < 3 ? 10 : ( tplDiag < 10 ? 5 : 0 ) ) : 0 );
        }
        const int32_t* fbPar = R.parBits[ctxOffset];
        const int32_t* fbGt1 = R.gt1Bits[ctxOffset];
        const int32_t* fbGt2 = R.gt2Bits[ctxOffset];
        const int32_t* fbSig = R.sigBits[sigCtx];
        uint32_t riceZero = 0;

        if( remRegBins < 4 )                                      // :731-736
        {
          int sum = 0;      // templateAbsSum sums abs() of the stored TCoeffSig (ContextModelling.h:242-265): a level from 32768 to 65535 is stored negative
#define RQ_SUM( v ) { sum += rq_abs( v ); }
          VVB_RQ_TEMPLATE( q, W, H, posX, posY, RQ_SUM )
#undef RQ_SUM
          const int sumAbs = rq_max( rq_min( sum, 31 ), 0 );      // templateAbsSum( ., ., 0 )
          rice = c_rqGoRicePars[sumAbs];
          riceZero  = 1u << rice;                        // g_auiGoRicePosCoeff0( 0, . ), Rom.h:137-140
        }

        zeroCost[inGrp] = rq_dist( scaledMag, errScl );

        uint32_t lvlPick = 0;
        if( roundedLvl == 0 )                                      // :748-770
        {
          sigCost  [inGrp] = rq_icost( P, fbSig[0] );
          keepCost[inGrp] = zeroCost[inGrp] + sigCost[inGrp];
          if( bSBH )
          {
            const cost_t errOne  = scaledMag - ( (int64_t) 1 << qShift );
            const cost_t distOne = rq_dist( errOne, errScl );
            const cost_t rateOne = remRegBins < 4 ? rq_level_rate_cost( P, 1, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice ) -
                                                   rq_level_rate_cost( P, 0, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice )
                                                 : (cost_t) fbGt1[0];
            const cost_t costOne = distOne + rateOne + rq_icost( P, fbSig[1] );
            flipDelta[inGrp] = costOne - keepCost[inGrp];
            flipStep      [inGrp] = 1;
          }
        }
        else
        {
          const int lvlDown = (int)( scaledMag >> qShift );
          const int lvlUp  = lvlDown + 1;

          if( remRegBins >= 4 && spos != lastPosNow && lvlUp >= 4 )     // :777-781
          {
            int sum = 0;
#define RQ_SUM( v ) { sum += rq_abs( v ); }
            VVB_RQ_TEMPLATE( q, W, H, posX, posY, RQ_SUM )
#undef RQ_SUM
            rice = c_rqGoRicePars[rq_max( rq_min( sum - 5 * 4, 31 ), 0 )];
          }

          if( spos == lastPosNow )                          // last level, :783-835
          {
            sigCost[inGrp] = 0;
            cost_t lastDown = zeroCost[inGrp];
            if( lvlDown )
            {
              const cost_t errDown = scaledMag - ( lvlDown << qShift );
              lastDown = rq_dist( errDown, errScl ) + rq_level_rate_cost( P, lvlDown, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
            }
            const cost_t errUp = scaledMag - ( lvlUp << qShift );
            const cost_t lastUp = rq_dist( errUp, errScl ) + rq_level_rate_cost( P, lvlUp, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );

            if( lastUp < lastDown )
            {
              lvlPick = lvlUp;
              keepCost[inGrp] = lastUp;
              if( bSBH ) { flipDelta[inGrp] = lastDown - lastUp; flipStep[inGrp] = -1; }
            }
            else
            {
              if( lvlDown == 0 )                                   // the candidate last position quantises to zero: look for the next one (goto findlast2, :816-827)
              {
                lastPosNow = -1; lastGrp = -1;
                spos--; inGrp--;
                again = true;
                break;
              }
              lvlPick = lvlDown;
              keepCost[inGrp] = lastDown;
              if( bSBH ) { flipDelta[inGrp] = lastUp - lastDown; flipStep[inGrp] = 1; }
            }
          }
          else
          {
            const cost_t sigOne = rq_icost( P, fbSig[1] );
            if( lvlUp < 3 )                                       // levels 0, 1, 2, :840-907
            {
              const cost_t sigZero = rq_icost( P, fbSig[0] );
              cost_t bestLvlCost = zeroCost[inGrp] + sigZero;
              cost_t bestSig = sigZero;
              cost_t costDown = bestLvlCost;
              lvlPick = 0;
              if( lvlDown == 1 )
              {
                const cost_t errDown = scaledMag - ( lvlDown << qShift );
                costDown = rq_dist( errDown, errScl ) + sigOne + rq_level_rate_cost( P, lvlDown, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
                if( costDown < bestLvlCost )
                {
                  lvlPick = lvlDown; bestLvlCost = costDown; bestSig = sigOne;
                  if( bSBH ) { flipDelta[inGrp] = bestLvlCost - costDown; flipStep[inGrp] = -1; }
                }
                else
                {
                  if( bSBH ) { flipDelta[inGrp] = costDown - bestLvlCost; flipStep[inGrp] = 1; }
                }
              }
              const cost_t errUp = scaledMag - ( lvlUp << qShift );
              const cost_t costUp = rq_dist( errUp, errScl ) + sigOne + rq_level_rate_cost( P, lvlUp, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
              if( costUp < bestLvlCost )
              {
                lvlPick = lvlUp;
                keepCost[inGrp] = costUp;
                sigCost[inGrp]   = sigOne;
                if( bSBH ) { flipDelta[inGrp] = costDown - costUp; flipStep[inGrp] = -1; }
              }
              else
              {
                keepCost[inGrp] = bestLvlCost;
                sigCost[inGrp]   = bestSig;
                if( bSBH ) { flipDelta[inGrp] = costUp - costDown; flipStep[inGrp] = 1; }
              }
            }
            else                                                  // levels x, x + 1, :908-940
            {
              const cost_t errDown = scaledMag - ( lvlDown << qShift );
              const cost_t costDown = rq_dist( errDown, errScl ) + sigOne + rq_level_rate_cost( P, lvlDown, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
              const cost_t errUp = scaledMag - ( lvlUp << qShift );
              const cost_t costUp = rq_dist( errUp, errScl ) + sigOne + rq_level_rate_cost( P, lvlUp, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
              sigCost[inGrp] = sigOne;
              if( costUp < costDown )
              {
                lvlPick = lvlUp;
                keepCost[inGrp] = costUp;
                if( bSBH ) { flipDelta[inGrp] = costDown - costUp; flipStep[inGrp] = -1; }
              }
              else
              {
                lvlPick = lvlDown;
                keepCost[inGrp] = costDown;
                if( bSBH ) { flipDelta[inGrp] = costUp - costDown; flipStep[inGrp] = 1; }
              }
            }
          }
          q[cpos] = (int16_t) lvlPick;                        // :942
          if( lvlPick )
          {
            sumGrp    += lvlPick;
            nzWeight += inGrp;
            grpFlags |= cgBit;                               // setSigGroup
          }
        }

        if( ( ( spos & grpMask ) == 0 ) && ( spos > 0 ) ) rice = 0;                      // :956-963
        else if( remRegBins >= 4 ) remRegBins -= ( lvlPick < 2 ? (int) lvlPick : 3 ) + ( spos != lastPosNow );

        uncodedGrp += zeroCost[inGrp];
        codedGrp   += keepCost[inGrp];
      }
      if( !again ) break;
      seekLast = true;
    }

    //================== group significance flag, :971-1036 ===================
    cost_t grpFlagCost = 0;
    if( lastGrp >= 0 )
    {
      if( grp )
      {
        const cost_t grpFlag0 = rq_icost( P, R.sigGroupBits[grpCtx][0] );
        if( !( grpFlags & cgBit ) )
        {
          codedGrp = uncodedGrp + grpFlag0;
          grpFlagCost = grpFlag0;
        }
        else
        {
          if( grp < lastGrp )
          {
            const cost_t grpFlag1 = rq_icost( P, R.sigGroupBits[grpCtx][1] );
            grpFlagCost = grpFlag1;
            if( !nzWeight ) codedGrp -= sigCost[0];
            const cost_t uncodedGrpAlt = uncodedGrp + grpFlag0;
            codedGrp += grpFlag1;
            if( uncodedGrpAlt < codedGrp )                // cheaper as an all-zero group
            {
              grpFlags &= ~cgBit;                            // resetSigGroup
              codedGrp = uncodedGrpAlt;
              grpFlagCost = grpFlag0;
              remRegBins = binsAtGrpStart;
              for( int p = grpLen - 1; p >= 0; p-- ) q[RQ_BLKPOS( grp * grpLen + p )] = 0;
              sumGrp = 0;
              if( lastGrp == grp ) { codedGrp = 0; uncodedGrp = 0; lastPosNow = -1; lastGrp = -1; }
            }
          }
          else grpFlags |= cgBit;
        }
      }
    }

    //===== last position cost, :1038-1095 =====
    bestTuCost += codedGrp;
    if( !lastSearchDone )
    {
      if( grpFlags & cgBit )
      {
        cost_t runningCost = uncodedTu + codedGrp - grpFlagCost;
        const int startIn = grp == lastGrp ? lastPosNow % grpLen : grpMask;
        int runningSum = sumGrp;
        int bestEnd = lastPosNow + 1;
        for( int pc = startIn; pc >= 0; pc-- )
        {
          const int sp = ( grp << lgGrpLen ) + pc;
          const int raster = scan[sp], px = raster & ( P.regionW - 1 ), py = raster >> lrw;
          const int bp = ( py << lw ) + px;
          if( q[bp] )
          {
            // xiGetCostLast, :445-461
            const uint32_t ctxX = c_rqGroupIdx[px], ctxY = c_rqGroupIdx[py];
            uint32_t lastBits = (uint32_t) R.lastBitsX[ctxX] + (uint32_t) R.lastBitsY[ctxY];
            if( ctxX > 3 ) lastBits += ( 1u << RQ_SCALE_BITS ) * ( ( ctxX - 2 ) >> 1 );
            if( ctxY > 3 ) lastBits += ( 1u << RQ_SCALE_BITS ) * ( ( ctxY - 2 ) >> 1 );
            const cost_t lastCost = rq_icost( P, (int) lastBits );
            const cost_t candCost = runningCost + lastCost - sigCost[pc];
            if( candCost < bestTuCost )
            {
              bestEnd = sp + 1; bestTuCost = candCost; lastGrp = grp; sumGrp = runningSum; sumTu = 0;
            }
            if( q[bp] > 1 ) { lastSearchDone = true; break; }
            runningSum -= 1;
            runningCost -= keepCost[pc];
            runningCost += zeroCost[pc];
          }
          else runningCost -= sigCost[pc];
        }
        for( int sp = bestEnd; sp <= lastPosNow; sp++ ) q[RQ_BLKPOS( sp )] = 0;
        lastPosNow = bestEnd - 1;
      }
    }

    //=============== sign bit hiding, :1097-1167 ================
    if( bSBH )
    {
      if( sumGrp >= 2 )
      {
        const int grpBase = grp * grpLen;
        int lastNz = -1, firstNz = grpLen;
        for( int n = 0; n < grpLen; n++ ) if( q[RQ_BLKPOS( n + grpBase )] ) { firstNz = n; break; }
        if( lastGrp == grp )
        {
          lastNz = lastPosNow % grpLen;
          if( q[RQ_BLKPOS( lastPosNow )] == 1 && flipStep[lastNz] == -1 ) flipDelta[lastNz] -= ( 4 << RQ_SCALE_BITS );
        }
        else
        {
          for( int n = grpLen - 1; n >= 0; n-- ) if( q[RQ_BLKPOS( n + grpBase )] ) { lastNz = n; break; }
        }
        if( lastNz - firstNz >= RQ_SBH_THRESHOLD )
        {
          codedGrp -= rq_icost( P, 1 << RQ_SCALE_BITS );
          const bool negFirst = coef[RQ_BLKPOS( grpBase + firstNz )] < 0;
          if( (int) negFirst != ( sumGrp & 0x1 ) )
          {
            const int lastIn = ( lastGrp == grp ) ? lastNz : grpLen - 1;
            int64_t minDelta = INT64_MAX;
            int minAt = -1;
            if( q[RQ_BLKPOS( firstNz + grpBase )] > 1 ) { minDelta = flipDelta[firstNz]; minAt = firstNz; }
            for( int n = 0; n < firstNz; n++ )
              if( ( coef[RQ_BLKPOS( grpBase + n )] < 0 ) == negFirst )
                if( flipDelta[n] < minDelta ) { minDelta = flipDelta[n]; minAt = n; }
            for( int n = firstNz + 1; n <= lastIn; n++ )
              if( flipDelta[n] < minDelta ) { minDelta = flipDelta[n]; minAt = n; }
            const int bp = RQ_BLKPOS( minAt + grpBase );
            q[bp] = (int16_t)( q[bp] + flipStep[minAt] );
            sumGrp   += flipStep[minAt];
            codedGrp += minDelta;
          }
        }
      }
    }

    codedTu   += codedGrp;
    uncodedTu += uncodedGrp;
    sumTu += sumGrp;
  }

  codedTu = bestTuCost;                                // :1177

  if( lastPosNow < 0 ) { *absSumOut = sumTu; *lastPosOut = -1; return; }         // :1179-1183 (sumTu is 0 there)

  uncodedTu += rq_icost( P, R.cbfBits[0] );               // :1185-1226 (the caller resolved which context applies; zeros when the flag is inferred)
  codedTu   += rq_icost( P, R.cbfBits[1] );

  if( uncodedTu <= codedTu )                      // :1228-1233
  {
    for( int i = 0; i < W * H; i++ ) q[i] = 0;
    *absSumOut = 0; *lastPosOut = -1;
    return;
  }
  if( bSBH && q[RQ_BLKPOS( lastPosNow )] == 0 )                 // :1237-1249
  {
    int sp = lastPosNow - 1;
    for( ; sp >= 0; sp-- ) if( q[RQ_BLKPOS( sp )] ) break;
    lastPosNow = sp;
  }
  for( int sp = 0; sp <= lastPosNow; sp++ )                     // signs, :1251-1257
  {
    const int bp = RQ_BLKPOS( sp );
    const int level = q[bp];
    const int iSign = coef[bp] >> 31;
    q[bp] = (int16_t)( ( iSign ^ level ) - iSign );
  }
  *absSumOut = sumTu; *lastPosOut = lastPosNow;
#undef RQ_BLKPOS
}

// Second engine of the same routine (vvb_set_rdoq_engine 2): identical decisions, fewer instructions per coefficient.
//  * The template of a position is not gathered from its five neighbours when the position is visited (a quarter of the executed instructions of the first engine,
//    in a per-source-line breakdown): it is ACCUMULATED, as the reference does in m_tplBuf (absVal1stPass / remAbsVal1stPass, ContextModelling.h:180-225), in the
//    level slot of the position itself -- a position that has not been visited yet holds no level, so its slot carries ( count << 5 | sum ) of the decided neighbours; when a
//    level is set, changed (sign-bit hiding) or cleared (group zero-out, last-position optimisation), the five positions to the left / above that are still unvisited are
//    updated.  A position is unvisited iff its coefficient group comes earlier in the scan than the group being worked on (cgIdx: group raster position -> group scan index).
//  * lambda * bits of the significance flags and of the levels 1..3 with context-coded bins come from tables computed once per call (RqCost, same double product).
struct RqCost
{
  int64_t sig[12][2];                // xiGetICost( sigBits[ctx][bin] )
  int64_t lvl[21][3];                // xiGetICRateCost( 1 / 2 / 3, ... ) with remRegBins >= 4 for greater-1 / parity / greater-2 context offset ctx
};
// the member adds the term of the full level when it decides one (:950) and removes min( 4 + ( a & 1 ), a ) of a = abs( TCoeffSig ) of the stored one (:1016, 1088, 1157)
#define VVB_RQ_ENC( L ) ( ( L ) ? 32 + rq_min( 4 + ( ( L ) & 1 ), ( L ) ) : 0 )
// add `delta` to the accumulators of the unvisited dependents of (x, y): every dependent when ALL is set (the position itself is being visited: everything to its left /
// above is still ahead), else only those in groups that come earlier in the scan than group `curCG`
#define VVB_RQ_DEPS( q, W, x, y, delta, ALL, cgIdx, wInGroups, curCG ) { int16_t* pq_ = ( q ) + ( y ) * ( W ) + ( x ); \
  if( ( y ) > 1 && ( ( ALL ) || cgIdx[( ( ( y ) - 2 ) >> 2 ) * ( wInGroups ) + ( ( x ) >> 2 )] < ( curCG ) ) ) pq_[-2 * ( W )] = (int16_t)( pq_[-2 * ( W )] + ( delta ) ); \
  if( ( y ) > 0 && ( x ) > 0 && ( ( ALL ) || cgIdx[( ( ( y ) - 1 ) >> 2 ) * ( wInGroups ) + ( ( ( x ) - 1 ) >> 2 )] < ( curCG ) ) ) pq_[-( W ) - 1] = (int16_t)( pq_[-( W ) - 1] + ( delta ) ); \
  if( ( y ) > 0 && ( ( ALL ) || cgIdx[( ( ( y ) - 1 ) >> 2 ) * ( wInGroups ) + ( ( x ) >> 2 )] < ( curCG ) ) ) pq_[-( W )] = (int16_t)( pq_[-( W )] + ( delta ) ); \
  if( ( x ) > 1 && ( ( ALL ) || cgIdx[( ( y ) >> 2 ) * ( wInGroups ) + ( ( ( x ) - 2 ) >> 2 )] < ( curCG ) ) ) pq_[-2] = (int16_t)( pq_[-2] + ( delta ) ); \
  if( ( x ) > 0 && ( ( ALL ) || cgIdx[( ( y ) >> 2 ) * ( wInGroups ) + ( ( ( x ) - 1 ) >> 2 )] < ( curCG ) ) ) pq_[-1] = (int16_t)( pq_[-1] + ( delta ) ); }
VVB_HD void rq_quant_tu_v2( const RqPar& P, const RqRates& R, const RqCost& C, const int32_t* scan, const uint8_t* cgIdx, const int32_t* coef, int16_t* q, int32_t* absSumOut, int32_t* lastPosOut )
{
  const int W = P.width, H = P.height, lw = P.log2W;
  const int lrw = ( P.regionW == 32 ? 5 : P.regionW == 16 ? 4 : P.regionW == 8 ? 3 : 2 );
  const bool bSBH = P.signHiding != 0, luma = P.isChroma == 0;
  const int qShift = P.qBits, quantScale = P.quantScale;
  const int qHalf = 1 << ( qShift - 1 );
  const cost_t errScl = P.errScale;
  const int widthInGroups = rq_min( 32, W ) >> 2, heightInGroups = rq_min( 32, H ) >> 2;
#define RQ_BLKPOS( sp ) ( ( ( scan[sp] >> lrw ) << lw ) + ( scan[sp] & ( P.regionW - 1 ) ) )

  for( int i = 0; i < W * H; i++ ) q[i] = 0;                      // :513

#define RQ_LVL_COST( L, par_, gt1_, gt2_, rrb_, grz_, grp_ ) ( ( ( rrb_ ) >= 4 && (uint32_t)( L ) - 1u < 3u ) ? C.lvl[ctxOffset][(uint32_t)( L ) - 1u] : rq_level_rate_cost( P, ( L ), par_, gt1_, gt2_, rrb_, grz_, grp_ ) )
  cost_t keepCost[16], sigCost[16], zeroCost[16], flipDelta[16];
  int    flipStep[16];
  for( int i = 0; i < 16; i++ ) { keepCost[i] = 0; sigCost[i] = 0; zeroCost[i] = 0; flipDelta[i] = 0; flipStep[i] = 0; }

  cost_t codedTu = 0, uncodedTu = 0;
  int    lastPosNow = -1, lastGrp = -1;
  bool   lastSearchDone = false;
  cost_t bestTuCost = INT64_MAX / 2;
  int    remRegBins = P.remRegBins;
  uint32_t rice = 0;
  int    sumTu = 0;
  const int grpLen = 16, grpMask = 15, lgGrpLen = 4;
  uint64_t grpFlags = 0;                                     // m_sigCoeffGroupFlag, indexed by the raster position of the group
  int    tplDiag = -1, tplSum1 = -1;                        // CoeffCodingContext::m_tmplCpDiag / m_tmplCpSum1 (persist from position to position)

  int spos = P.firstScanPos;
  for( ; spos > 0; spos-- ) if( coef[RQ_BLKPOS( spos )] ) break;        // :561-567

  int grp = spos >> lgGrpLen;
  for( ; grp >= 0; grp-- )
  {
    int    nzWeight = 0, sumGrp = 0;
    cost_t codedGrp = 0, uncodedGrp = 0;
    int    inGrp = spos & ( grpLen - 1 );

    if( lastPosNow < 0 && spos >= 16 )                      // :599-656 (the SIMD and the scalar form test the same positions: everything above spos is zero)
    {
      bool allBelow = true;
      for( int xp = inGrp, xs = spos; allBelow && xp >= 0; xp--, xs-- ) allBelow &= rq_abs( coef[RQ_BLKPOS( xs )] ) <= P.useThres;
      if( allBelow ) { spos -= inGrp + 1; continue; }
    }

    // group position and the context of its significant-group flag (initSubblock, ContextModelling.cpp:113-133)
    const int cgRaster = scan[grp << 4], cgX = ( cgRaster & ( P.regionW - 1 ) ) >> 2, cgY = ( cgRaster >> lrw ) >> 2;
    const int grpRaster = cgY * widthInGroups + cgX;
    const uint64_t cgBit = (uint64_t) 1 << grpRaster;
    int binsAtGrpStart = remRegBins;
    int grpCtx = 0;

    bool seekLast = lastPosNow < 0;
    for( ;; )
    {
      if( seekLast )                                              // findlast2, :658-686
      {
        for( ; inGrp >= 0; inGrp--, spos-- )
        {
          const uint32_t maxAbsLevel = (uint32_t)( ( rq_abs( coef[RQ_BLKPOS( spos )] ) * quantScale + qHalf ) >> qShift );
          if( maxAbsLevel ) { lastPosNow = spos; lastGrp = grp; break; }
        }
        seekLast = false;
      }
      {
        const unsigned sigRight = ( cgX + 1 ) < widthInGroups  ? (unsigned)( ( grpFlags >> ( grpRaster + 1 ) ) & 1 ) : 0u;
        const unsigned sigLower = ( cgY + 1 ) < heightInGroups ? (unsigned)( ( grpFlags >> ( grpRaster + widthInGroups ) ) & 1 ) : 0u;
        grpCtx = (int)( sigRight | sigLower );
      }
      binsAtGrpStart = remRegBins;

      bool again = false;
      for( ; inGrp >= 0; inGrp--, spos-- )      // :697-969
      {
        const int raster = scan[spos], posX = raster & ( P.regionW - 1 ), posY = raster >> lrw;
        const int cpos = ( posY << lw ) + posX;
        const int scaledMag = rq_abs( coef[cpos] ) * quantScale;
        const int roundedLvl = ( scaledMag + qHalf ) >> qShift;

        int sigCtx = 0;
        if( spos != lastPosNow )                            // sigCtxIdAbsWithAcc( iScanPos, 0 ), ContextModelling.h:158-178
        {
          const int acc = q[cpos];                                // the accumulator the decided neighbours left in this (still unvisited) slot
          const int numPos = acc >> 5, sumAbs = acc & 31;
          const int diag = posX + posY;
          sigCtx = rq_min( ( sumAbs + 1 ) >> 1, 3 ) + ( diag < 2 ? 4 : 0 );
          if( luma ) sigCtx += diag < 5 ? 4 : 0;
          tplDiag = diag; tplSum1 = sumAbs - numPos;
        }
        int ctxOffset = 0;                                        // ctxOffsetAbs, ContextModelling.h:227-236
        if( tplDiag != -1 )
        {
          ctxOffset  = rq_min( tplSum1, 4 ) + 1;
          ctxOffset += ( !tplDiag ? ( luma ? 15 : 5 ) : luma ? ( tplDiag < 3 ? 10 : ( tplDiag < 10 ? 5 : 0 ) ) : 0 );
        }
        const int32_t* fbPar = R.parBits[ctxOffset];
        const int32_t* fbGt1 = R.gt1Bits[ctxOffset];
        const int32_t* fbGt2 = R.gt2Bits[ctxOffset];
        uint32_t riceZero = 0;

        if( remRegBins < 4 )                                      // :731-736
        {
          int sum = 0;      // templateAbsSum sums abs() of the stored TCoeffSig (ContextModelling.h:242-265): a level from 32768 to 65535 is stored negative
#define RQ_SUM( v ) { sum += rq_abs( v ); }
          VVB_RQ_TEMPLATE( q, W, H, posX, posY, RQ_SUM )
#undef RQ_SUM
          const int sumAbs = rq_max( rq_min( sum, 31 ), 0 );      // templateAbsSum( ., ., 0 )
          rice = c_rqGoRicePars[sumAbs];
          riceZero  = 1u << rice;                        // g_auiGoRicePosCoeff0( 0, . ), Rom.h:137-140
        }

        zeroCost[inGrp] = rq_dist( scaledMag, errScl );

        uint32_t lvlPick = 0;
        if( roundedLvl == 0 )                                      // :748-770
        {
          sigCost  [inGrp] = C.sig[sigCtx][0];
          keepCost[inGrp] = zeroCost[inGrp] + sigCost[inGrp];
          if( bSBH )
          {
            const cost_t errOne  = scaledMag - ( (int64_t) 1 << qShift );
            const cost_t distOne = rq_dist( errOne, errScl );
            const cost_t rateOne = remRegBins < 4 ? RQ_LVL_COST( 1, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice ) -
                                                   RQ_LVL_COST( 0, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice )
                                                 : (cost_t) fbGt1[0];
            const cost_t costOne = distOne + rateOne + C.sig[sigCtx][1];
            flipDelta[inGrp] = costOne - keepCost[inGrp];
            flipStep      [inGrp] = 1;
          }
        }
        else
        {
          const int lvlDown = (int)( scaledMag >> qShift );
          const int lvlUp  = lvlDown + 1;

          if( remRegBins >= 4 && spos != lastPosNow && lvlUp >= 4 )     // :777-781
          {
            int sum = 0;
#define RQ_SUM( v ) { sum += rq_abs( v ); }
            VVB_RQ_TEMPLATE( q, W, H, posX, posY, RQ_SUM )
#undef RQ_SUM
            rice = c_rqGoRicePars[rq_max( rq_min( sum - 5 * 4, 31 ), 0 )];
          }

          if( spos == lastPosNow )                          // last level, :783-835
          {
            sigCost[inGrp] = 0;
            cost_t lastDown = zeroCost[inGrp];
            if( lvlDown )
            {
              const cost_t errDown = scaledMag - ( lvlDown << qShift );
              lastDown = rq_dist( errDown, errScl ) + RQ_LVL_COST( lvlDown, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
            }
            const cost_t errUp = scaledMag - ( lvlUp << qShift );
            const cost_t lastUp = rq_dist( errUp, errScl ) + RQ_LVL_COST( lvlUp, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );

            if( lastUp < lastDown )
            {
              lvlPick = lvlUp;
              keepCost[inGrp] = lastUp;
              if( bSBH ) { flipDelta[inGrp] = lastDown - lastUp; flipStep[inGrp] = -1; }
            }
            else
            {
              if( lvlDown == 0 )                                   // the candidate last position quantises to zero: look for the next one (goto findlast2, :816-827)
              {
                lastPosNow = -1; lastGrp = -1;
                spos--; inGrp--;
                again = true;
                break;
              }
              lvlPick = lvlDown;
              keepCost[inGrp] = lastDown;
              if( bSBH ) { flipDelta[inGrp] = lastUp - lastDown; flipStep[inGrp] = 1; }
            }
          }
          else
          {
            const cost_t sigOne = C.sig[sigCtx][1];
            if( lvlUp < 3 )                                       // levels 0, 1, 2, :840-907
            {
              const cost_t sigZero = C.sig[sigCtx][0];
              cost_t bestLvlCost = zeroCost[inGrp] + sigZero;
              cost_t bestSig = sigZero;
              cost_t costDown = bestLvlCost;
              lvlPick = 0;
              if( lvlDown == 1 )
              {
                const cost_t errDown = scaledMag - ( lvlDown << qShift );
                costDown = rq_dist( errDown, errScl ) + sigOne + RQ_LVL_COST( lvlDown, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
                if( costDown < bestLvlCost )
                {
                  lvlPick = lvlDown; bestLvlCost = costDown; bestSig = sigOne;
                  if( bSBH ) { flipDelta[inGrp] = bestLvlCost - costDown; flipStep[inGrp] = -1; }
                }
                else
                {
                  if( bSBH ) { flipDelta[inGrp] = costDown - bestLvlCost; flipStep[inGrp] = 1; }
                }
              }
              const cost_t errUp = scaledMag - ( lvlUp << qShift );
              const cost_t costUp = rq_dist( errUp, errScl ) + sigOne + RQ_LVL_COST( lvlUp, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
              if( costUp < bestLvlCost )
              {
                lvlPick = lvlUp;
                keepCost[inGrp] = costUp;
                sigCost[inGrp]   = sigOne;
                if( bSBH ) { flipDelta[inGrp] = costDown - costUp; flipStep[inGrp] = -1; }
              }
              else
              {
                keepCost[inGrp] = bestLvlCost;
                sigCost[inGrp]   = bestSig;
                if( bSBH ) { flipDelta[inGrp] = costUp - costDown; flipStep[inGrp] = 1; }
              }
            }
            else                                                  // levels x, x + 1, :908-940
            {
              const cost_t errDown = scaledMag - ( lvlDown << qShift );
              const cost_t costDown = rq_dist( errDown, errScl ) + sigOne + RQ_LVL_COST( lvlDown, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
              const cost_t errUp = scaledMag - ( lvlUp << qShift );
              const cost_t costUp = rq_dist( errUp, errScl ) + sigOne + RQ_LVL_COST( lvlUp, fbPar, fbGt1, fbGt2, remRegBins, riceZero, rice );
              sigCost[inGrp] = sigOne;
              if( costUp < costDown )
              {
                lvlPick = lvlUp;
                keepCost[inGrp] = costUp;
                if( bSBH ) { flipDelta[inGrp] = costDown - costUp; flipStep[inGrp] = -1; }
              }
              else
              {
                lvlPick = lvlDown;
                keepCost[inGrp] = costDown;
                if( bSBH ) { flipDelta[inGrp] = costUp - costDown; flipStep[inGrp] = 1; }
              }
            }
          }
          if( lvlPick )
          {
            sumGrp    += lvlPick;
            nzWeight += inGrp;
            grpFlags |= cgBit;                               // setSigGroup
            const int enc_ = VVB_RQ_ENC( (int) lvlPick );         // absVal1stPass
            VVB_RQ_DEPS( q, W, posX, posY, enc_, true, cgIdx, widthInGroups, grp )
          }
        }
        q[cpos] = (int16_t) lvlPick;                          // :942; also takes the accumulator out of a slot that stays zero

        if( ( ( spos & grpMask ) == 0 ) && ( spos > 0 ) ) rice = 0;                      // :956-963
        else if( remRegBins >= 4 ) remRegBins -= ( lvlPick < 2 ? (int) lvlPick : 3 ) + ( spos != lastPosNow );

        uncodedGrp += zeroCost[inGrp];
        codedGrp   += keepCost[inGrp];
      }
      if( !again ) break;
      seekLast = true;
    }

    //================== group significance flag, :971-1036 ===================
    cost_t grpFlagCost = 0;
    if( lastGrp >= 0 )
    {
      if( grp )
      {
        const cost_t grpFlag0 = rq_icost( P, R.sigGroupBits[grpCtx][0] );
        if( !( grpFlags & cgBit ) )
        {
          codedGrp = uncodedGrp + grpFlag0;
          grpFlagCost = grpFlag0;
        }
        else
        {
          if( grp < lastGrp )
          {
            const cost_t grpFlag1 = rq_icost( P, R.sigGroupBits[grpCtx][1] );
            grpFlagCost = grpFlag1;
            if( !nzWeight ) codedGrp -= sigCost[0];
            const cost_t uncodedGrpAlt = uncodedGrp + grpFlag0;
            codedGrp += grpFlag1;
            if( uncodedGrpAlt < codedGrp )                // cheaper as an all-zero group
            {
              grpFlags &= ~cgBit;                            // resetSigGroup
              codedGrp = uncodedGrpAlt;
              grpFlagCost = grpFlag0;
              remRegBins = binsAtGrpStart;
              for( int p = grpLen - 1; p >= 0; p-- )
              {
                const int rs_ = scan[grp * grpLen + p], px_ = rs_ & ( P.regionW - 1 ), py_ = rs_ >> lrw;
                const int bp_ = ( py_ << lw ) + px_;
                if( q[bp_] ) { const int enc_ = -VVB_RQ_ENC( rq_abs( (int) q[bp_] ) ); VVB_RQ_DEPS( q, W, px_, py_, enc_, false, cgIdx, widthInGroups, grp ) q[bp_] = 0; }      // remAbsVal1stPass
              }
              sumGrp = 0;
              if( lastGrp == grp ) { codedGrp = 0; uncodedGrp = 0; lastPosNow = -1; lastGrp = -1; }
            }
          }
          else grpFlags |= cgBit;
        }
      }
    }

    //===== last position cost, :1038-1095 =====
    bestTuCost += codedGrp;
    if( !lastSearchDone )
    {
      if( grpFlags & cgBit )
      {
        cost_t runningCost = uncodedTu + codedGrp - grpFlagCost;
        const int startIn = grp == lastGrp ? lastPosNow % grpLen : grpMask;
        int runningSum = sumGrp;
        int bestEnd = lastPosNow + 1;
        for( int pc = startIn; pc >= 0; pc-- )
        {
          const int sp = ( grp << lgGrpLen ) + pc;
          const int raster = scan[sp], px = raster & ( P.regionW - 1 ), py = raster >> lrw;
          const int bp = ( py << lw ) + px;
          if( q[bp] )
          {
            // xiGetCostLast, :445-461
            const uint32_t ctxX = c_rqGroupIdx[px], ctxY = c_rqGroupIdx[py];
            uint32_t lastBits = (uint32_t) R.lastBitsX[ctxX] + (uint32_t) R.lastBitsY[ctxY];
            if( ctxX > 3 ) lastBits += ( 1u << RQ_SCALE_BITS ) * ( ( ctxX - 2 ) >> 1 );
            if( ctxY > 3 ) lastBits += ( 1u << RQ_SCALE_BITS ) * ( ( ctxY - 2 ) >> 1 );
            const cost_t lastCost = rq_icost( P, (int) lastBits );
            const cost_t candCost = runningCost + lastCost - sigCost[pc];
            if( candCost < bestTuCost )
            {
              bestEnd = sp + 1; bestTuCost = candCost; lastGrp = grp; sumGrp = runningSum; sumTu = 0;
            }
            if( q[bp] > 1 ) { lastSearchDone = true; break; }
            runningSum -= 1;
            runningCost -= keepCost[pc];
            runningCost += zeroCost[pc];
          }
          else runningCost -= sigCost[pc];
        }
        for( int sp = bestEnd; sp <= lastPosNow; sp++ )
        {
          const int rs_ = scan[sp], px_ = rs_ & ( P.regionW - 1 ), py_ = rs_ >> lrw;
          const int bp_ = ( py_ << lw ) + px_;
          if( q[bp_] ) { const int enc_ = -VVB_RQ_ENC( rq_abs( (int) q[bp_] ) ); VVB_RQ_DEPS( q, W, px_, py_, enc_, false, cgIdx, widthInGroups, grp ) q[bp_] = 0; }
        }
        lastPosNow = bestEnd - 1;
      }
    }

    //=============== sign bit hiding, :1097-1167 ================
    if( bSBH )
    {
      if( sumGrp >= 2 )
      {
        const int grpBase = grp * grpLen;
        int lastNz = -1, firstNz = grpLen;
        for( int n = 0; n < grpLen; n++ ) if( q[RQ_BLKPOS( n + grpBase )] ) { firstNz = n; break; }
        if( lastGrp == grp )
        {
          lastNz = lastPosNow % grpLen;
          if( q[RQ_BLKPOS( lastPosNow )] == 1 && flipStep[lastNz] == -1 ) flipDelta[lastNz] -= ( 4 << RQ_SCALE_BITS );
        }
        else
        {
          for( int n = grpLen - 1; n >= 0; n-- ) if( q[RQ_BLKPOS( n + grpBase )] ) { lastNz = n; break; }
        }
        if( lastNz - firstNz >= RQ_SBH_THRESHOLD )
        {
          codedGrp -= rq_icost( P, 1 << RQ_SCALE_BITS );
          const bool negFirst = coef[RQ_BLKPOS( grpBase + firstNz )] < 0;
          if( (int) negFirst != ( sumGrp & 0x1 ) )
          {
            const int lastIn = ( lastGrp == grp ) ? lastNz : grpLen - 1;
            int64_t minDelta = INT64_MAX;
            int minAt = -1;
            if( q[RQ_BLKPOS( firstNz + grpBase )] > 1 ) { minDelta = flipDelta[firstNz]; minAt = firstNz; }
            for( int n = 0; n < firstNz; n++ )
              if( ( coef[RQ_BLKPOS( grpBase + n )] < 0 ) == negFirst )
                if( flipDelta[n] < minDelta ) { minDelta = flipDelta[n]; minAt = n; }
            for( int n = firstNz + 1; n <= lastIn; n++ )
              if( flipDelta[n] < minDelta ) { minDelta = flipDelta[n]; minAt = n; }
            const int rs_ = scan[minAt + grpBase], px_ = rs_ & ( P.regionW - 1 ), py_ = rs_ >> lrw;
            const int bp = ( py_ << lw ) + px_;
            const int encDelta_ = VVB_RQ_ENC( rq_abs( (int)(int16_t)( q[bp] + flipStep[minAt] ) ) ) - VVB_RQ_ENC( rq_abs( (int) q[bp] ) );   // :1157-1161, on the TCoeffSig
            if( encDelta_ ) VVB_RQ_DEPS( q, W, px_, py_, encDelta_, false, cgIdx, widthInGroups, grp )
            q[bp] = (int16_t)( q[bp] + flipStep[minAt] );
            sumGrp   += flipStep[minAt];
            codedGrp += minDelta;
          }
        }
      }
    }

    codedTu   += codedGrp;
    uncodedTu += uncodedGrp;
    sumTu += sumGrp;
  }

  codedTu = bestTuCost;                                // :1177

  if( lastPosNow < 0 ) { *absSumOut = sumTu; *lastPosOut = -1; return; }         // :1179-1183 (sumTu is 0 there)

  uncodedTu += rq_icost( P, R.cbfBits[0] );               // :1185-1226 (the caller resolved which context applies; zeros when the flag is inferred)
  codedTu   += rq_icost( P, R.cbfBits[1] );

  if( uncodedTu <= codedTu )                      // :1228-1233
  {
    for( int i = 0; i < W * H; i++ ) q[i] = 0;
    *absSumOut = 0; *lastPosOut = -1;
    return;
  }
  if( bSBH && q[RQ_BLKPOS( lastPosNow )] == 0 )                 // :1237-1249
  {
    int sp = lastPosNow - 1;
    for( ; sp >= 0; sp-- ) if( q[RQ_BLKPOS( sp )] ) break;
    lastPosNow = sp;
  }
  for( int sp = 0; sp <= lastPosNow; sp++ )                     // signs, :1251-1257
  {
    const int bp = RQ_BLKPOS( sp );
    const int level = q[bp];
    const int iSign = coef[bp] >> 31;
    q[bp] = (int16_t)( ( iSign ^ level ) - iSign );
  }
  *absSumOut = sumTu; *lastPosOut = lastPosNow;
#undef RQ_BLKPOS
#undef RQ_LVL_COST
}


// ------------------------------------------------------------------------------------------------------------------------------------------------------------------
// Transform-skip residual coding: QuantRDOQ::rateDistOptQuantTS (CommonLib/QuantRDOQ.cpp:1124-1336) with xGetCodedLevelTSPred (:1578-1661), xGetICRateTS (:1663-1807) and
// the transform-skip members of CoeffCodingContext (ContextModelling.h:271-407, ContextModelling.cpp:130-132) -- what QuantRDOQ2::quant runs for a transform-skipped TU
// without BDPCM (QuantRDOQ2.cpp:275-285) when Quant::m_useRDOQTS is set.  The scan runs FORWARD (group 0 first, position 0 first), the context of a position comes from its
// left and upper neighbours, costs are doubles (distortion = err * err * errorScale, rate = lambda * bits) summed in the reference's order.  The per-position cost arrays
// of the reference (m_pdCostCoeff, m_pdCostSig, m_pdCostCoeff0, m_pdCostCoeffGroupSig) are only ever read at the position that has just been written, so scalars stand in.
struct RqTsRates                     // BinFracBits::intBits of the transform-skip context sets (Contexts.cpp:821-868)
{
  int32_t sigBits[3][2];             // Ctx::TsSigFlag( numPos ), numPos = number of non-zero left / upper neighbours
  int32_t parBits[2];                // Ctx::TsParFlag( 0 )
  int32_t gtxBits[5][2];             // Ctx::TsGtxFlag( cutoffVal >> 1 ): entries 1..4 are read
  int32_t lrg1Bits[4][2];            // Ctx::TsLrg1Flag( numPos )
  int32_t signBits[6][2];            // Ctx::TsResidualSign( signCtx )
  int32_t sigGroupBits[3][2];        // Ctx::TsSigCoeffGroup( sigLeft + sigAbove )
};                                   // 44 int32

struct RqTsPar
{
  int32_t width, height, log2W;
  int32_t quantScale;                // g_quantScales[0][ qp.rem( true ) ], :1160
  int32_t qBits;                     // QUANT_SHIFT + qp.per( true ), :1159 (no transform shift, no sqrt(2) compensation)
  int32_t maxCtxBins;                // ( w * h * 7 ) >> 2, :1183
  int32_t pad[2];
  double  errorScale;                // xGetErrScaleCoeff( false, w, h, rem, 15, bitDepth, true ), QuantRDOQ.cpp:319-329
  double  lambda;                    // Quant::m_dLambda
};

VVB_HD int rq_golomb_bits( uint32_t symbol, uint32_t ricePar )            // the Golomb-Rice / exp-Golomb length of xGetICRateTS, in whole bits
{
  uint32_t length;
  const uint32_t threshold = RQ_REMAIN_BIN_REDUCTION;
  if( symbol < ( threshold << ricePar ) ) { length = symbol >> ricePar; return (int)( length + 1 + ricePar ); }
  length = ricePar;
  symbol = symbol - ( threshold << ricePar );
  while( symbol >= ( 1u << length ) ) symbol -= ( 1u << ( length++ ) );
  return (int)( threshold + length + 1 - ricePar + length );
}

// xGetICRateTS, :1663-1807
VVB_HD int rq_ts_level_rate( const RqTsRates& R, uint32_t lv, int remRegBins, const int32_t* fbSign, const int32_t* fbGt1, int& binsOfCand, int sign, uint32_t ricePar )
{
  if( remRegBins < 4 )                                            // everything by-pass coded
  {
    int rate = lv ? ( 1 << RQ_SCALE_BITS ) : 0;
    rate += rq_golomb_bits( lv, ricePar ) << RQ_SCALE_BITS;
    return rate;
  }
  else if( remRegBins < 8 )                                       // first pass context coded, the rest by-pass
  {
    int rate = fbSign[sign];
    if( lv ) binsOfCand++;
    if( lv > 1 )
    {
      rate += fbGt1[1];
      rate += R.parBits[( lv - 2 ) & 1];
      binsOfCand += 2;
      rate += rq_golomb_bits( ( lv - 2 ) >> 1, ricePar ) << RQ_SCALE_BITS;
    }
    else if( lv == 1 ) { rate += fbGt1[0]; binsOfCand++; }
    else rate = 0;
    return rate;
  }
  int rate = fbSign[sign];
  if( lv ) binsOfCand++;
  if( lv > 1 )
  {
    rate += fbGt1[1];
    rate += R.parBits[( lv - 2 ) & 1];
    binsOfCand += 2;
    uint32_t cutoffVal = 2;
    for( int i = 0; i < 4; i++ )
    {
      if( lv >= cutoffVal )
      {
        rate += R.gtxBits[cutoffVal >> 1][lv >= ( cutoffVal + 2 ) ? 1 : 0];
        binsOfCand++;
      }
      cutoffVal += 2;
    }
    if( lv >= cutoffVal ) rate += rq_golomb_bits( ( lv - cutoffVal ) >> 1, ricePar ) << RQ_SCALE_BITS;
  }
  else if( lv == 1 ) { rate += fbGt1[0]; binsOfCand++; }
  else rate = 0;
  return rate;
}

// deriveModCoeff( right, below, absCoeff, 0 ), ContextModelling.h:363-386
VVB_HD int rq_ts_mod_coeff( int leftLvl, int upLvl, int absCoeff )
{
  if( absCoeff == 0 ) return 0;
  const int pred1 = rq_max( rq_abs( upLvl ), rq_abs( leftLvl ) );
  if( absCoeff == pred1 ) return 1;
  return absCoeff < pred1 ? absCoeff + 1 : absCoeff;
}

// one transform-skipped TU.  scan as for rq_quant_tu; coef [h][w]: the residual as xTransformSkip copies it; q [h][w] levels (signed, written); absSum as the reference leaves it
VVB_HD void rq_ts_quant_tu( const RqTsPar& P, const RqTsRates& R, const int32_t* scan, const int32_t* coef, int16_t* q, int32_t* absSumOut )
{
  const int W = P.width, H = P.height, lw = P.log2W;
  const int regionW = rq_min( 32, W );
  const int lrw = ( regionW == 32 ? 5 : regionW == 16 ? 4 : regionW == 8 ? 3 : 2 );
  const int qBits = P.qBits;
  const int widthInGroups = W >> 2, heightInGroups = H >> 2;
  const int numGrp = ( W * H ) >> 4;
  const uint32_t entropyCodingMaximum = ( 1u << 15 ) - 1;
  uint64_t grpFlags = 0;
  bool anyCodedGrp = false;
  int remRegBins = P.maxCtxBins;
  int absSum = 0;

  for( int i = 0; i < W * H; i++ ) q[i] = 0;                      // the caller's level buffer starts cleared (TrQuant::transformNxN works on a cleared TU, and neighbours ahead in the scan read as zero)

  for( int grpTs = 0; grpTs < numGrp; grpTs++ )
  {
    // initSubblock: group position, the context of its significant-group flag from the left and upper groups (ContextModelling.cpp:113-133)
    const int cgRaster = scan[grpTs << 4], cgX = ( cgRaster & ( regionW - 1 ) ) >> 2, cgY = ( cgRaster >> lrw ) >> 2;
    const int grpRaster = cgY * widthInGroups + cgX;
    const uint64_t cgBit = (uint64_t) 1 << grpRaster;
    const int sigLeft  = cgX > 0 ? (int)( ( grpFlags >> ( grpRaster - 1 ) ) & 1 ) : 0;
    const int sigAbove = cgY > 0 ? (int)( ( grpFlags >> ( grpRaster - widthInGroups ) ) & 1 ) : 0;
    const int32_t* grpBitsTs = R.sigGroupBits[sigLeft + sigAbove];
    (void) heightInGroups;

    int codedInGrp = 0;
    double grpCost = 0.0;
    double keptSum = 0.0, zeroSum = 0.0, sigSum = 0.0;      // coeffGroupRDStats
    int grpBins = 0;

    for( int inGrpTs = 0; inGrpTs <= 15; inGrpTs++ )
    {
      const int scanPos = ( grpTs << 4 ) + inGrpTs;
      const int raster = scan[scanPos], posX = raster & ( regionW - 1 ), posY = raster >> lrw;
      const int blkPos = ( posY << lw ) + posX;

      const int64_t wide = (int64_t) rq_abs( coef[blkPos] ) * P.quantScale;
      const int64_t cap = (int64_t) INT32_MAX - ( (int64_t) 1 << ( qBits - 1 ) );
      const int32_t mag = (int32_t)( wide < cap ? wide : cap );

      const uint32_t lvlNear = (uint32_t) rq_min( (int) entropyCodingMaximum, (int)( (uint32_t)( mag + ( (int32_t) 1 << ( qBits - 1 ) ) ) >> qBits ) );
      const uint32_t lvlBelow = lvlNear > 1 ? lvlNear - 1 : 1;
      const uint32_t lvlFloor = (uint32_t) rq_min( (int) entropyCodingMaximum, (int)( mag >> qBits ) );
      const uint32_t lvlAbove = (uint32_t) rq_min( (int) entropyCodingMaximum, (int)( lvlFloor + 1 ) );

      uint32_t cand[3];
      int numCand = 0;
      cand[numCand++] = lvlNear;
      if( lvlBelow != lvlNear ) cand[numCand++] = lvlBelow;

      const int leftLvl = posX > 0 ? q[blkPos - 1] : 0;        // neighTS: the left and the upper neighbour (named as in the reference)
      const int upLvl = posY > 0 ? q[blkPos - W] : 0;
      const int mappedUp = rq_ts_mod_coeff( leftLvl, upLvl, (int) lvlAbove );
      if( lvlAbove != lvlNear && lvlAbove != lvlBelow && mappedUp == 1 ) cand[numCand++] = lvlAbove;

      const double e0 = (double) mag;
      const double zeroCostTs = e0 * e0 * P.errorScale;

      // contexts from the two neighbours: significance and greater-1 count the non-zero ones, the sign context looks at their signs (ContextModelling.h:271-357)
      const int numPos = ( leftLvl != 0 ) + ( upLvl != 0 );
      const int32_t* fbSig = R.sigBits[numPos];
      const int32_t* fbGt1 = R.lrg1Bits[numPos];
      int signCtx;
      if( ( leftLvl == 0 && upLvl == 0 ) || ( leftLvl * upLvl ) < 0 ) signCtx = 0;
      else if( leftLvl >= 0 && upLvl >= 0 ) signCtx = 1;
      else signCtx = 2;
      const int32_t* fbSign = R.signBits[signCtx];
      const int sign = coef[blkPos] < 0 ? 1 : 0;
      const uint32_t rice = 1;
      const bool soleCand = inGrpTs == 15 && codedInGrp == 0;

      // xGetCodedLevelTSPred, :1578-1661
      double lvlCostTs, sigCostTs = 0.0;
      uint32_t pickTs = 0;
      int binsUsed = 0;
      {
        double sigOneTs = 0;
        int binsOfBest = 0;
        bool done = false;
        if( !soleCand && cand[0] < 3 )
        {
          if( remRegBins >= 4 ) sigCostTs = P.lambda * (double) fbSig[0];
          else                  sigCostTs = P.lambda * (double)( 1 << RQ_SCALE_BITS );
          lvlCostTs = zeroCostTs + sigCostTs;
          if( remRegBins >= 4 ) binsUsed++;
          if( cand[0] == 0 ) done = true;
        }
        else lvlCostTs = 1.7e+308;                                // MAX_DOUBLE (CommonDef.h)
        if( !done )
        {
          if( !soleCand )
          {
            if( remRegBins >= 4 ) sigOneTs = P.lambda * (double) fbSig[1];
            else                  sigOneTs = P.lambda * (double)( 1 << RQ_SCALE_BITS );
            if( cand[0] >= 3 && remRegBins >= 4 ) binsUsed++;
          }
          for( int ci = 1; ci <= numCand; ci++ )
          {
            const int lv = (int) cand[ci - 1];
            const double eCand = (double)( mag - ( (int32_t) lv << qBits ) );
            const double candErr = eCand * eCand * P.errorScale;
            int mappedLvl = lv;
            if( remRegBins >= 4 ) mappedLvl = rq_ts_mod_coeff( leftLvl, upLvl, lv );
            int binsOfCand = 0;
            double candCostTs = candErr + P.lambda * (double) rq_ts_level_rate( R, (uint32_t) mappedLvl, remRegBins, fbSign, fbGt1, binsOfCand, sign, rice );
            if( remRegBins >= 4 ) candCostTs += sigOneTs;
            if( candCostTs < lvlCostTs ) { pickTs = (uint32_t) lv; lvlCostTs = candCostTs; sigCostTs = sigOneTs; binsOfBest = binsOfCand; }
          }
          binsUsed += binsOfBest;
        }
      }

      remRegBins -= binsUsed;
      grpBins += binsUsed;
      if( pickTs > 0 ) codedInGrp++;
      const int level = (int) pickTs;
      q[blkPos] = (int16_t)( ( level != 0 && coef[blkPos] < 0 ) ? -level : level );
      grpCost   += lvlCostTs;
      sigSum += sigCostTs;
      if( q[blkPos] )
      {
        grpFlags |= cgBit;
        keptSum += lvlCostTs - sigCostTs;
        zeroSum       += zeroCostTs;
      }
    }

    if( !( grpFlags & cgBit ) )                              // :1271-1277
    {
      grpCost += P.lambda * (double) grpBitsTs[0] - sigSum;
      remRegBins += grpBins;
    }
    else if( grpTs != numGrp - 1 || anyCodedGrp )                      // :1278-1322
    {
      double zeroGrpCost = grpCost;
      grpCost   += P.lambda * (double) grpBitsTs[1];
      zeroGrpCost += P.lambda * (double) grpBitsTs[0];
      zeroGrpCost += zeroSum;
      zeroGrpCost -= keptSum;
      zeroGrpCost -= sigSum;
      if( zeroGrpCost < grpCost )
      {
        grpFlags &= ~cgBit;
        grpCost = zeroGrpCost;
        remRegBins += grpBins;
        for( int p = 0; p <= 15; p++ )
        {
          const int raster = scan[( grpTs << 4 ) + p];
          q[( ( raster >> lrw ) << lw ) + ( raster & ( regionW - 1 ) )] = 0;
        }
      }
      else anyCodedGrp = true;
    }
  }

  for( int i = 0; i < W * H; i++ ) absSum += rq_abs( q[i] );     // :1325-1335 (every position is inside the scan: transform skip exists up to 32 x 32)
  *absSumOut = absSum;
}


// ------------------------------------------------------------------------------------------------------------------------------------------------------------------
// BDPCM: QuantRDOQ::forwardRDPCM (CommonLib/QuantRDOQ.cpp:1338-1562), the quantiser of a transform-skipped TU whose CU carries a block-DPCM direction (1 horizontal, 2 vertical).
// The routine of rq_ts_quant_tu with three differences: what is quantised is the residual minus the RECONSTRUCTED left / upper neighbour (xDequantSample :1564-1576 of the level
// just chosen plus its own prediction, kept in recon), the contexts take their BDPCM variants (greater-1: numPos 3; sign: + 3; no neighbour-based level mapping), and only
// the rounded level and the one below are tried.  recon: w * h int32 of scratch per TU.  One quirk is kept on purpose: when a group is zeroed out, the member refreshes
// m_fullCoeff at index scanPos instead of blkPos (:1539) -- the reconstruction other positions predict from is the one the member has.
struct RqBdpcmPar
{
  int32_t dirMode;                   // tu.cu->bdpcmM[chType]: 1 horizontal, 2 vertical
  int32_t dqScale;                   // g_invQuantScales[0][ qp.rem( true ) ], :1383
  int32_t dqRightShift;              // IQUANT_SHIFT - qp.per( true ), :1382
  int32_t pad;
};

VVB_HD int32_t rq_dequant_sample( int level, const RqBdpcmPar& B )          // xDequantSample, :1564-1576
{
  if( B.dqRightShift > 0 )
  {
    const int32_t qAdd = (int32_t) 1 << ( B.dqRightShift - 1 );
    return (int32_t)( ( (int32_t) level * B.dqScale + qAdd ) >> B.dqRightShift );
  }
  return (int32_t)( ( (int32_t) level * B.dqScale ) * ( 1 << -B.dqRightShift ) );
}

VVB_HD void rq_bdpcm_quant_tu( const RqTsPar& P, const RqBdpcmPar& B, const RqTsRates& R, const int32_t* scan, const int32_t* coef, int16_t* q, int32_t* recon, int32_t* absSumOut )
{
  const int W = P.width, H = P.height, lw = P.log2W;
  const int regionW = rq_min( 32, W );
  const int lrw = ( regionW == 32 ? 5 : regionW == 16 ? 4 : regionW == 8 ? 3 : 2 );
  const int qBits = P.qBits;
  const int widthInGroups = W >> 2;
  const int numGrp = ( W * H ) >> 4;
  const uint32_t entropyCodingMaximum = ( 1u << 15 ) - 1;
  const int dirMode = B.dirMode;
  uint64_t grpFlags = 0;
  bool anyCodedGrp = false;
  int remRegBins = P.maxCtxBins;
  int absSum = 0;

  for( int i = 0; i < W * H; i++ ) { q[i] = 0; recon[i] = 0; }       // :1368-1370

  for( int grpTs = 0; grpTs < numGrp; grpTs++ )
  {
    const int cgRaster = scan[grpTs << 4], cgX = ( cgRaster & ( regionW - 1 ) ) >> 2, cgY = ( cgRaster >> lrw ) >> 2;
    const int grpRaster = cgY * widthInGroups + cgX;
    const uint64_t cgBit = (uint64_t) 1 << grpRaster;
    const int sigLeft  = cgX > 0 ? (int)( ( grpFlags >> ( grpRaster - 1 ) ) & 1 ) : 0;
    const int sigAbove = cgY > 0 ? (int)( ( grpFlags >> ( grpRaster - widthInGroups ) ) & 1 ) : 0;
    const int32_t* grpBitsTs = R.sigGroupBits[sigLeft + sigAbove];

    int codedInGrp = 0;
    double grpCost = 0.0;
    double keptSum = 0.0, zeroSum = 0.0, sigSum = 0.0;
    int grpBins = 0;

    for( int inGrpTs = 0; inGrpTs <= 15; inGrpTs++ )
    {
      const int scanPos = ( grpTs << 4 ) + inGrpTs;
      const int raster = scan[scanPos], posX = raster & ( regionW - 1 ), posY = raster >> lrw;
      const int blkPos = ( posY << lw ) + posX;
      const int posS = ( 1 == dirMode ) ? posX : posY;
      const int posNb = ( 1 == dirMode ) ? ( posX - 1 ) + posY * W : posX + ( posY - 1 ) * W;
      const int32_t pred = ( 0 != posS ) ? recon[posNb] : 0;

      const int64_t wide = (int64_t) rq_abs( coef[blkPos] - pred ) * P.quantScale;
      const int64_t cap = (int64_t) INT32_MAX - ( (int64_t) 1 << ( qBits - 1 ) );
      const int32_t mag = (int32_t)( wide < cap ? wide : cap );
      const uint32_t lvlNear = (uint32_t) rq_min( (int) entropyCodingMaximum, (int)( (uint32_t)( mag + ( (int32_t) 1 << ( qBits - 1 ) ) ) >> qBits ) );
      const uint32_t lvlBelow = lvlNear > 1 ? lvlNear - 1 : 1;
      uint32_t cand[3];
      int numCand = 0;
      cand[numCand++] = lvlNear;
      if( lvlBelow != lvlNear ) cand[numCand++] = lvlBelow;

      const double e0 = (double) mag;
      const double zeroCostTs = e0 * e0 * P.errorScale;

      const int leftLvl = posX > 0 ? q[blkPos - 1] : 0;
      const int upLvl = posY > 0 ? q[blkPos - W] : 0;
      const int numPos = ( leftLvl != 0 ) + ( upLvl != 0 );
      const int32_t* fbSig = R.sigBits[numPos];                  // sigCtxIdAbsTS has no BDPCM variant
      const int32_t* fbGt1 = R.lrg1Bits[3];                      // lrg1CtxIdAbsTS( ., ., bdpcm ): numPos = 3
      int signCtx;
      if( ( leftLvl == 0 && upLvl == 0 ) || ( leftLvl * upLvl ) < 0 ) signCtx = 0;
      else if( leftLvl >= 0 && upLvl >= 0 ) signCtx = 1;
      else signCtx = 2;
      const int32_t* fbSign = R.signBits[signCtx + 3];           // signCtxIdAbsTS( ., ., bdpcm ): + 3
      const int sign = coef[blkPos] - pred < 0 ? 1 : 0;
      const uint32_t rice = 1;
      const bool soleCand = inGrpTs == 15 && codedInGrp == 0;

      double lvlCostTs, sigCostTs = 0.0;
      uint32_t pickTs = 0;
      int binsUsed = 0;
      {
        double sigOneTs = 0;
        int binsOfBest = 0;
        bool done = false;
        if( !soleCand && cand[0] < 3 )
        {
          if( remRegBins >= 4 ) sigCostTs = P.lambda * (double) fbSig[0];
          else                  sigCostTs = P.lambda * (double)( 1 << RQ_SCALE_BITS );
          lvlCostTs = zeroCostTs + sigCostTs;
          if( remRegBins >= 4 ) binsUsed++;
          if( cand[0] == 0 ) done = true;
        }
        else lvlCostTs = 1.7e+308;
        if( !done )
        {
          if( !soleCand )
          {
            if( remRegBins >= 4 ) sigOneTs = P.lambda * (double) fbSig[1];
            else                  sigOneTs = P.lambda * (double)( 1 << RQ_SCALE_BITS );
            if( cand[0] >= 3 && remRegBins >= 4 ) binsUsed++;
          }
          for( int ci = 1; ci <= numCand; ci++ )
          {
            const int lv = (int) cand[ci - 1];
            const double eCand = (double)( mag - ( (int32_t) lv << qBits ) );
            const double candErr = eCand * eCand * P.errorScale;
            int binsOfCand = 0;                                   // deriveModCoeff( ., ., lv, bdpcm != 0 ) leaves the level as it is
            double candCostTs = candErr + P.lambda * (double) rq_ts_level_rate( R, (uint32_t) lv, remRegBins, fbSign, fbGt1, binsOfCand, sign, rice );
            if( remRegBins >= 4 ) candCostTs += sigOneTs;
            if( candCostTs < lvlCostTs ) { pickTs = (uint32_t) lv; lvlCostTs = candCostTs; sigCostTs = sigOneTs; binsOfBest = binsOfCand; }
          }
          binsUsed += binsOfBest;
        }
      }

      remRegBins -= binsUsed;
      grpBins += binsUsed;
      if( pickTs > 0 ) codedInGrp++;
      q[blkPos] = (int16_t)( sign ? -(int) pickTs : (int) pickTs );
      recon[blkPos] = rq_dequant_sample( q[blkPos], B ) + pred;          // :1491-1492
      grpCost   += lvlCostTs;
      sigSum += sigCostTs;
      if( q[blkPos] )
      {
        grpFlags |= cgBit;
        keptSum += lvlCostTs - sigCostTs;
        zeroSum       += zeroCostTs;
      }
    }

    if( !( grpFlags & cgBit ) )
    {
      grpCost += P.lambda * (double) grpBitsTs[0] - sigSum;
      remRegBins += grpBins;
    }
    else if( grpTs != numGrp - 1 || anyCodedGrp )
    {
      double zeroGrpCost = grpCost;
      grpCost   += P.lambda * (double) grpBitsTs[1];
      zeroGrpCost += P.lambda * (double) grpBitsTs[0];
      zeroGrpCost += zeroSum;
      zeroGrpCost -= keptSum;
      zeroGrpCost -= sigSum;
      if( zeroGrpCost < grpCost )
      {
        grpFlags &= ~cgBit;
        grpCost = zeroGrpCost;
        remRegBins += grpBins;
        for( int p = 0; p <= 15; p++ )
        {
          const int scanPos = ( grpTs << 4 ) + p;
          const int raster = scan[scanPos], posX = raster & ( regionW - 1 ), posY = raster >> lrw;
          const int blkPos = ( posY << lw ) + posX;
          const int posS = ( 1 == dirMode ) ? posX : posY;
          const int posNb = ( 1 == dirMode ) ? ( posX - 1 ) + posY * W : posX + ( posY - 1 ) * W;
          recon[scanPos] = ( 0 != posS ) ? recon[posNb] : 0;              // the member indexes by scanPos here (:1539)
          q[blkPos] = 0;
        }
      }
      else anyCodedGrp = true;
    }
  }

  for( int i = 0; i < W * H; i++ ) absSum += rq_abs( q[i] );
  *absSumOut = absSum;
}

} // namespace vvbrq
