/* tests/mock/vvb_mock.c -- TEST INFRASTRUCTURE: the subset of the C ABI (include/vvenc_b200.h) that the reference-side bindings in integration/ call,
 * answered by the CPU oracle (oracle/oracle.c is compiled into this library).  It lets the host logic of integration/ headers -- argument marshalling, the
 * replay of the selection rounds on the returned tables -- run next to the reference's own member functions on a machine without a GPU
 * (tests/test_integration_host.py).  It is never shipped, never loaded by the product package, and no `-m gpu` test or bench leg uses it. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/vvenc_b200.h"

typedef int16_t Pel;
/* oracle entry points (oracle/oracle.c) */
void     orc_full_search( const Pel* orgPlane, int so, const Pel* refPlane, int sr, const int32_t* blk, int n, int subShift, double lambda, int costScale, int imvShift,
                          int32_t* out, uint32_t* sadTables, int tableStride );
uint64_t orc_mv_cost( double lambda, int x, int y, int predHor, int predVer, int costScale, int imvShift );
void     orc_frac_cost_grid( const Pel* orgPlane, int so, const Pel* refPlane, int sr, const int32_t* blk, int n, int family, int bitDepth, int reduceTap, int altHpel, uint32_t* out );
int      orc_dep_quant( int w, int h, int bitDepth, int qp, double lambda, int dqThrVal, int zeroOut, int lfnst, int scalarMembers, const int32_t* rates, const int32_t* coef, int n,
                        int16_t* q, int32_t* absSum, int32_t* lastPos );   /* oracle/depquant_oracle.cpp */
int      orc_dep_quant_chroma( int w, int h, int bitDepth, int qp, double lambda, int dqThrVal, int lfnst, int scalarMembers, const int32_t* rates, const int32_t* coef, int n,
                               int16_t* q, int32_t* absSum, int32_t* lastPos );
int      orc_rdoq( int w, int h, int bitDepth, int qp, int isChroma, int lfnst, int sbtZeroOut, int signHiding, double lambda, int thrVal, const int32_t* rates,
                   const int32_t* coef, int n, int16_t* q, int32_t* absSum, int32_t* lastPos );   /* oracle/rdoq_oracle.cpp */
int      orc_rdoq_ts( int w, int h, int bitDepth, int qp, int inputDelta, double lambda, const int32_t* rates, const int32_t* coef, int n, int16_t* q, int32_t* absSum );
int      orc_rdoq_bdpcm( int w, int h, int bitDepth, int qp, int inputDelta, int dirMode, double lambda, const int32_t* rates, const int32_t* coef, int n, int16_t* q, int32_t* absSum );
void     orc_mctf_err_list( int tap4, const Pel* orgPlane, int so, const Pel* bufPlane, int sb, const int32_t* desc, int n, int bitDepth, int32_t* out );

#define MOCK_PLANES 64
typedef struct { Pel* mem; Pel* origin; int stride, width, height, margin, bitDepth; } mock_plane;
struct vvb_ctx { mock_plane pl[MOCK_PLANES]; char err[256]; uint64_t calls; };

static int fail( vvb_ctx* c, int code, const char* msg ) { snprintf( c->err, sizeof( c->err ), "%s", msg ); return code; }

int vvb_create( vvb_ctx** out, int device ) { (void) device; if( !out ) return VVB_ERR_ARG; *out = (vvb_ctx*) calloc( 1, sizeof( vvb_ctx ) ); return *out ? VVB_OK : VVB_ERR_NOMEM; }
void vvb_destroy( vvb_ctx* c ) { if( !c ) return; for( int i = 0; i < MOCK_PLANES; i++ ) free( c->pl[i].mem ); free( c ); }
const char* vvb_last_error( const vvb_ctx* c ) { return c ? c->err : "no context"; }
int vvb_launch_count( const vvb_ctx* c, uint64_t* n ) { if( !c || !n ) return VVB_ERR_ARG; *n = c->calls; return VVB_OK; }

int vvb_set_tma_staging( vvb_ctx* c, int enable ) { if( !c || enable < 0 || enable > 2 ) return VVB_ERR_ARG; return VVB_OK; }   /* staging choice of the real kernel: nothing to do here */

int vvb_plane_upload( vvb_ctx* c, int id, const int16_t* origin, int stride, int width, int height, int margin, int bitDepth )
{
  if( !c || id < 0 || id >= MOCK_PLANES - 2 || !origin || width <= 0 || height <= 0 || margin < 0 || stride < width + 2 * margin ) return c ? fail( c, VVB_ERR_ARG, "bad plane arguments" ) : VVB_ERR_ARG;
  mock_plane* p = &c->pl[id];
  free( p->mem );
  const int s = width + 2 * margin;
  p->mem = (Pel*) malloc( sizeof( Pel ) * (size_t) s * ( height + 2 * margin ) );
  if( !p->mem ) return fail( c, VVB_ERR_NOMEM, "plane" );
  for( int y = -margin; y < height + margin; y++ ) memcpy( p->mem + (size_t)( y + margin ) * s, origin + (ptrdiff_t) y * stride - margin, sizeof( Pel ) * s );
  p->origin = p->mem + (size_t) margin * s + margin; p->stride = s; p->width = width; p->height = height; p->margin = margin; p->bitDepth = bitDepth;
  return VVB_OK;
}
int vvb_plane_free( vvb_ctx* c, int id ) { if( !c || id < 0 || id >= MOCK_PLANES ) return VVB_ERR_ARG; free( c->pl[id].mem ); memset( &c->pl[id], 0, sizeof( mock_plane ) ); return VVB_OK; }

static int is_pow2( int v ) { return v > 0 && ( v & ( v - 1 ) ) == 0; }
/* The argument checks below repeat those of vvenc_b200/csrc/capi.cu, so that a binding which passes here does not trip over a validation on the real library. */
static mock_plane* plane( vvb_ctx* c, int id ) { return ( id >= 0 && id < MOCK_PLANES && c->pl[id].mem ) ? &c->pl[id] : NULL; }

int vvb_sad_search( vvb_ctx* c, int orgPlane, int refPlane, const vvb_block* blocks, int n, int w, int h, const vvb_me_par* par, uint32_t* sadTables, int tableStride, vvb_best* bestOut )
{
  if( !c ) return VVB_ERR_ARG;
  mock_plane* o = plane( c, orgPlane ); mock_plane* r = plane( c, refPlane );
  if( !o || !r || !blocks || !par || !bestOut || n < 0 ) return fail( c, VVB_ERR_ARG, "bad search arguments" );
  if( !is_pow2( w ) || !is_pow2( h ) || w < 4 || h < 4 || w > 128 || h > 128 ) return fail( c, VVB_ERR_UNSUPPORTED, "search blocks are 4..128 powers of two" );
  if( par->sub_shift && ( h & ( ( 1 << par->sub_shift ) - 1 ) ) ) return fail( c, VVB_ERR_UNSUPPORTED, "subShift needs an even height" );
  for( int i = 0; i < n; i++ )
  {
    const vvb_block* b = &blocks[i];
    if( -b->left > r->margin || b->right > r->margin || -b->top > r->margin || b->bottom > r->margin ) return fail( c, VVB_ERR_ARG, "search range exceeds the plane margin" );
    const int nx = b->right - b->left + 1, ny = b->bottom - b->top + 1;
    if( nx < 1 || ny < 1 ) return fail( c, VVB_ERR_ARG, "empty search range" );
    if( sadTables && nx * ny > tableStride ) return fail( c, VVB_ERR_ARG, "table_stride smaller than the window" );
    if( nx * ny > 65536 ) return fail( c, VVB_ERR_UNSUPPORTED, "search window above 65536 positions" );
    if( (size_t)( w + nx ) * ( h + ny ) * 2 > 220 * 1024 ) return fail( c, VVB_ERR_UNSUPPORTED, "search window does not fit shared memory (reduce the range)" );
    const int32_t blk[10] = { b->x, b->y, w, h, b->left, b->right, b->top, b->bottom, b->pred_hor, b->pred_ver };
    int32_t out[4];
    orc_full_search( o->origin, o->stride, r->origin, r->stride, blk, 1, par->sub_shift, par->lambda, par->cost_scale, par->imv_shift, out,
                     sadTables ? sadTables + (size_t) i * tableStride : NULL, tableStride );
    const uint64_t cost = (uint32_t) out[2] | ( (uint64_t)(uint32_t) out[3] << 32 );
    bestOut[i].dx = (int16_t) out[0]; bestOut[i].dy = (int16_t) out[1]; bestOut[i].cost = cost;
    bestOut[i].sad = (uint32_t)( cost - orc_mv_cost( par->lambda, out[0], out[1], b->pred_hor, b->pred_ver, par->cost_scale, par->imv_shift ) );
  }
  c->calls++;
  return VVB_OK;
}

int vvb_frac_cost_grid( vvb_ctx* c, int dfunc, int orgPlane, int refPlane, const vvb_block* blocks, int n, int w, int h, int reduceTap, int altHpel, uint32_t* costOut )
{
  if( !c ) return VVB_ERR_ARG;
  mock_plane* o = plane( c, orgPlane ); mock_plane* r = plane( c, refPlane );
  if( !o || !r || !blocks || !costOut || n < 0 ) return fail( c, VVB_ERR_ARG, "bad grid arguments" );
  if( dfunc != VVB_DF_SAD && dfunc != VVB_DF_HAD && dfunc != VVB_DF_HAD_FAST ) return fail( c, VVB_ERR_UNSUPPORTED, "fractional grid: SAD, HAD or HAD_fast" );
  if( !is_pow2( w ) || !is_pow2( h ) || w < 4 || h < 4 || w > 64 || h > 64 ) return fail( c, VVB_ERR_UNSUPPORTED, "fractional grid: PU sides 4..64, powers of two" );
  if( reduceTap < 0 || reduceTap > 2 ) return fail( c, VVB_ERR_ARG, "reduce_tap is 0, 1 or 2" );
  for( int i = 0; i < n; i++ )
  {
    const vvb_block* b = &blocks[i];
    const int reach = ( abs( b->start_x ) > abs( b->start_y ) ? abs( b->start_x ) : abs( b->start_y ) ) + 5;
    if( reach > r->margin ) return fail( c, VVB_ERR_ARG, "vector + filter reach exceeds the plane margin" );
    const int32_t blk[6] = { b->x, b->y, w, h, b->start_x, b->start_y };
    orc_frac_cost_grid( o->origin, o->stride, r->origin, r->stride, blk, 1, dfunc == VVB_DF_HAD_FAST ? 3 : ( dfunc == VVB_DF_HAD ? 2 : 1 ), o->bitDepth, reduceTap, altHpel, costOut + (size_t) i * 49 );
  }
  c->calls++;
  return VVB_OK;
}

int vvb_mctf_error_batch( vvb_ctx* c, int orgPlane, int refPlane, const vvb_mctf_cand* cands, int n, int lowRes, int32_t* errOut )
{
  if( !c ) return VVB_ERR_ARG;
  mock_plane* o = plane( c, orgPlane ); mock_plane* r = plane( c, refPlane );
  if( !o || !r || !cands || !errOut || n < 0 ) return fail( c, VVB_ERR_ARG, "bad mctf arguments" );
  if( o->bitDepth > 10 || r->bitDepth > 10 ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF supports up to 10 bit (MCTF.cpp:1313 CHECKD)" );
  for( int i = 0; i < n; i++ )
    if( cands[i].w < 8 || cands[i].h < 8 || cands[i].w > 64 || cands[i].h > 64 || ( cands[i].w & 7 ) || ( cands[i].h & 7 ) ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF blocks are multiples of 8 up to 64" );
  for( int i = 0; i < n; i++ )
  {
    const int32_t d[6] = { cands[i].x, cands[i].y, cands[i].mvx, cands[i].mvy, cands[i].w, cands[i].h };
    orc_mctf_err_list( lowRes, o->origin, o->stride, r->origin, r->stride, d, 1, o->bitDepth, errOut + i );
  }
  c->calls++;
  return VVB_OK;
}

int vvb_mctf_search_grid( vvb_ctx* c, int orgPlane, int refPlane, const vvb_mctf_cand* blocks, int n, int step, int radius, int lowRes, int32_t* errOut )
{
  if( !c ) return VVB_ERR_ARG;
  mock_plane* o = plane( c, orgPlane ); mock_plane* r = plane( c, refPlane );
  if( !o || !r || !blocks || !errOut || n < 0 ) return fail( c, VVB_ERR_ARG, "bad mctf grid arguments" );
  if( o->bitDepth > 10 || r->bitDepth > 10 ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF supports up to 10 bit (MCTF.cpp:1313 CHECKD)" );
  if( step < 1 || step > 16 || radius < 0 || radius > 8 ) return fail( c, VVB_ERR_ARG, "MCTF grid: step 1..16 (1/16 pel), radius 0..8 steps" );
  for( int i = 0; i < n; i++ )
    if( blocks[i].w < 8 || blocks[i].h < 8 || blocks[i].w > 64 || blocks[i].h > 64 || ( blocks[i].w & 7 ) || ( blocks[i].h & 7 ) ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF blocks are multiples of 8 up to 64" );
  const int side = 2 * radius + 1;
  for( int i = 0; i < n; i++ )
    for( int j = 0; j < side; j++ )
      for( int k = 0; k < side; k++ )
      {
        const int32_t d[6] = { blocks[i].x, blocks[i].y, blocks[i].mvx + ( k - radius ) * step, blocks[i].mvy + ( j - radius ) * step, blocks[i].w, blocks[i].h };
        orc_mctf_err_list( lowRes, o->origin, o->stride, r->origin, r->stride, d, 1, o->bitDepth, errOut + ( (size_t) i * side + j ) * side + k );
      }
  c->calls++;
  return VVB_OK;
}

int orc_transform_quant_lfnst( const Pel* resi, int stride, int w, int h, int bitDepth, int qp, int isIRAP, int signHiding, int set, int lfnstIdx, int transpose, int32_t* coef, int16_t* q, int32_t* absSum, int32_t* lastPos );
int orc_transform_quant_ex( int trHor, int trVer, const Pel* resi, int stride, int w, int h, int bitDepth, int qp, int isIRAP, int signHiding, int32_t* coef, int16_t* q, int32_t* absSum, int32_t* lastPos );
int orc_need_rdoq( const int32_t* coef, int w, int h, int bitDepth, int qp, int depQuant );
int orc_need_rdoq_ex( const int32_t* coef, int w, int h, int bitDepth, int qp, int depQuant, int transformSkip, int inputDelta, int chroma );
int orc_transform_quant_ts( const Pel* resi, int stride, int w, int h, int bitDepth, int qp, int isIRAP, int signHiding, int inputDelta, int32_t* coef, int16_t* q, int32_t* absSum, int32_t* lastPos );
int orc_inv_transform_quant_ts( const int16_t* q, int w, int h, int bitDepth, int qp, int inputDelta, int32_t* coef, Pel* resi, int stride );
int orc_inv_transform_quant_dq( int trHor, int trVer, const int16_t* q, int w, int h, int bitDepth, int qp, int32_t* coef, Pel* resi, int stride );
int orc_inv_transform_quant_lfnst( const int16_t* q, int w, int h, int bitDepth, int qp, int depQuant, int set, int lfnstIdx, int transpose, int32_t* coef, Pel* resi, int stride );
int orc_inv_transform_quant( int trHor, int trVer, const int16_t* q, int w, int h, int bitDepth, int qp, int32_t* coef, Pel* resi, int stride );

static int tu_par_ok( vvb_ctx* c, const vvb_tu_par* p )
{
  if( !is_pow2( p->w ) || !is_pow2( p->h ) || p->w < 4 || p->h < 4 || p->w > 64 || p->h > 64 ) return fail( c, VVB_ERR_UNSUPPORTED, "TU sizes are 4..64" );
  if( p->tr_hor < 0 || p->tr_hor > 2 || p->tr_ver < 0 || p->tr_ver > 2 ) return fail( c, VVB_ERR_ARG, "unknown transform type" );
  if( ( p->tr_hor && p->w > 32 ) || ( p->tr_ver && p->h > 32 ) ) return fail( c, VVB_ERR_UNSUPPORTED, "DST-VII/DCT-VIII exist for 4..32 only" );
  if( p->bit_depth < 8 || p->bit_depth > 12 ) return fail( c, VVB_ERR_UNSUPPORTED, "bit depth 8..12" );
  return VVB_OK;
}

int vvb_fwd_trquant( vvb_ctx* c, const vvb_tu_par* par, const int16_t* resi, int n, int32_t* coef, int16_t* q, int32_t* absSum, int32_t* lastPos, uint8_t* needRdoq )
{
  if( !c ) return VVB_ERR_ARG;
  if( !par || !resi || !q || n < 0 ) return fail( c, VVB_ERR_ARG, "bad trquant arguments" );
  if( tu_par_ok( c, par ) ) return VVB_ERR_UNSUPPORTED;
  const size_t area = (size_t) par->w * par->h;
  int32_t* tmp = (int32_t*) malloc( sizeof( int32_t ) * area );
  if( !tmp ) return fail( c, VVB_ERR_NOMEM, "trquant" );
  for( int i = 0; i < n; i++ )
  {
    int32_t s = 0, l = -1;
    int32_t* co = coef ? coef + area * i : tmp;
    const int rc = par->transform_skip
      ? orc_transform_quant_ts( resi + area * i, par->w, par->w, par->h, par->bit_depth, par->qp, par->is_irap, par->sign_hiding, par->input_bit_depth_delta, co, q + area * i, &s, &l )
      : par->lfnst_idx
      ? orc_transform_quant_lfnst( resi + area * i, par->w, par->w, par->h, par->bit_depth, par->qp, par->is_irap, par->sign_hiding, par->lfnst_set, par->lfnst_idx, par->lfnst_transpose, co, q + area * i, &s, &l )
      : orc_transform_quant_ex( par->tr_hor, par->tr_ver, resi + area * i, par->w, par->w, par->h, par->bit_depth, par->qp, par->is_irap, par->sign_hiding, co, q + area * i, &s, &l );
    if( rc ) { free( tmp ); return fail( c, VVB_ERR_UNSUPPORTED, "transform shape" ); }
    if( absSum ) absSum[i] = s;
    if( lastPos ) lastPos[i] = l;
    if( needRdoq ) needRdoq[i] = (uint8_t) orc_need_rdoq_ex( co, par->w, par->h, par->bit_depth, par->qp, par->dep_quant, par->transform_skip, par->input_bit_depth_delta, par->is_chroma );
  }
  free( tmp );
  c->calls++;
  return VVB_OK;
}

int vvb_inv_trquant( vvb_ctx* c, const vvb_tu_par* par, const int16_t* q, int n, int16_t* resi )
{
  if( !c ) return VVB_ERR_ARG;
  if( !par || !resi || !q || n < 0 ) return fail( c, VVB_ERR_ARG, "bad inverse arguments" );
  if( tu_par_ok( c, par ) ) return VVB_ERR_UNSUPPORTED;
  const size_t area = (size_t) par->w * par->h;
  int32_t* tmp = (int32_t*) malloc( sizeof( int32_t ) * area );
  if( !tmp ) return fail( c, VVB_ERR_NOMEM, "inverse" );
  for( int i = 0; i < n; i++ )
    if( par->transform_skip ? orc_inv_transform_quant_ts( q + area * i, par->w, par->h, par->bit_depth, par->qp, par->input_bit_depth_delta, tmp, resi + area * i, par->w )
        : par->lfnst_idx    ? orc_inv_transform_quant_lfnst( q + area * i, par->w, par->h, par->bit_depth, par->qp, par->dep_quant, par->lfnst_set, par->lfnst_idx, par->lfnst_transpose, tmp, resi + area * i, par->w )
        : par->dep_quant    ? orc_inv_transform_quant_dq( par->tr_hor, par->tr_ver, q + area * i, par->w, par->h, par->bit_depth, par->qp, tmp, resi + area * i, par->w )
                            : orc_inv_transform_quant( par->tr_hor, par->tr_ver, q + area * i, par->w, par->h, par->bit_depth, par->qp, tmp, resi + area * i, par->w ) )
    { free( tmp ); return fail( c, VVB_ERR_UNSUPPORTED, "transform shape" ); }
  free( tmp );
  c->calls++;
  return VVB_OK;
}

double orc_mctf_calc_var( const Pel* org, int so, int w, int h );
int vvb_mctf_calc_var( vvb_ctx* c, int planeId, const vvb_mctf_cand* blocks, int n, double* varOut )
{
  if( !c ) return VVB_ERR_ARG;
  mock_plane* o = plane( c, planeId );
  if( !o || !blocks || !varOut || n < 0 ) return fail( c, VVB_ERR_ARG, "bad calc_var arguments" );
  if( o->bitDepth > 10 ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF supports up to 10 bit (MCTF.cpp:1313 CHECKD)" );
  for( int i = 0; i < n; i++ ) varOut[i] = orc_mctf_calc_var( o->origin + (ptrdiff_t) blocks[i].y * o->stride + blocks[i].x, o->stride, blocks[i].w, blocks[i].h );
  c->calls++;
  return VVB_OK;
}

void orc_mctf_finalize_block( const Pel* orgPlane, int so, const Pel* const* refs, int rs, int numRefs, const int32_t* mv4, int bx, int by, int w, int h,
                              int bitDepth, int tap4, int planarEnabled, const double* refStrengths, double weightScaling, double sigmaSq, Pel* dstPlane, int ds );
int vvb_mctf_apply( vvb_ctx* c, int orgPlane, const vvb_mctf_apply_par* par, const vvb_mctf_mv* mvs, int16_t* out, int outStride )
{
  if( !c ) return VVB_ERR_ARG;
  mock_plane* o = plane( c, orgPlane );
  if( !o || !par || !mvs || !out || par->num_refs < 1 || par->num_refs > 8 ) return fail( c, VVB_ERR_ARG, "bad apply arguments" );
  if( par->block_size != 8 && par->block_size != 16 && par->block_size != 32 ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF unit size 8, 16 or 32" );
  if( ( o->width & 7 ) || ( o->height & 7 ) ) return fail( c, VVB_ERR_UNSUPPORTED, "picture dimensions must be multiples of 8" );
  if( o->bitDepth > 10 ) return fail( c, VVB_ERR_UNSUPPORTED, "MCTF supports up to 10 bit" );
  const Pel* refs[8]; int rs = 0;
  for( int i = 0; i < par->num_refs; i++ )
  {
    mock_plane* r = plane( c, par->ref_plane[i] );
    if( !r || ( i && r->stride != rs ) ) return fail( c, VVB_ERR_ARG, "reference planes missing or of different geometry" );
    refs[i] = r->origin; rs = r->stride;
  }
  const int B = par->block_size, bxN = ( o->width + B - 1 ) / B, byN = ( o->height + B - 1 ) / B;
  for( int by = 0; by < byN; by++ )
    for( int bx = 0; bx < bxN; bx++ )
    {
      int32_t mv4[8 * 4];
      for( int i = 0; i < par->num_refs; i++ )
      {
        const vvb_mctf_mv* v = &mvs[( (size_t) i * byN + by ) * bxN + bx];
        mv4[4 * i] = v->x; mv4[4 * i + 1] = v->y; mv4[4 * i + 2] = v->error; mv4[4 * i + 3] = v->rmsme;
      }
      const int x = bx * B, y = by * B, w = o->width - x < B ? o->width - x : B, h = o->height - y < B ? o->height - y : B;
      orc_mctf_finalize_block( o->origin, o->stride, refs, rs, par->num_refs, mv4, x, y, w, h, o->bitDepth, par->low_res_filter, par->planar_correction,
                               par->ref_strength, par->weight_scaling, par->sigma_sq, out, outStride );
    }
  c->calls++;
  return VVB_OK;
}

void orc_sobel( int vertical, const Pel* p, int ps, Pel* d, int ds, int w, int h );
void orc_equal_coeff( int sixParam, const Pel* resi, int rs, const Pel* gx, const Pel* gy, int ds, int w, int h, int64_t* eq );
int vvb_affine_sobel( vvb_ctx* c, int vertical, const int16_t* pred, int ps, int16_t* deriv, int ds, int w, int h )
{
  if( !c ) return VVB_ERR_ARG;
  if( !pred || !deriv ) return fail( c, VVB_ERR_ARG, "null pointer" );
  if( w < 4 || h < 4 || w > 128 || h > 128 ) return fail( c, VVB_ERR_UNSUPPORTED, "affine blocks are 4..128" );
  orc_sobel( vertical, pred, ps, deriv, ds, w, h );
  c->calls++;
  return VVB_OK;
}
int vvb_affine_equal_coeff( vvb_ctx* c, int sixParam, const int16_t* resi, int rs, const int16_t* dx, const int16_t* dy, int ds, int w, int h, int64_t eq[49] )
{
  if( !c ) return VVB_ERR_ARG;
  if( !resi || !dx || !dy || !eq ) return fail( c, VVB_ERR_ARG, "bad equal_coeff arguments" );
  orc_equal_coeff( sixParam, resi, rs, dx, dy, ds, w, h, eq );
  c->calls++;
  return VVB_OK;
}

/* per-block entry points (FpDistFunc-shaped, RdCostB200.h) */
uint64_t orc_dist( int family, const Pel* org, int so, const Pel* cur, int sc, int w, int h, int subShift );
uint64_t orc_sad_mask( const Pel* org, int so, const Pel* cur, int sc, int w, int h, const Pel* mask, int maskStride, int stepX, int maskStride2, int subShift );
void     orc_sad_x5( const Pel* org, int so, const Pel* cur, int sc, int w, int h, int subShift, int calcCentre, uint64_t* cost5 );
uint64_t orc_fix_wsse( const Pel* org, int so, const Pel* cur, int sc, int w, int h, uint32_t weight );

uint64_t vvb_dist_block( vvb_ctx* c, int dfunc, const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, int bitDepth, int subShift, int* err )
{
  (void) bitDepth;
  if( err ) *err = VVB_OK;
  if( !c || !org || !cur || dfunc < 0 || dfunc > 4 ) { if( err ) *err = VVB_ERR_ARG; return 0; }
  c->calls++;
  return orc_dist( dfunc, org, so, cur, sc, w, h, subShift );
}
uint64_t vvb_sad_mask_block( vvb_ctx* c, const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, const int16_t* mask, int maskStride, int stepX, int maskStride2,
                             int subShift, int* err )
{
  if( err ) *err = VVB_OK;
  if( !c || !org || !cur || !mask ) { if( err ) *err = VVB_ERR_ARG; return 0; }
  c->calls++;
  return orc_sad_mask( org, so, cur, sc, w, h, mask, maskStride, stepX, maskStride2, subShift );
}
int vvb_sad_x5_block( vvb_ctx* c, const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, int subShift, int calcCentre, uint64_t cost5[5] )
{
  if( !c || !org || !cur || !cost5 ) return VVB_ERR_ARG;
  c->calls++;
  orc_sad_x5( org, so, cur, sc, w, h, subShift, calcCentre, cost5 );
  return VVB_OK;
}
uint64_t vvb_fix_wsse_block( vvb_ctx* c, const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, uint32_t weight, int* err )
{
  if( err ) *err = VVB_OK;
  if( !c || !org || !cur ) { if( err ) *err = VVB_ERR_ARG; return 0; }
  c->calls++;
  return orc_fix_wsse( org, so, cur, sc, w, h, weight );
}

int vvb_dep_quant( vvb_ctx* c, const vvb_tu_par* par, const vvb_dq_par* dq, const vvb_dq_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n,
                   int16_t* q, int32_t* abs_sum, int32_t* last_pos )
{
  if( !c ) return VVB_ERR_ARG;
  if( !par || !dq || !rates || !coef || !q || n < 0 || !( dq->lambda > 0.0 ) ) return fail( c, VVB_ERR_ARG, "bad dependent quantisation arguments" );
  const size_t area = (size_t) par->w * par->h;
  for( int i = 0; i < n; i++ )
  {
    int32_t s = 0, l = -1;
    if( need_rdoq && !need_rdoq[i] ) memset( q + i * area, 0, sizeof( int16_t ) * area );
    else if( par->is_chroma ? orc_dep_quant_chroma( par->w, par->h, par->bit_depth, par->qp, dq->lambda, dq->dq_thr_val, par->lfnst_idx > 0, dq->scalar_members, (const int32_t*) rates,
                                                    coef + i * area, 1, q + i * area, &s, &l )
                            : orc_dep_quant( par->w, par->h, par->bit_depth, par->qp, dq->lambda, dq->dq_thr_val, dq->zero_out, par->lfnst_idx > 0, dq->scalar_members, (const int32_t*) rates,
                                             coef + i * area, 1, q + i * area, &s, &l ) ) return fail( c, VVB_ERR_UNSUPPORTED, "TU shape" );
    if( abs_sum ) abs_sum[i] = s;
    if( last_pos ) last_pos[i] = l;
  }
  c->calls++;
  return VVB_OK;
}

int vvb_rdoq( vvb_ctx* c, const vvb_tu_par* par, const vvb_rdoq_par* rq, const vvb_rdoq_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n,
              int16_t* q, int32_t* abs_sum, int32_t* last_pos )
{
  if( !c ) return VVB_ERR_ARG;
  if( !par || !rq || !rates || !coef || !q || n < 0 || !( rq->lambda > 0.0 ) ) return fail( c, VVB_ERR_ARG, "bad RDOQ arguments" );
  if( par->transform_skip ) return fail( c, VVB_ERR_UNSUPPORTED, "transform-skipped TUs go through vvb_rdoq_ts" );
  const size_t area = (size_t) par->w * par->h;
  for( int i = 0; i < n; i++ )
  {
    int32_t s = 0, l = -1;
    if( need_rdoq && !need_rdoq[i] ) memset( q + i * area, 0, sizeof( int16_t ) * area );
    else if( orc_rdoq( par->w, par->h, par->bit_depth, par->qp, par->is_chroma, par->lfnst_idx > 0, rq->sbt_zero_out, par->sign_hiding, rq->lambda, rq->thr_val, (const int32_t*) rates,
                       coef + i * area, 1, q + i * area, &s, &l ) ) return fail( c, VVB_ERR_UNSUPPORTED, "TU shape" );
    if( abs_sum ) abs_sum[i] = s;
    if( last_pos ) last_pos[i] = l;
  }
  c->calls++;
  return VVB_OK;
}

int vvb_rdoq_ts( vvb_ctx* c, const vvb_tu_par* par, double lambda, const vvb_rdoq_ts_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n, int16_t* q, int32_t* abs_sum )
{
  if( !c ) return VVB_ERR_ARG;
  if( !par || !rates || !coef || !q || n < 0 || !( lambda > 0.0 ) ) return fail( c, VVB_ERR_ARG, "bad transform-skip RDOQ arguments" );
  const size_t area = (size_t) par->w * par->h;
  for( int i = 0; i < n; i++ )
  {
    int32_t s = 0;
    if( need_rdoq && !need_rdoq[i] ) memset( q + i * area, 0, sizeof( int16_t ) * area );
    else if( orc_rdoq_ts( par->w, par->h, par->bit_depth, par->qp, par->input_bit_depth_delta, lambda, (const int32_t*) rates, coef + i * area, 1, q + i * area, &s ) )
      return fail( c, VVB_ERR_UNSUPPORTED, "TU shape" );
    if( abs_sum ) abs_sum[i] = s;
  }
  c->calls++;
  return VVB_OK;
}

int vvb_rdoq_bdpcm( vvb_ctx* c, const vvb_tu_par* par, double lambda, int dir_mode, const vvb_rdoq_ts_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n, int16_t* q, int32_t* abs_sum )
{
  if( !c ) return VVB_ERR_ARG;
  if( !par || !rates || !coef || !q || n < 0 || !( lambda > 0.0 ) || dir_mode < 1 || dir_mode > 2 ) return fail( c, VVB_ERR_ARG, "bad BDPCM RDOQ arguments" );
  const size_t area = (size_t) par->w * par->h;
  for( int i = 0; i < n; i++ )
  {
    int32_t s = 0;
    if( need_rdoq && !need_rdoq[i] ) memset( q + i * area, 0, sizeof( int16_t ) * area );
    else if( orc_rdoq_bdpcm( par->w, par->h, par->bit_depth, par->qp, par->input_bit_depth_delta, dir_mode, lambda, (const int32_t*) rates, coef + i * area, 1, q + i * area, &s ) )
      return fail( c, VVB_ERR_UNSUPPORTED, "TU shape" );
    if( abs_sum ) abs_sum[i] = s;
  }
  c->calls++;
  return VVB_OK;
}

int vvb_set_rdoq_engine( vvb_ctx* c, int engine ) { if( !c || engine < 1 || engine > 2 ) return VVB_ERR_ARG; return VVB_OK; }   /* kernel choice of the real library: nothing to do here */
