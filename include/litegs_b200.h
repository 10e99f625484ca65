/*
 * litegs_b200.h -- C ABI of liblitegs_b200.so, the H100-native (sm_90a) replacement for the hot path of
 * MooreThreads/LiteGS' `litegs_fused` extension (reference: litegs/submodules/gaussian_raster/, "GR/").
 *
 * The reference binds this path through a pybind11 module on at::Tensor (GR/ext_cuda.cpp:9-35); its
 * 26 entry points are the interface a maintainer re-binds.  Here every entry point is a plain C
 * function on raw DEVICE pointers, sizes and a CUDA stream handle -- no torch types -- and the
 * host-side mirror of the pybind surface (litegs_b200/fused.py, same names, same positional
 * arguments, same return lists) sits above it.  INTEGRATION.md shows the binding stubs.
 *
 * Conventions
 *   - all pointers are device pointers unless a comment says otherwise; layouts are the reference's
 *     SoA with the point index innermost: [C,N], [V,C,N]; matrices are row-vector style [V,4,4];
 *   - `valid_length` is a nullable DEVICE int[1]: entries with index >= *valid_length are not computed
 *     (GPU-driven pipeline, no host sync), exactly as in the reference;
 *   - `stream` is a cudaStream_t passed as void*; every launch goes to it (the reference launches on
 *     the legacy default stream, SURVEY Q10);
 *   - return value: 0 on success, otherwise a cudaError_t value or one of LGS_ERR_*; the message is
 *     available from lgs_last_error() (thread-local).  Launches are checked.
 *   - tile sizes: 8x16 (reference default), 12x16, 16x16, 8x8 (GR/raster.cu:375-383).
 */
#ifndef LITEGS_B200_H
#define LITEGS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LGS_ERR_ARG 10001
#define LGS_ERR_WORKSPACE 10002
#define LGS_REC_FLOATS 12  /* floats per packed splat record  (px py A B | C o r g | b depth - -) */
#define LGS_GRAD_FLOATS 12 /* floats per gradient accumulator: raw moments of dL/dpower over the splat's pixels
                              (sum dx*s0, sum s1, sum dx^2*s0, sum dx*s1 | sum s2, dr, dg, db | sum s0, err_sq, -, -);
                              the consumers (unpack inside lgs_rasterize_backward, lgs_project_backward) apply the conic */

const char* lgs_last_error(void);
int lgs_abi_version(void);

/* ---- chunk culling + activation ------------------------------------------------------------------ */

/* replaces frustum_culling_aabb, GR/compact.cu:419-551 (GR/compact.h:28).
 * aabb_origin/aabb_ext f32[3,M]; frustumplane f32[V,6,4]; visibility u8[M]; visible_num i32[1];
 * visible_chunk_id i64[M] receives the visible chunk ids in ASCENDING order (first *visible_num valid). */
int lgs_frustum_culling_aabb(const float* aabb_origin, const float* aabb_ext, const float* frustumplane, int M, int V,
                             uint8_t* visibility, int* visible_num, int64_t* visible_chunk_id, void* stream);

/* replaces cull_compact_activate, GR/compact.cu:825-893,983-1085 (GR/compact.h:3-8).
 * params [..,C,S] (C chunks of S points); outputs [..,A,S] with A = allocated chunks:
 * act_position f32[4,A,S] (w=1), act_scale f32[3,A,S]=exp, act_rotation f32[4,A,S] normalised,
 * color f32[V,3,A,S] = SH(deg)+0.5 (no clamp, SURVEY Q13), act_opacity f32[1,A,S]=sigmoid, 0 for chunks
 * >= *visible_chunks_num. */
int lgs_cull_compact_activate(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                              const float* view_matrix, int V, const float* position, const float* scale,
                              const float* rotation, const float* sh_base, const float* sh_rest, const float* opacity,
                              int C, int S, int A, float* act_position, float* act_scale, float* act_rotation,
                              float* color, float* act_opacity, void* stream);

/* replaces activate_backward, GR/compact.cu:895-980,1087-1212 (GR/compact.h:10-16).
 * true_sigmoid_grad = 0 reproduces the reference's opacity-logit gradient d_o*sigma(x)
 * (GR/compact.cu:952, SURVEY Q15); 1 gives sigma(1-sigma).  Outputs are compacted [..,A,S];
 * g_sh_rest f32[rest_dim,3,A,S] is zeroed first. */
int lgs_activate_backward(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                          const float* view_matrix, int V, const float* position, const float* scale,
                          const float* rotation, const float* opacity, int C, int S, int A, int rest_dim,
                          int true_sigmoid_grad, const float* g_act_position, const float* g_act_scale,
                          const float* g_act_rotation, const float* g_color, const float* g_act_opacity,
                          float* g_position, float* g_scale, float* g_rotation, float* g_sh_base, float* g_sh_rest,
                          float* g_opacity, void* stream);

/* ---- per-Gaussian projection operators ------------------------------------------------------------- */

/* mvp_transform_forward/backward, GR/transform.cu:378-598 (GR/transform.h:11-16). world f32[4,N] ->
 * view,ndc f32[V,4,N]; backward sums over views into f32[4,N]. */
int lgs_mvp_transform_forward(const float* world_position, const float* view_matrix, const float* proj_matrix,
                              const int* valid_length, int V, int N, float* view_position, float* ndc_position, void* stream);
int lgs_mvp_transform_backward(const float* grad_ndc_pos, const float* grad_view_pos, const float* view_matrix,
                               const float* proj_matrix, const float* view_pos, const int* valid_length, int V, int N,
                               float* grad_world_pos, void* stream);

/* createTransformMatrix_forward/backward, GR/transform.cu:92-256 (GR/transform.h:5-6). quaternion f32[4,N]
 * (r,x,y,z), scale f32[3,N] -> T = diag(s) R(q) f32[3,3,N]. */
int lgs_create_transform_matrix_forward(const float* quaternion, const float* scale, const int* valid_length, int N,
                                        float* transform, void* stream);
int lgs_create_transform_matrix_backward(const float* transform_grad, const float* quaternion, const float* scale,
                                         const int* valid_length, int N, float* grad_quaternion, float* grad_scale,
                                         void* stream);

/* jacobianRayspace, GR/transform.cu:22-90 (GR/transform.h:3). view_pos f32[V,4,N] -> J f32[V,3,3,N]
 * (all nine rows written, five of them zero). */
int lgs_jacobian_rayspace(const float* view_pos, const float* proj_matrix, const int* valid_length, int V, int N,
                          int output_h, int output_w, float* jacobian, void* stream);

/* createCov2dDirectly_forward/backward, GR/transform.cu:736-927 (GR/transform.h:19-20). */
int lgs_create_cov2d_forward(const float* J, const float* view_matrix, const float* transform_matrix,
                             const int* valid_length, int V, int N, float* cov2d, void* stream);
int lgs_create_cov2d_backward(const float* cov2d_grad, const float* J, const float* view_matrix,
                              const float* transform_matrix, const int* valid_length, int V, int N,
                              float* transform_matrix_grad, void* stream);

/* eigh_and_inv_2x2matrix_forward / inv_2x2matrix_backward, GR/transform.cu:1364-1518 (GR/transform.h:25-26). */
int lgs_eigh_and_inv_2x2_forward(const float* input, const int* valid_length, int V, int N, float* val, float* vec,
                                 float* inv, void* stream);
int lgs_inv_2x2_backward(const float* inv_matrix, const float* grad_inv, const int* valid_length, int V, int N,
                         float* grad_matrix, void* stream);

/* sh2rgb_forward/backward, GR/transform.cu:951-1361 (GR/transform.h:22-23): cluster_size=0 path. */
int lgs_sh2rgb_forward(int degree, const float* sh_base, const float* sh_rest, const float* dirs, int V, int N,
                       float* rgb, void* stream);
int lgs_sh2rgb_backward(int degree, const float* rgb_grad, int sh_rest_dim, const float* dirs, int V, int N,
                        float* sh_base_grad, float* sh_rest_grad, float* dir_grad, void* stream);

/* ---- binning ----------------------------------------------------------------------------------------- */

/* get_allocate_size, GR/binning.cu:289-440 (GR/binning.h:11-15): visibility + exact ellipse/tile overlap
 * count (GR/speedy_splat.cuh:33-149). left_up/right_down i32[V,2,N], allocate_size i32[V,N] (zeroed).
 * The tile rectangle's last row / column follows lgs_set_exact_tile_bound. */
int lgs_get_allocate_size(const float* ndc, const float* view_space_z, const float* inv_cov2d, const float* opacity,
                          const int* valid_length, int V, int N, int height, int width, int tile_h, int tile_w,
                          int* left_up, int* right_down, int* allocate_size, void* stream);

/* create_table, GR/binning.cu:33-226 (GR/binning.h:5-9): emit (tile+1, splat) in depth order at `offset`
 * (inclusive scan, i32[V,N]) then a stable radix sort on the tile bits.  cap = table length; outputs
 * i32[V,cap].  The reference sizes the table from a pinned feedback buffer (GR/binning.cu:137-163);
 * that policy lives in the host mirror, the C entry point takes `cap` explicitly.
 * The counts in `offset` must have been made under the same lgs_set_exact_tile_bound setting. */
int lgs_create_table_workspace_bytes(int V, int cap, size_t* bytes);
int lgs_create_table(const float* ndc, const float* inv_cov2d, const float* opacity, const int* offset,
                     const int64_t* depth_sorted_pointid, int V, int N, int cap, int height, int width, int tile_h,
                     int tile_w, int* sorted_tile_id, int* sorted_point_id, void* workspace, size_t workspace_bytes,
                     void* stream);

/* Tile rectangle of lgs_get_allocate_size / lgs_create_table.  1 (default): it ends after the tile holding bbox_max,
 * floor((bbox_max + T) / T), so every tile holding a pixel centre where the splat's alpha reaches 1/255 is listed;
 * 0: the reference's floor((bbox_max + T - 1) / T) (GR/binning.cu:88-91), which drops a tile the ellipse reaches by less
 * than a pixel (DESIGN.md section 7, D14).  The fused pipeline always uses 1.  Process-wide, like lgs_set_staging. */
int lgs_set_exact_tile_bound(int on);

/* tileRange, GR/binning.cu:228-287 (GR/binning.h:10). tile_range i32[V,max_tile_id+2], -1 = empty.
 * fix_last=1 closes the last populated tile (the reference leaves it open: SURVEY Q3); 0 = bit-compatible. */
int lgs_tile_range(const int* table_tile_id, int V, int table_length, int max_tile_id, int fix_last, int* tile_range,
                   void* stream);

int lgs_tile_range_u16(const unsigned short* table_tile_id, int V, int table_length, int max_tile_id, int fix_last,
                       int* tile_range, void* stream);

/* building blocks of the fused pipeline, on the caller's stream and workspace.  Stable LSD radix sort of (key, value)
 * pairs on the bits [begin_bit, end_bit): replaces torch.sort (wrapper.py:739) for the depth order and
 * cub::DeviceRadixSort::SortPairs (GR/binning.cu:204-221) for the tile sort.  keys_in/vals_in are not modified.
 * lgs_set_sort_impl: 1 = own histogram/scan/scatter passes (default), 0 = cub::DeviceRadixSort; env LGS_SORT=lgs|cub.
 * Either value forces that sort for every later call; -1 returns to the unforced state of a fresh process (LGS_SORT is
 * read again, and without it the tile sort of more than 14 key bits on more than 8 << 20 pairs takes cub's onesweep). */
int lgs_set_sort_impl(int impl);
/* form of the own radix sort: 0 = histogram / row-scan / scatter passes (default), 1 = onesweep (global
 * histograms in one read + decoupled look-back per pass); env LGS_RS=passes|onesweep */
int lgs_set_radix_form(int onesweep);
int lgs_sort_pairs_u16_workspace_bytes(int n, size_t* bytes);
int lgs_sort_pairs_u16(const unsigned short* keys_in, unsigned short* keys_out, const unsigned* vals_in, unsigned* vals_out,
                       int n, int begin_bit, int end_bit, void* workspace, size_t workspace_bytes, void* stream);
int lgs_sort_pairs_u32_workspace_bytes(int n, size_t* bytes);
int lgs_sort_pairs_u32(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out, int n,
                       int begin_bit, int end_bit, void* workspace, size_t workspace_bytes, void* stream);
/* order by (key - bias) on bits [0, end_bit): the full-key order for keys inside [bias, bias + 2^end_bit), fewer passes */
int lgs_sort_pairs_u32_rebased(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out, int n,
                               unsigned bias, int end_bit, void* workspace, size_t workspace_bytes, void* stream);
int lgs_scan_gathered_workspace_bytes(int n, size_t* bytes);
int lgs_scan_gathered(const int* counts, const unsigned* order, int n, int* out, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ---- GPU-driven sizing: the same building blocks with the live counts read ON THE DEVICE -------------------------------
 * `capacity` bounds the launch geometry and the buffers; the live count comes from a device int (clamped to the capacity), the
 * depth-key bias from a device word.  Nothing is read back, so a whole view can be enqueued -- or captured in a CUDA graph --
 * without a host synchronisation.  The reference gets the same effect by sizing from LAST epoch's counts through pinned
 * feedback buffers (GR/compact.cu:527-549, GR/binning.cu:137-163, data.py:238); here the capacity is the caller's prediction
 * and lgs_view_params raises a device-side flag when it was too small. */
int lgs_view_params(const int* counters /* i32[4]: visible chunks, pairs, ~min depth key, max depth key */, int S, int pair_capacity,
                    int planned_depth_bits, int* params /* i32[8], see csrc/fused.cu */,
                    int* sticky /* nullable i32[4]: |= flags, max pairs, max depth bits, views -- accumulated over views */, void* stream);
int lgs_sort_pairs_u32_dev(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out, int capacity,
                           const int* n_dev, const unsigned* bias_dev, int end_bit, void* workspace, size_t workspace_bytes, void* stream);
int lgs_sort_pairs_u16_dev(const unsigned short* keys_in, unsigned short* keys_out, const unsigned* vals_in, unsigned* vals_out,
                           int capacity, const int* n_dev, int begin_bit, int end_bit, void* workspace, size_t workspace_bytes,
                           void* stream);
int lgs_sort_pairs_u32k_dev(const unsigned* keys_in, unsigned* keys_out, const unsigned* vals_in, unsigned* vals_out, int capacity,
                            const int* n_dev, int begin_bit, int end_bit, void* workspace, size_t workspace_bytes, void* stream);
int lgs_scan_gathered_dev(const int* counts, const unsigned* order, int capacity, const int* n_dev, int* out, void* workspace,
                          size_t workspace_bytes, void* stream);
int lgs_emit_pairs_dev(const float* packed_params, const int* offset, const unsigned* order, int n_capacity, const int* n_dev, int cap,
                       int img_h, int img_w, int tile_h, int tile_w, int key_bits /* 16 | 32 */, void* keys, int* vals,
                       int* valid_pairs /* nullable: lowered to the written length when runs were dropped */, void* stream);
int lgs_tile_range_u16_dev(const unsigned short* table_tile_id, int capacity, const int* length_dev, int max_tile_id, int fix_last,
                           int* tile_range, void* stream);
int lgs_tile_range_dev(const int* table_tile_id, int capacity, const int* length_dev, int max_tile_id, int fix_last, int* tile_range,
                       void* stream);

/* ---- rasterisation ------------------------------------------------------------------------------------- */

/* pack_forward_params, GR/raster.cu:334-356 -> packed f32[V,N,12] (fp32 record, see LGS_REC_FLOATS). */
int lgs_pack_params(const float* ndc, const float* cov2d_inv, const float* color, const float* opacity, int V, int N,
                    int img_h, int img_w, float* packed_params, void* stream);

/* rasterize_forward(_packed), GR/raster.cu:161-332,386-586 (GR/raster.h:3-32).  Images are padded to
 * whole tiles: img f32[V,3,Hp,Wp], transmittance f32[V,1,Hp,Wp], last_contributor i16[V,1,Hp,Wp];
 * fragment_count i32[V,1,N] / fragment_weight f32[V,1,N] are accumulated when enable_statistic (caller
 * zeroes them).  specific_tiles i32[V,n_specific] (1-based tile ids, 0 = skip) or NULL.  clamp_zero=0 writes
 * min(c,1) as the reference kernel does; 1 writes clamp(c,0,1), i.e. also the clamp render() applies in Python
 * (render/__init__.py:87) -- then pass the image back to lgs_rasterize_backward as `clamped_img`.
 * last_contributor holds an UNSIGNED 16-bit count (the reference reads it back as unsigned short, GR/raster.cu:683-686),
 * saturated at 65535.  tile_work i32[V,tiles] (nullable): per tile, the deepest list position any of its pixels consumed
 * = the backward's trip count, input of lgs_tile_order (zero it first when specific_tiles is given).
 * depth f32[V,1,Hp,Wp] or NULL, ours (the reference leaves its depth image zero): per pixel D = sum_i w_i z_i with the weights of
 * the colour and z_i the record's depth slot (the view-space z on the fused path), not clamped (DESIGN.md section 1, "Depth").
 * Only the default kernel renders depth: with bulk staging or the pixel-pair forward selected, a non-NULL depth is refused.
 * NULL = no depth, the same kernels as before.
 * normal_rec f32[V,N,4] (lgs_project_forward's side rows, aligned with packed_params) and normal f32[V,3,Hp,Wp], both given or
 * both NULL, ours (DESIGN.md section 1, "Normals"): per pixel N = sum_i w_i n_i with the weights of the colour, neither clamped
 * nor normalised.  Like depth, only the default kernel renders it: with bulk staging or the pixel-pair forward selected, a
 * non-NULL normal is refused.  NULL = no normal, the same kernels as before. */
int lgs_rasterize_forward_packed(const int* sorted_points, const int* start_index, const float* packed_params,
                                 const int* specific_tiles, int n_specific, int V, int N, int cap, int img_h, int img_w,
                                 int tile_h, int tile_w, int enable_statistic, int clamp_zero, float* img,
                                 float* transmittance, short* last_contributor, int* fragment_count,
                                 float* fragment_weight, int* tile_work, float* depth, const float* normal_rec, float* normal,
                                 void* stream);

/* order i32[V,tiles] = 1-based tile ids by descending work (heaviest lists first), to be passed as specific_tiles:
 * the device-side form of the reference's tile scheduling by last epoch's blend count (render/__init__.py:75-79,
 * utils/statistic_helper.py:68-79). */
int lgs_tile_order(const int* work, int V, int ntile, int* order, void* stream);

/* rasterize_backward, GR/raster.cu:599-886,917-1037 (GR/raster.h:34-50).  packed_grad f32[V,N,12] is
 * scratch (zeroed here); d_trans_img, clamped_img (the forward's clamp_zero=1 output: blocks the gradient where a
 * colour was clamped up to 0) and grad_inv_scaler (DEVICE f32[1]) may be NULL.  Outputs d_ndc
 * f32[V,4,N], d_cov2d_inv f32[V,2,2,N], d_color f32[V,3,N], d_opacity f32[1,N] (view 0 only, as the
 * reference), err_sum/err_square_sum f32[V,1,N].  Pass d_ndc=NULL to skip the unpack (fused path).
 * d_depth f32[V,1,Hp,Wp] or NULL, ours: dL/dD of the forward's depth image.  It joins the alpha gradient as one more colour
 * channel with colour z, and packed_grad slot 10 receives sum_pixels w g_z = dL/dz (consumed by lgs_project_backward with depth
 * = 1; the unpack ignores it).  Only the pixel-pair kernel (the default, and the deterministic mode) takes it: with the scalar
 * kernel or bulk staging selected, a non-NULL d_depth is refused.  NULL = no depth gradient, the same kernels as before.
 * normal_rec f32[V,N,4] (the forward's side rows), d_normal f32[V,3,Hp,Wp] = dL/dN and grad_normal f32[V,N,4] (zeroed here), all
 * given or all NULL, ours: dL/dN joins the alpha gradient as three more colour channels with colour n (after the depth term), and
 * grad_normal receives sum_pixels w g_N = dL/dn (consumed by lgs_project_backward).  Pixel-pair kernel and deterministic mode
 * only, as d_depth.  NULL = no normal gradient, the same kernels as before. */
int lgs_rasterize_backward(const int* sorted_points, const int* start_index, const float* packed_params,
                           const int* specific_tiles, int n_specific, const float* final_transmittance,
                           const short* last_contributor, const float* d_img, const float* d_trans_img,
                           const float* clamped_img, const float* grad_inv_scaler, int V, int N, int cap, int img_h, int img_w, int tile_h,
                           int tile_w, int enable_statistic, float* packed_grad, float* d_ndc, float* d_cov2d_inv,
                           float* d_color, float* d_opacity, float* err_sum, float* err_square_sum, const float* d_depth,
                           const float* normal_rec, const float* d_normal, float* grad_normal, void* stream);

/* staging selector for the raster kernels: 0 = cp.async / LDGSTS (default), 1 = cp.async.bulk + mbarrier */
int lgs_set_staging(int bulk);
/* warp reduction of the per-(tile,splat) gradient in the backward: 1 = deferred through shared memory (default),
 * 0 = register butterfly */
int lgs_set_backward_reduce(int deferred);
/* tiles (warps) per CTA of the raster kernels: 1, 2 or 4 (default 4, env LGS_WPB) */
int lgs_set_warps_per_block(int wpb);
/* forward blend on pixel pairs (two scalar chains side by side): 1 on, 0 = scalar predicated body.  env LGS_FWD_PAIRS=0|1 */
int lgs_set_forward_pairs(int on);
/* backward kernel: 2 = pixel pairs, branch-free pixel body (default); 1 = scalar kernel.  env LGS_BWD=v1|v2 */
int lgs_set_backward_kernel(int version);
/* 1 = deterministic backward: per-(tile, splat) sums accumulated as fixed point, two 64-bit words per value (range 3.6e16,
 * resolution 3.6e-15), with integer atomics (associative, so two runs give bit-identical gradients; scratch from the
 * stream-ordered allocator); 0 = fp32 RED atomics (default, faster).
 * env LGS_DETERMINISTIC=1 */
int lgs_set_deterministic(int on);
/* err_square_sum under enable_statistic: 1 = the reference's lane-running recurrence (GR/raster.cu:779-784, default),
 * 0 = sum over pixels of (G dalpha)^2 */
int lgs_set_err_square_mode(int mode);

/* ---- fused per-view pipeline ("Level B") ---------------------------------------------------------------- */

/* One kernel for the whole projection chain of one view: replaces cull_compact_activate + mvp_transform_forward +
 * createTransformMatrix_forward + jacobianRayspace + createCov2dDirectly_forward + eigh_and_inv_2x2matrix_forward +
 * get_allocate_size + pack_forward_params (render/__init__.py:26-61, wrapper.py:727-731, GR/raster.cu:334-356).
 * A = number of allocated chunks (launch width; chunks >= *visible_chunks_num produce invisible records).
 * Outputs over A*S compacted slots: packed_params f32[A*S,12] (slots 10,11 carry ndc.x, ndc.y for the emit pass),
 * depth_key u32 (float bits of view z, 0xFFFFFFFF when invisible), iota u32 (slot index), tile_count i32,
 * totals i32[3] = { number of (tile,splat) pairs, ~min and max of the depth keys of the splats that have pairs }
 * (so the depth sort can be limited to the bits in which those keys differ; splats without pairs may land anywhere
 * in the order, they emit nothing).
 * antialiased != 0: antialiased mode, ours (the reference has none).  The record's opacity is sigmoid(opacity) * rho with
 * rho = sqrt(det(M^T M) / det(M^T M + 0.3 I)), the opacity compensation of the 2D low-pass filter (DESIGN.md section 1);
 * the visibility test, the tile walk and the rasteriser all see that opacity.  0 = the reference's behaviour.
 * filter_3d f32[C*S] (clustered like opacity) or NULL: Mip-Splatting's 3D smoothing filter, ours (the reference has none).  Each
 * Gaussian's activated scale becomes s' = sqrt(s^2 + f^2) in the whole chain (S.R, M, the 2D covariance, the tile walk) and its
 * opacity sigmoid(opacity) * rho3 with rho3 = sqrt(prod_k s_k^2 / (s_k^2 + f^2)), before the antialiased factor
 * (DESIGN.md section 1, "3D smoothing filter").  NULL = no filter, the same kernels as before.
 * normal_rec f32[A*S,4] or NULL, ours (DESIGN.md section 1, "Normals"): receives (n0, n1, n2, 0) per slot, the view-space normal
 * of the Gaussian's shortest axis (argmin of the raw log-scales), turned to face the camera; slots of chunks at or past the
 * visible count get zeros.  NULL = no normals, the same kernels as before. */
int lgs_project_forward(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                        const float* view_matrix, const float* proj_matrix, const float* position, const float* scale,
                        const float* rotation, const float* sh_base, const float* sh_rest, const float* opacity, int C,
                        int S, int A, int img_h, int img_w, int tile_h, int tile_w, float* packed_params,
                        unsigned* depth_key, unsigned* iota, int* tile_count, int* totals, const float* filter_3d, int antialiased,
                        float* normal_rec, void* stream);

/* duplicate_with_keys (GR/binning.cu:33-110) reading the packed record: offset = inclusive scan of the depth-ordered
 * counts, order = depth-sorted slot ids; keys/vals i32[cap] must be zero-initialised by the caller. */
int lgs_emit_pairs(const float* packed_params, const int* offset, const unsigned* order, int n, int cap, int img_h,
                   int img_w, int tile_h, int tile_w, int* keys, int* vals, void* stream);
/* same with 16-bit tile keys (tiles + 1 < 65536): 25 % fewer bytes through emit, the tile sort and tile_range */
int lgs_emit_pairs_u16(const float* packed_params, const int* offset, const unsigned* order, int n, int cap, int img_h,
                       int img_w, int tile_h, int tile_w, unsigned short* keys, int* vals, void* stream);

/* Record gradient (packed_grad f32[A*S,12] from lgs_rasterize_backward) -> the six compacted parameter gradients;
 * replaces unpack_gradient + inv_2x2matrix_backward(+nan_to_num) + createCov2dDirectly_backward +
 * createTransformMatrix_backward + mvp_transform_backward + activate_backward (wrapper.py:481-524,588-592,404-407,
 * 190-193,278-285,820-845).  zero_outputs: 0 = assign compacted [..,A,S] outputs, 1 = clear them first,
 * 2 = ACCUMULATE into dense [..,C,S] gradient tensors at the source chunk (multi-view / data-parallel path).
 * touched (f32[C], may be NULL) receives 1 at every visible chunk: the marks lgs_adam_step_dense consumes.
 * cam_partials (f32[A,32]) and d_cam (f32[32]), both NULL or both given: d_cam receives the gradient of the view matrix
 * (d_cam[0..15], row-vector [k*4+j]) and of the projection matrix (d_cam[16..31]) through the NDC mean and the V3x3 factor of
 * the 2D covariance, with J and the SH direction held constant (the convention of the position gradient, DESIGN.md section 1).
 * The reference's operators return no view-matrix gradient (wrapper.py:285,407,845); this one is new.  Summed in a fixed
 * order (bit-reproducible), no host synchronisation; needs S % 32 == 0.
 * antialiased: must equal the value the forward of this view was given (ours, no reference counterpart).  The record
 * gradient is then taken at the compensated opacity and the gradient of rho flows into scale, rotation and the camera.
 * filter_3d: the tensor the forward of this view was given, or NULL.  The filter is held constant: the raw scale gradient
 * gains the rho3 term, and no gradient flows into the filter, the positions or the cameras through it.
 * exact_grad != 0: exact gradient mode, ours (the reference drops both terms).  g_position, and d_cam when given, also
 * receive the terms through the ray-space Jacobian J (its dependence on the view-space position and on proj[0][0],
 * proj[1][1]) and through the SH view direction (its dependence on the position and on the camera centre) (DESIGN.md
 * section 1, "Exact gradient mode").  The other five gradients are unchanged.  sh_base, sh_rest: the coefficients the forward
 * was given.  sh_base is not read (the constant band has no direction term; it may be NULL).  sh_rest is read only when
 * exact_grad != 0 and sh_degree > 0 (its rows of the active degree) and must be non-NULL then; at degree 0 it may be NULL, as
 * an empty tensor's pointer is.  With exact_grad != 0 the chunk size S is limited by the register use of the instantiation
 * (384 for the heaviest; a larger S is refused with an error naming the limit).  0 = the kernels without the terms.
 * depth != 0: depth mode, ours.  packed_grad slot 10 (dL/dz from lgs_rasterize_backward's d_depth) is added to the view-space
 * z gradient: it reaches g_position through the view matrix and d_cam as d view[k][2] += p~_k dz; d proj gets nothing from it.
 * It is exact in both gradient conventions (z depends on neither J nor the SH direction).  0 = slot 10 is not read.
 * grad_normal f32[A*S,4] (lgs_rasterize_backward's) or NULL, ours: with dn_c = sigma dn and dn_w = V3x3 dn_c, dn_w is added to
 * row a (the shortest axis) of the rotation-matrix gradient, so it reaches g_rotation; d_cam gains d view[k][j] += n_w[k] dn_c[j]
 * for k, j < 3.  Nothing reaches g_position, g_scale or d proj; a and the facing sign sigma are held constant.  The same in both
 * gradient conventions.  NULL = no normal term, the same kernels as before. */
int lgs_project_backward(int sh_degree, const int64_t* visible_chunk_id, const int* visible_chunks_num,
                         const float* view_matrix, const float* proj_matrix, const float* position, const float* scale,
                         const float* rotation, const float* opacity, int C, int S, int A, int rest_dim, int img_h,
                         int img_w, int true_sigmoid_grad, const float* packed_grad, const float* grad_inv_scaler,
                         int zero_outputs, float* g_position, float* g_scale, float* g_rotation, float* g_sh_base,
                         float* g_sh_rest, float* g_opacity, float* touched, float* cam_partials, float* d_cam,
                         const float* filter_3d, int antialiased, const float* sh_base, const float* sh_rest, int exact_grad,
                         int depth, const float* grad_normal, void* stream);

/* create_viewproj_forward, GR/compact.cu:17-141: view_params f32[V,7] (qw qx qy qz tx ty tz), recp_tan_half_fov_x f32[1] ->
 * view, proj, viewproj f32[V,4,4] (row-vector convention) and frustumplane f32[V,6,4].  One thread per view. */
int lgs_create_viewproj_forward(const float* view_params, const float* recp_tan_half_fov_x, int V, int img_h, int img_w,
                                float z_near, float z_far, float* view_matrix, float* proj_matrix, float* viewproj_matrix,
                                float* frustumplane, void* stream);
/* create_viewproj_backward, GR/compact.cu:143-316, with the reference's arithmetic (DESIGN.md section 7): the fov gradient scales
 * d proj[1][1] by the integer quotient img_w / img_h, and the quaternion gradient is the true one times |q|.  grad_recp f32[1] is
 * the sum over views in a fixed order (the reference's is a race for V > 1).  Outputs are assigned, not accumulated. */
int lgs_create_viewproj_backward(const float* view_matrix_grad, const float* proj_matrix_grad, const float* viewproj_matrix_grad,
                                 const float* view_params, const float* recp_tan_half_fov_x, int V, int img_h, int img_w,
                                 float z_near, float z_far, float* grad_view_params, float* grad_recp_tan_half_fov_x, void* stream);

/* ---- optimiser / statistics (next rows, SURVEY 8f) ------------------------------------------------------ */

/* adamUpdate, GR/compact.cu:320-417 (GR/compact.h:18-23): Adam WITHOUT bias correction. */
int lgs_adam_update_chunk(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                          const int64_t* visible_index, const int* valid_length, int R, int C, int S, int A, double lr,
                          double b1, double b2, double eps, void* stream);
int lgs_adam_update_primitive(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                              const int64_t* primitive_visible, int R, int N, double lr, double b1, double b2,
                              double eps, void* stream);

/* The optimizer step of the multi-view / data-parallel path: ONE launch for all six parameter tensors, from the dense
 * gradient buffer grad f32[rows, C, S] (rows = sum rows_per_param, parameter k occupies its rows in the order xyz,
 * scale, rot, sh_0, sh_rest, opacity) and moment buffers of the same shape.  Replaces the six adamUpdate calls of
 * optimizer.py:14-44 with the same arithmetic (GR/compact.cu:320-344, no bias correction).  params, rows_per_param,
 * lr_per_param are HOST arrays of 6.  touched f32[C] (may be NULL = all chunks): only chunks with touched != 0 update;
 * lgs_mark_visible_chunks sets it from a view's visible-chunk list.  clear_grad: also zero the consumed gradient
 * rows and marks (so the buffer needs no memset between steps). */
int lgs_mark_visible_chunks(const int64_t* visible_chunk_id, const int* visible_chunks_num, int A, float* touched, void* stream);
int lgs_adam_step_dense(float* const* params, const int* rows_per_param, const float* lr_per_param, float* grad,
                        float* exp_avg, float* exp_avg_sq, float* touched, int C, int S, double b1, double b2, double eps,
                        int clear_grad, void* stream);

/* gpu_driven_pipeline_sparse_op, GR/compact.cu:1221-1336 (GR/compact.h:30-36).  dtype 0=f32 1=i32 2=f64 3=i64 4=i16 5=i8 6=u8
 * (the reference dispatches AT_DISPATCH_ALL_TYPES, :1305); op 0=add 1=min 2=max */
int lgs_sparse_chunk_op(void* A, const void* B, const int64_t* visible_chunk_ids, const int* visible_count, int dtype,
                        int op, int ele_num, int chunks, int alloc_chunks, int chunk_size, void* stream);

/* ---- multi-GPU exchange (SURVEY 8e; new: the reference is single-GPU) ---------------------------------------------------------
 * The per-step all-reduce of the dense gradient buffer as one kernel over the buffer's NVSwitch MULTICAST address
 * (multimem.ld_reduce / multimem.st, reduction inside the switch).  multicast_ptr: multicast mapping of a symmetric allocation of
 * n_floats floats (multiple of 4) present on every rank; the caller puts a cross-GPU barrier on the stream before and after.
 * ctas = 0 selects the default grid. */
int lgs_nvls_allreduce_f32(float* multicast_ptr, size_t n_floats, int rank, int world, int ctas, void* stream);

/* ---- chunk maintenance between epochs (SURVEY 8f rank 4) ----------------------------------------------------------------- */

/* Morton codes of _gen_morton_code (litegs/scene/point.py:38-81): xyz f32[3,N], lo3/hi3 DEVICE f32[3] (per-axis min / max),
 * bits per axis (the reference uses 21) -> codes i64[N].  spatial_refine (point.py:85-154) = stable sort of these codes. */
int lgs_morton_codes(const float* xyz, const float* lo3, const float* hi3, int N, int bits, long long* codes, void* stream);
/* dst[r, j] = src[r, idx[j]], all R rows of a [R,N] matrix in one launch (parameters / gradients / Adam moments reordered
 * by the sorted Morton order, point.py:104-140). */
int lgs_permute_rows(const float* src, const long long* idx, int R, int N, float* dst, void* stream);
/* get_cluster_AABB (litegs/scene/cluster.py:29-46) from the RAW clustered parameters xyz/scale f32[3,C,S], rot f32[4,C,S]
 * -> origin, extend f32[3,C]. */
int lgs_cluster_aabb(const float* xyz, const float* scale, const float* rot, int C, int S, float* origin, float* extend, void* stream);
/* Mip-Splatting's 3D smoothing filter (compute_3D_filter), ours: position f32[3,C,S] (every slot, the tail padding included),
 * V cameras view / proj f32[V,4,4] (row-vector convention) and hw i32[V,2] (height, width) -> filter_3d f32[C*S].  Per Gaussian,
 * f = (dist / focal) * sqrt(0.2), dist = the smallest view depth over the cameras that see it (depth > 0.2, projection within
 * 15 % of the image border), focal = the largest P[0][0] W / 2.  Unseen Gaussians get the largest seen f (0 when none is seen).
 * Exact fp32 operation order in DESIGN.md section 1; bit-reproducible, no host synchronisation, no gradient. */
int lgs_filter_3d(const float* position, int C, int S, const float* view, const float* proj, const int* hw, int V,
                  float* filter_3d, void* stream);

/* ---- fused SSIM / L1 + SSIM loss (next row, SURVEY 8f rank 2; what trainer.py:145 calls) ------------------ */

/* fusedssim / fusedl1ssim_loss, fused_ssim/ssim.cu:444-479, 855-900 (kernels :64-274, :528-712).  img1, img2 f32[B,CH,H,W]
 * on the device.  l1_mode 0: map = SSIM;  1: map = w (1 - SSIM) + (1 - w) |img1 - img2|.  11-tap sigma-1.5 Gaussian,
 * zero padding ("same").  Outputs, each optional: map f32[B,CH,H,W]; the three partials dm_dmu1, dm_dsigma1_sq,
 * dm_dsigma12 (all or none; NULL = the reference's train=false); block_sums f32[count of lgs_ssim_num_block_sums] = the sum
 * of the map over each CTA's tile (the training path needs only the mean of the map: sum these in order). */
int lgs_ssim_num_block_sums(int B, int CH, int H, int W, int* count);
int lgs_ssim_forward(const float* img1, const float* img2, int B, int CH, int H, int W, float C1, float C2, int l1_mode,
                     float ssim_weight, float* map, float* dm_dmu1, float* dm_dsigma1_sq, float* dm_dsigma12,
                     float* block_sums, void* stream);
/* fusedssim_backward / fusedl1ssim_loss_backward, fused_ssim/ssim.cu:487-524, 904-942 (kernels :277-437, :719-850):
 * dL/dimg1 from dL/dmap and the saved partials.  dL_dmap NULL = the uniform value uniform_chain (loss = mean(map)). */
int lgs_ssim_backward(const float* img1, const float* img2, const float* dL_dmap, float uniform_chain, const float* dm_dmu1,
                      const float* dm_dsigma1_sq, const float* dm_dsigma12, int B, int CH, int H, int W, int l1_mode,
                      float ssim_weight, float* dL_dimg1, void* stream);

/* ---- depth-normal consistency (ours) --------------------------------------------------------------------------------- */

/* Depth-normal consistency of one view, ours (DESIGN.md section 1, "Depth-normal consistency"; 2DGS, PGSR, RaDe-GS).  Inputs on
 * the device: the depth mode's D and the transmittance T, f32[H,W] planes with row strides depth_row_stride, trans_row_stride
 * (elements); the normal mode's N, three f32[H,W] planes with the given row and channel strides (nullable when neither the
 * loss nor the gradient is asked for); proj f32[4,4] (row-vector), of which P[0][0] and P[1][1] are read on the device.
 * With alpha = 1 - T, ED = D / alpha, fx = P[0][0] W / 2, fy = P[1][1] H / 2 and r(u,v) = ((u + 0.5 - W/2) / fx,
 * (v + 0.5 - H/2) / fy, 1), X = ED r: at pixel p, a = X(u+1,v) - X(u-1,v), b = X(u,v+1) - X(u,v-1), n_d = (b x a) / |b x a|,
 * defined where p is at least one pixel from the border, alpha > alpha_min at p and its four neighbours, and |b x a| > 0.
 * There, with |N_p| > 1e-6 as well, l_p = 1 - n_d . N_p / |N_p|.  Outputs, contiguous, each optional:
 *   n_d f32[3,H,W] (zero where n_d is undefined);
 *   d_depth, d_trans f32[H,W] and d_normal f32[3,H,W], all or none: grad_scale * d(sum_p l_p) / d(D, T, N), the masks held constant
 *     (grad_scale = weight * upstream / (H W) gives the gradient of L = weight * mean_p l_p);
 *   block_sums f32[count of lgs_depth_normal_num_block_sums] = sum of l_p over each CTA's tile (sum them in order).
 * alpha_min in [0, 1).  One kernel, no atomics (bit-reproducible), no host synchronisation. */
int lgs_depth_normal_num_block_sums(int H, int W, int* count);
int lgs_depth_normal(const float* depth, int depth_row_stride, const float* trans, int trans_row_stride, const float* normal,
                     int normal_row_stride, int normal_channel_stride, const float* proj, int H, int W, float alpha_min, float grad_scale,
                     float* n_d, float* d_depth, float* d_trans, float* d_normal, float* block_sums, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* LITEGS_B200_H */
