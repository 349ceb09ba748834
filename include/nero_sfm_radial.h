/* libnero_b200 -- C ABI of bundle adjustment with SIMPLE_RADIAL cameras: the radial counterparts of the filter and the
 * Levenberg-Marquardt entry points of include/nero_sfm.h, with the lens's k estimated beside the focal.
 *
 * Same library and conventions as include/nero_sfm.h (DEVICE pointers, `stream` a cudaStream_t passed as void*, no
 * allocation or host synchronisation inside, 0 / 1 bad argument / 2 launch error, fp64, no floating-point atomics, every
 * sum in a fixed order).  The kernels are the ones of nero_sfm.h instantiated for two camera parameters.  The protocol is
 * stated in nero_b200/sfm.py and restated in numpy by oracle/nero_oracle_sfm_radial.py.
 *
 * Model (include/nero_undistort.h): a camera has a focal f, a principal point (cx, cy) and radial[c] = k.  Y = R X + t,
 * x = Y_x / Y_z, y = Y_y / Y_z, r2 = x^2 + y^2, d = 1 + k r2, u = (f x) d + cx, v = (f y) d + cy.  Every residual and
 * reprojection error is measured in this distorted image, where the keypoints are.
 *
 * Jacobian.  du/dx = f (d + 2 k x^2), du/dy = dv/dx = 2 f k x y, dv/dy = f (d + 2 k y^2); d(x, y)/dY = (1 / Y_z)
 * [[1, 0, -x], [0, 1, -y]]; du/df = x d, du/dk = f x r2, dv/df = y d, dv/dk = f y r2.  dY/dw = -[R X]x, dY/dt = I,
 * dY/dX = R as in nero_sfm.h.
 *
 * Layout.  Per observation the 8 camera-side columns are (w, t, f, k): Jc [n, 2, 8], Y [n, 8, 3].  The reduced system has
 * 6 nimg + 2 ncam columns: image k's (w, t) at 6 k .. 6 k + 5, camera c's f at 6 nimg + 2 c and its k at 6 nimg + 2 c + 1.
 * Block nimg + c of the (o, o') and right-hand-side lists is camera c's two columns; the 36-slot partials hold any pair
 * of blocks.
 */
#ifndef NERO_SFM_RADIAL_H_
#define NERO_SFM_RADIAL_H_

#ifdef __cplusplus
extern "C" {
#endif

/* nero_sfm_filter through the distortion: per observation (depth, reprojection error px) in err [n, 2], per point the
 * largest pairwise ray angle (radians) in angle [P]. */
int nero_sfm_radial_filter(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                           const double* focal, const double* pp, const double* radial, const double* X, double* err, double* angle,
                           void* stream);

/* Per observation: res [n, 2] (distorted projection - observation), Jc [n, 2, 8] (w, t, f, k) and Jp [n, 2, 3]. */
int nero_sfm_radial_ba_linearize(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose,
                                 const int* img_cam, const double* focal, const double* pp, const double* radial, const double* X,
                                 double* res, double* Jc, double* Jp, void* stream);

/* nero_sfm_ba_points on 8-column Jc: Vinv [P, 9], gp [P, 3], Y [n, 8, 3]. */
int nero_sfm_radial_ba_points(const long long* pt_off, int P, const double* res, const double* Jc, const double* Jp, double lambda,
                              int fix_points, double* Vinv, double* gp, double* Y, void* stream);

/* nero_sfm_ba_reduce with 2-column camera blocks: S [ncol, ncol] and b [ncol], ncol = 6 nimg + 2 ncam. */
int nero_sfm_radial_ba_reduce(const int* ent, const long long* chunk, const int* chunk_key, int nchunk, const long long* seg_chunk,
                              const int* seg_key, int nseg, const int* obs_seg, const long long* rchunk, const int* rchunk_blk, int nrchunk,
                              const long long* rseg_chunk, const int* rseg_blk, int nrseg, const int* obs_pt, const int* img_cam, int nimg,
                              int ncam, const double* Jc, const double* Jp, const double* res, const double* Y, const double* gp,
                              double lambda, const unsigned char* fixed, double* partial, double* rpartial, double* S, double* b,
                              void* stream);

/* nero_sfm_ba_backsub with the 8 camera-side columns; also radial_new = k + dk from dc [6 nimg + 2 c + 1]. */
int nero_sfm_radial_ba_backsub(const long long* pt_off, int P, const int* obs_img, const int* img_cam, int nimg, int ncam, const double* Jc,
                               const double* Jp, const double* Vinv, const double* gp, const double* dc, const double* pose,
                               const double* focal, const double* radial, const double* X, double* pose_new, double* focal_new,
                               double* radial_new, double* X_new, void* stream);

/* nero_sfm_ba_cost through the distortion, in the same fixed order.  P >= 1. */
int nero_sfm_radial_ba_cost(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                            const double* focal, const double* pp, const double* radial, const double* X, double* partial, double* cost,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_SFM_RADIAL_H_ */
