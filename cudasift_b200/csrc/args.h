// args.h -- the argument checks of the C ABI's matching, verification, tracks, triangulation, bundle adjustment and
// absolute pose calls (args.cu).  Each returns 0, or CS_E_ARG with cs_last_error() naming the offending argument; none
// makes a CUDA call, so they hold on a machine without a device.
#pragma once

#include "../../include/cudasift_b200.h"

namespace cs {

// CS_E_ARG, with "<fn>: invalid argument (CS_E_ARG): <fmt ...>" as the last error.
int arg_error(const char *fn, const char *fmt, ...) __attribute__((format(printf, 2, 3)));

// The two record sets and the path mode (0 auto, 1 exact, 2 tensor).
int check_sets(const char *fn, const void *s1, int n1, const void *s2, int n2, int mode);
// cs_match_mutual*: the sets, and a pairs buffer of maxPairs int2.  Both sets are written, so they must not overlap.
int mutual_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const void *pairs, int maxPairs,
                int mode);
// cs_match_ratio* and cs_match_guided*: the sets, the ratio parameters and a pairs buffer of maxPairs int2.
int ratio_args(const char *fn, const void *s1, int n1, const void *s2, int n2, float maxRatio, float maxDistance,
               const void *pairs, int maxPairs, int mode);
// cs_verify_pairs* and cs_verify_models: the records are only read (they may overlap each other); the pair and inlier
// buffers may overlap nothing.
int verify_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const void *pairs, int numPairs,
                int model, int numLoops, float thresh, const double *model_out, const void *inliers, int maxInliers);
// The idx / score buffers of a knn call: [n1][2] each.
int knn_out_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const int *idx, const float *score);
// The model and threshold of a guided call (the records and buffers are checked as for cs_match_knn2 / cs_match_ratio).
int guided_args(const char *fn, int model, const double *model_in, float thresh);
// cs_verify_essential*: those of cs_verify_pairs except model, the intrinsics and the three outputs.
int essential_args(const char *fn, const void *s1, int n1, const void *s2, int n2, const void *pairs, int numPairs,
                   const double *K1, const double *K2, int numLoops, float thresh, const double *E, const double *R,
                   const double *t, const void *inliers, int maxInliers);
// The batch calls: cs_verify_pairs_batch (essential false) and cs_verify_essential_batch, cs_match_ratio_batch,
// cs_match_guided_batch, cs_build_tracks (*N and *P receive the feature and pair totals), cs_triangulate_tracks,
// cs_bundle_adjust, and cs_absolute_pose_batch and cs_absolute_pose_models.
int verify_batch_args(const char *fn, const cs_verify_job *jobs, int numJobs, int model, int numLoops, float thresh,
                      const double *K1s, const double *K2s, bool essential);
int ratio_batch_args(const char *fn, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                     float maxRatio, float maxDistance, const int *counts_out);
int guided_batch_args(const char *fn, const cs_match_set *sets, int numSets, const cs_match_job *jobs, int numJobs,
                      const int *models, const double *models_in, float thresh, float maxRatio, float maxDistance,
                      const int *counts_out);
int tracks_args(const char *fn, const int *imageSizes, int numImages, const cs_track_list *lists, int numLists,
                int minLength, const int *trackOf, const int *offsets, int maxTracks, const int *members,
                int maxMembers, int *N, int *P);
int triangulate_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                     const double *ts, const int *offsets, int numTracks, const int *members, int numMembers,
                     int numTrials, double maxError, double minTriAngle, const double *points, const int *counts,
                     const float *errors, const unsigned char *inlier);
int bundle_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                const double *ts, const unsigned char *fixed, const int *offsets, int numTracks, const int *members,
                int numMembers, const unsigned char *use, const double *points, int maxIterations,
                int maxLinearIterations, double linearTol, double maxError, const double *R_out, const double *t_out,
                const float *errors, const unsigned char *inlier, const double *cost_out);
// cs_bundle_adjust_intrinsics past bundle_args: refine, loss, lossScale, dists and the host output aliasing rule.
int bundle_intrinsics_args(const char *fn, int numImages, const double *Ks, const double *dists,
                           const unsigned char *refine, int loss, double lossScale, const double *Rs, const double *ts,
                           const double *K_out, const double *dist_out, const double *R_out, const double *t_out);
// cs_undistort_records; *total receives the record total.
int undistort_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *dists,
                   void *const *d_out, long long *total);
// cs_rotation_averaging: the graph, its relative rotations and weights, the parameters and the host outputs.
int rotavg_args(const char *fn, int numImages, const int *edges, int numEdges, const double *Rrel,
                const double *weights, int refImage, int maxIterations, int maxLinearIterations, double linearTol,
                double sigmaDeg, double maxAngleDeg, const double *R_out, const double *residuals,
                const unsigned char *inlier, const double *cost_out, const double *trace_out);
// cs_global_positioning: the images (Rs[a] a rotation or all NaN), the tracks, the parameters and both range sweeps.
int globalpos_args(const char *fn, const cs_match_set *sets, int numImages, const double *Ks, const double *Rs,
                   const int *offsets, int numTracks, const int *members, int numMembers, const unsigned char *use,
                   int refImage, int loss, double lossScale, int maxIterations, int maxLinearIterations,
                   double linearTol, const double *t_out, const double *points, const double *cost_out,
                   const double *trace_out);
// cs_undistort_images, cs_patch_match_stereo(_geometric) and cs_fuse_depth_maps: the images and cameras, the jobs, the
// parameters and the range sweep.
int undistort_images_args(const char *fn, const cs_image *images, int numImages, const double *Ks,
                          const double *dists, float *const *d_out);
int patch_match_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                     const double *ts, const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep,
                     int numIterations, int topK);
int patch_match_geometric_args(const char *fn, const cs_image *images, int numImages, const double *Ks,
                               const double *Rs, const double *ts, const cs_depth_prior *priors,
                               const cs_stereo_job *jobs, int numJobs, int windowRadius, int windowStep,
                               int numIterations, int topK, double geomWeight, double geomMaxError);
int fuse_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
              const double *ts, const cs_stereo_job *jobs, int numJobs, float maxCost, int minConsistent,
              double maxReprojError, double maxDepthError, double maxNormalErrorDeg, const float *xyz,
              const float *normal, const float *intensity, const int *source, int maxPoints);
// cs_poisson_mesh: the points, the parameters, the buffers and the range sweep.
int mesh_args(const char *fn, const float *xyz, const float *normal, const float *intensity, int numPoints, int depth,
              double scale, int maxIterations, double tol, double trim, const float *vertices,
              const float *vertexIntensity, int maxVertices, const int *triangles, int maxTriangles, const float *chi);
// cs_poisson_mesh_screened: pointWeight, then mesh_args.
int mesh_screened_args(const char *fn, const float *xyz, const float *normal, const float *intensity, int numPoints,
                       int depth, double scale, double pointWeight, int maxIterations, double tol, double trim,
                       const float *vertices, const float *vertexIntensity, int maxVertices, const int *triangles,
                       int maxTriangles, const float *chi);
// cs_simplify_mesh: the mesh, the parameters, the buffers and the range sweep.
int simplify_args(const char *fn, const float *vertices, const float *vertexIntensity, int numVertices,
                  const int *triangles, int numTriangles, int targetTriangles, double maxError, double boundaryWeight,
                  const float *outVertices, const float *outIntensity, int maxOutVertices, const int *outTriangles,
                  int maxOutTriangles);
// cs_clean_mesh: the mesh size, the stage parameters, then simplify_args's buffer checks and range sweep.
int clean_args(const char *fn, const float *vertices, const float *vertexIntensity, int numVertices,
               const int *triangles, int numTriangles, int removeDegenerate, double longEdgeFactor,
               int removeNonManifold, int minComponentFaces, double minComponentFraction, int maxHoleEdges,
               int smoothIterations, double lambda, double mu, const float *outVertices, const float *outIntensity,
               int maxOutVertices, const int *outTriangles, int maxOutTriangles);
// cs_texture_mesh: the images and cameras, the mesh, the parameters, the buffers and the range sweep.
int texture_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                 const double *ts, const float *vertices, int numVertices, const int *triangles, int numTriangles,
                 double lambda, double maxViewAngleDeg, double depthTol, int padding, int atlasWidth, int maxSweeps,
                 const float *atlas, int maxAtlasRows, const float *uv, const int *faceView, const int *faceChart,
                 const int *chartsOut, int maxCharts);
// cs_texture_mesh_photo's three view-selection settings (after texture_args).
int texture_photo_args(const char *fn, int dataTerm, double outlierK, double outlierMinSigma);
// cs_texture_mesh_bp's sweep cap (after texture_photo_args).
int texture_bp_args(const char *fn, int maxBpSweeps);
// cs_level_texture_seams (local false: smoothness, regularization and d_cornerOffset checked) and
// cs_level_texture_seams_local (local true: stripWidth checked, no corner offsets): the mesh, the chart table, the
// parameters, the buffers and the range sweep.
int seams_args(const char *fn, const float *vertices, int numVertices, const int *triangles, int numTriangles,
               const int *faceView, const float *uv, const int *charts, int numCharts, const float *atlas,
               int atlasRows, int atlasWidth, int padding, double smoothness, double regularization, bool local,
               int stripWidth, int maxIterations, double tol, const float *outAtlas, const float *cornerOffset);
// cs_mesh_refine: the images and cameras, the mesh, the pairs, the parameters, the buffers and the range sweep.
int refine_args(const char *fn, const cs_image *images, int numImages, const double *Ks, const double *Rs,
                const double *ts, const float *vertices, int numVertices, const int *triangles, int numTriangles,
                const int *pairs, int numPairs, int windowRadius, double smoothness, double step, int maxIterations,
                double depthTol, const float *outVertices);
int pose_args(const char *fn, const double *points, int numPoints, const cs_pose_job *jobs, int numJobs,
              const double *Ks, int numLoops, double maxError);
// cs_vocab_assign, cs_vocab_train and cs_retrieve_pairs; *M and *N receive the feature totals.
int vocab_assign_args(const char *fn, const cs_match_set *sets, int numSets, const void *vocab, int numWords,
                      const int *wordOf, int *M);
int vocab_train_args(const char *fn, const cs_match_set *sets, int numSets, int numWords, int maxIterations,
                     const void *vocab, int *M);
int retrieve_args(const char *fn, const int *imageSizes, int numImages, const int *wordOf, int numWords, int topK,
                  const int *neighbours, const double *scores, const double *idf, const int *pairs, int maxPairs,
                  int *N);

}  // namespace cs
