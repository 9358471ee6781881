/* vf_b200_pose.h — the pose-scale augmentation of transformer training (MIGTConfig.random_pose_multiplier, models/migt.py:349-354,
 * 139-145, 158-160), in libvf_b200.so next to the entry points of vf_b200.h and under its conventions (raw device pointers, plain sizes,
 * vf_stream_t, 0 or a negative code with vf_last_error()).
 *
 * In training, scene b's views (views_per_scene consecutive poses [.,7] = xyz | wxyz) take one multiplier c_b = scene_mult[b]:
 *   vf_pose_model_input: the pose MLP's input out [rows,7] = [(xyz * pose_multiplier) * c_b | quaternion], one rounding per product;
 *     scene_mult null: [xyz * pose_multiplier | quaternion].
 *   vf_pose_loss_rows_scaled / vf_pose_loss_grad_scaled: vf_pose_loss_rows / vf_pose_loss_grad with the predicted xyz divided by c_b
 *     (its gradient carries 1 / c_b); tokens_per_view rows share a view.  scene_mult null: the unscaled entry points' bits.
 */
#ifndef VF_B200_POSE_H
#define VF_B200_POSE_H

#include "vf_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int vf_pose_model_input(const float* poses, int64_t rows, int views_per_scene, float pose_multiplier, const float* scene_mult, float* out,
                        vf_stream_t s);
int vf_pose_loss_rows_scaled(const float* raw, const float* poses, int64_t rows, int tokens_per_view, float pose_multiplier,
                             int views_per_scene, const float* scene_mult, float* pos_out, float* ori_out, vf_stream_t s);
int vf_pose_loss_grad_scaled(const float* raw, const float* poses, const float* row_weight, int64_t rows, int tokens_per_view,
                             float pose_multiplier, int views_per_scene, const float* scene_mult, float pos_scale, float ori_scale,
                             float* draw, vf_stream_t s);

#ifdef __cplusplus
}
#endif

#endif /* VF_B200_POSE_H */
