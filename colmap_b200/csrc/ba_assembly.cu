// ba_assembly.cu — problem assembly on flat scene views (DefaultBundleAdjuster's constructor) and the two-cams gauge.
#include "ba_common.cuh"

extern "C" {

// FixGaugeWithTwoCamsFromWorld (bundle_adjustment_ceres.cc:308-417), trivial frames, poses in ascending image id.
int b200ba_fix_gauge_two_cams_from_world(const b200ba_problem* p, const b200ba_options* o, uint8_t* pose_constant_out,
                                         int8_t* fixed_dim_out) {
  for (int i = 0; i < p->num_poses; ++i) {
    pose_constant_out[i] = p->pose_constant ? p->pose_constant[i] : 0;
    fixed_dim_out[i] = p->pose_fixed_translation_dim ? p->pose_fixed_translation_dim[i] : -1;
  }
  if (!o->refine_rig_from_world) return 0;
  int image1 = -1, image2 = -1, dim2 = 0;
  for (int i = 0; i < p->num_poses; ++i)
    if (pose_constant_out[i]) {
      if (image1 < 0) image1 = i;
      else return 0;  // two frames already fixed
    }
  for (int i = 0; i < p->num_poses; ++i) {
    if (image1 < 0) { image1 = i; continue; }
    if (i == image1) continue;
    // baseline = (frame1_from_world * inverse(frame_i_from_world)).translation = t1 - R1 R_i^T t_i
    const double* a = p->poses + 7 * image1;
    const double* b = p->poses + 7 * i;
    double Ra[9], Rb[9];
    ba_quat_to_R(a, Ra); ba_quat_to_R(b, Rb);
    double ci[3];  // -R_i^T t_i
    for (int r = 0; r < 3; ++r) ci[r] = -(Rb[r] * b[4] + Rb[3 + r] * b[5] + Rb[6 + r] * b[6]);
    double base[3];
    for (int r = 0; r < 3; ++r) base[r] = Ra[3 * r] * ci[0] + Ra[3 * r + 1] * ci[1] + Ra[3 * r + 2] * ci[2] + a[4 + r];
    int mi = 0;
    for (int r = 1; r < 3; ++r) if (fabs(base[r]) > fabs(base[mi])) mi = r;
    if (fabs(base[mi]) > 1e-9) { image2 = i; dim2 = mi; break; }
  }
  if (image1 < 0 || image2 < 0) return 1;
  pose_constant_out[image1] = 1;
  if (!pose_constant_out[image2]) fixed_dim_out[image2] = (int8_t)dim2;
  return 0;
}

// ---- problem assembly (see the header): DefaultBundleAdjuster's constructor on flat views ----
struct b200ba_assembly {
  std::vector<double> poses, cam_params, points, obs_xy;
  std::vector<uint8_t> pose_constant, cam_constant, point_constant;
  std::vector<int8_t> pose_fixed_dim;
  std::vector<int32_t> cam_model, cam_off, obs_pose, obs_cam, obs_point;
  std::vector<double> sensors;              // rigs: sensor_from_rig of the non-reference cameras
  std::vector<uint8_t> sensor_constant;
  std::vector<int32_t> cam_sensor;
  b200ba_problem problem;
};

int b200ba_assemble(const b200ba_options* o, const b200ba_scene* sc, const b200ba_config* cfg, b200ba_assembly_t* out) {
  if (!o || !sc || !cfg || !out) return ba_fail(-1, "null argument");
  const int NI = sc->num_images, NC = sc->num_cameras;
  const int64_t NPT = sc->num_points3D;
  auto flag = [](const uint8_t* f, int64_t i) { return f && f[i]; };
  for (int i = 0; i < NI; ++i) if (sc->image_camera[i] < 0 || sc->image_camera[i] >= NC) return ba_fail(-2, "image references a camera outside the scene");
  for (int c = 0; c < NC; ++c) if (ba_model_num_params(sc->camera_model_id[c]) < 0) return ba_fail(-2, "unsupported camera model");
  const int NF = sc->num_frames;
  const bool rigs = NF > 0;
  if (rigs) {
    if (!sc->image_frame || !sc->rig_from_world || !sc->frame_rig || !sc->rig_ref_camera || !sc->camera_rig || !sc->camera_sensor_from_rig)
      return ba_fail(-2, "frames need image_frame, rig_from_world, frame_rig, rig_ref_camera, camera_rig and camera_sensor_from_rig");
    for (int i = 0; i < NI; ++i) if (sc->image_frame[i] < 0 || sc->image_frame[i] >= NF) return ba_fail(-2, "image references a frame outside the scene");
    for (int f = 0; f < NF; ++f) if (sc->frame_rig[f] < 0 || sc->frame_rig[f] >= sc->num_rigs) return ba_fail(-2, "frame references a rig outside the scene");
    for (int c = 0; c < NC; ++c) if (sc->camera_rig[c] < 0 || sc->camera_rig[c] >= sc->num_rigs) return ba_fail(-2, "camera references a rig outside the scene");
    for (int r = 0; r < sc->num_rigs; ++r) if (sc->rig_ref_camera[r] < 0 || sc->rig_ref_camera[r] >= NC) return ba_fail(-2, "rig references a camera outside the scene");
  }
  b200ba_assembly* A = new b200ba_assembly();
  std::vector<int64_t> point_num_obs((size_t)NPT, 0);
  auto track_len = [&](int64_t pid) { return sc->track_offset[pid + 1] - sc->track_offset[pid]; };
  std::vector<int> extra_pose_of_image;     // rigs: constant pose entry of an image outside the config (-1 = none yet)
  if (rigs) { extra_pose_of_image.assign(NI, -1); A->poses.assign(sc->rig_from_world, sc->rig_from_world + 7 * (size_t)NF); }
  auto push = [&](int img, int64_t pid, const double* xy) {
    int pose = img;
    if (rigs) {
      if (flag(cfg->image_in_config, img)) pose = sc->image_frame[img];
      else {
        if (extra_pose_of_image[img] < 0) {
          extra_pose_of_image[img] = (int)(A->poses.size() / 7);
          const double* f = sc->rig_from_world + 7 * (size_t)sc->image_frame[img];
          A->poses.insert(A->poses.end(), f, f + 7);
        }
        pose = extra_pose_of_image[img];
      }
    }
    A->obs_pose.push_back(pose); A->obs_cam.push_back(sc->image_camera[img]); A->obs_point.push_back((int32_t)pid);
    A->obs_xy.push_back(xy[0]); A->obs_xy.push_back(xy[1]);
    point_num_obs[pid] += 1;
  };
  // AddImageToProblem: every observation of the config's images (:688-751); an image (and its camera) counts as
  // parameterized only if it contributed at least one observation (:745-748)
  std::vector<uint8_t> image_parameterized(NI, 0);
  for (int i = 0; i < NI; ++i) {
    if (!flag(cfg->image_in_config, i)) continue;
    const size_t before = A->obs_pose.size();
    for (int64_t k = sc->point2D_offset[i]; k < sc->point2D_offset[i + 1]; ++k) {
      const int64_t pid = sc->point2D_point3D[k];
      if (pid < 0) continue;
      if (pid >= NPT) { delete A; return ba_fail(-2, "point2D references a point outside the scene"); }
      if (flag(cfg->point_ignored, pid)) continue;
      if (track_len(pid) < cfg->min_track_length) continue;
      push(i, pid, sc->point2D_xy + 2 * k);
    }
    if (A->obs_pose.size() > before) image_parameterized[i] = 1;
  }
  // AddPointToProblem: explicit config points bring the observations made by images outside the config (:829-888)
  for (int64_t pid = 0; pid < NPT; ++pid) {
    if (!flag(cfg->point_variable, pid) && !flag(cfg->point_constant, pid)) continue;
    if (cfg->min_track_length > 0 && track_len(pid) < cfg->min_track_length) continue;   // :835-838
    if (point_num_obs[pid] == track_len(pid)) continue;
    for (int64_t t = sc->track_offset[pid]; t < sc->track_offset[pid + 1]; ++t) {
      const int img = sc->track_image[t];
      if (img < 0 || img >= NI) { delete A; return ba_fail(-2, "track references an image outside the scene"); }
      if (flag(cfg->image_in_config, img)) continue;
      const int64_t k = sc->point2D_offset[img] + sc->track_point2D[t];
      if (k < sc->point2D_offset[img] || k >= sc->point2D_offset[img + 1]) { delete A; return ba_fail(-2, "track references a point2D outside its image"); }
      push(img, pid, sc->point2D_xy + 2 * k);
    }
  }
  if (!rigs) A->poses.assign(sc->cam_from_world, sc->cam_from_world + 7 * (size_t)NI);
  const int NPOSE = (int)(A->poses.size() / 7);
  A->pose_constant.assign(NPOSE, 1);
  A->pose_fixed_dim.assign(NPOSE, -1);
  std::vector<uint8_t> cam_in_cfg(NC, 0);
  for (int i = 0; i < NI; ++i)
    if (flag(cfg->image_in_config, i)) {
      if (image_parameterized[i]) cam_in_cfg[sc->image_camera[i]] = 1;
      if (rigs) { if (!flag(cfg->frame_constant_pose, sc->image_frame[i])) A->pose_constant[sc->image_frame[i]] = 0; }
      else if (!flag(cfg->image_constant_pose, i)) A->pose_constant[i] = 0;
    }
  // cameras seen only through constant-pose factors of outside images stay constant (:863-878)
  A->cam_constant.resize(NC);
  for (int c = 0; c < NC; ++c) A->cam_constant[c] = (!cam_in_cfg[c] || flag(cfg->camera_constant, c)) ? 1 : 0;
  A->cam_model.assign(sc->camera_model_id, sc->camera_model_id + NC);
  A->cam_off.assign(sc->camera_param_offset, sc->camera_param_offset + NC);
  int64_t nparams = 0;
  for (int c = 0; c < NC; ++c) nparams = std::max<int64_t>(nparams, sc->camera_param_offset[c] + ba_model_num_params(sc->camera_model_id[c]));
  A->cam_params.assign(sc->camera_params, sc->camera_params + nparams);
  // ParameterizePoints (:540-565): variable iff refined and fully observed inside the problem; explicit constants win
  A->points.assign(sc->xyz, sc->xyz + 3 * (size_t)NPT);
  A->point_constant.assign((size_t)NPT, 1);
  for (int64_t pid = 0; pid < NPT; ++pid) {
    if (point_num_obs[pid] > 0 && o->refine_points3D && track_len(pid) <= point_num_obs[pid]) A->point_constant[pid] = 0;
    if (flag(cfg->point_constant, pid)) A->point_constant[pid] = 1;
  }
  b200ba_problem& P = A->problem;
  memset(&P, 0, sizeof(P));
  P.num_poses = NPOSE; P.poses = A->poses.data(); P.pose_constant = A->pose_constant.data(); P.pose_fixed_translation_dim = A->pose_fixed_dim.data();
  P.num_cameras = NC; P.camera_model_id = A->cam_model.data(); P.camera_param_offset = A->cam_off.data(); P.camera_params = A->cam_params.data();
  P.camera_constant = A->cam_constant.data();
  P.num_points = NPT; P.points = A->points.data(); P.point_constant = A->point_constant.data();
  P.num_observations = (int64_t)A->obs_pose.size();
  P.obs_pose_idx = A->obs_pose.data(); P.obs_camera_idx = A->obs_cam.data(); P.obs_point_idx = A->obs_point.data(); P.obs_xy = A->obs_xy.data();
  P.num_config_images = 0;
  for (int i = 0; i < NI; ++i) if (flag(cfg->image_in_config, i)) P.num_config_images += 1;   // config.NumImages() (:131)
  bool three_points = cfg->fixed_gauge == 2;
  if (rigs) {
    // ParameterizeRigsAndFrames (:470-538): sensor_from_rig is constant when not refined, constant in the config, or when
    // the reference sensor of its rig is not part of the problem.  Sensors = non-reference cameras, ascending camera index.
    A->cam_sensor.assign(NC, -1);
    for (int c = 0; c < NC; ++c)
      if (sc->rig_ref_camera[sc->camera_rig[c]] != c) {
        A->cam_sensor[c] = (int32_t)A->sensor_constant.size();
        A->sensors.insert(A->sensors.end(), sc->camera_sensor_from_rig + 7 * (size_t)c, sc->camera_sensor_from_rig + 7 * (size_t)c + 7);
        // (a parameter block only through a parameterized image of the config on that camera; outside images are baked)
        A->sensor_constant.push_back((!o->refine_sensor_from_rig || flag(cfg->camera_constant_sensor_from_rig, c) || !cam_in_cfg[c]) ? 1 : 0);
      }
    std::vector<uint8_t> rig_param(sc->num_rigs, 0);
    for (int i = 0; i < NI; ++i) if (flag(cfg->image_in_config, i) && image_parameterized[i]) rig_param[sc->frame_rig[sc->image_frame[i]]] = 1;
    for (int c = 0; c < NC; ++c) {
      const int r = sc->camera_rig[c];
      if (A->cam_sensor[c] >= 0 && rig_param[r] && !cam_in_cfg[sc->rig_ref_camera[r]]) A->sensor_constant[A->cam_sensor[c]] = 1;
    }
    P.num_sensors = (int)A->sensor_constant.size();
    P.sensor_from_rig = A->sensors.data(); P.sensor_constant = A->sensor_constant.data(); P.camera_sensor_idx = A->cam_sensor.data();
    // FixGaugeWithTwoCamsFromWorld with rigs (:308-417), over the parameterized images in ascending image id
    if (cfg->fixed_gauge == 1 && o->refine_rig_from_world) {
      auto const_sensor = [&](int img) { const int sidx = A->cam_sensor[sc->image_camera[img]]; return sidx < 0 || A->sensor_constant[sidx]; };   // IsParameterizedConstSensor
      int image1 = -1, image2 = -1, dim2 = 0;
      bool done = false;
      for (int i = 0; i < NI && !done; ++i) {
        if (!flag(cfg->image_in_config, i) || !image_parameterized[i]) continue;
        if (flag(cfg->frame_constant_pose, sc->image_frame[i]) && const_sensor(i)) {
          if (image1 < 0) image1 = i;
          else if (sc->image_frame[image1] != sc->image_frame[i]) done = true;   // two frames are already fixed
        }
      }
      if (!done) {
        for (int i = 0; i < NI; ++i) {
          if (!flag(cfg->image_in_config, i) || !image_parameterized[i]) continue;
          const int f = sc->image_frame[i];
          if (image1 < 0 && const_sensor(i)) { image1 = i; continue; }
          if (image1 >= 0 && sc->image_frame[image1] != f && const_sensor(i) && !flag(cfg->frame_constant_pose, f)) {
            // baseline = (frame1_from_world * inverse(frame_from_world)).translation = t1 - R1 R^T t
            const double* a = sc->rig_from_world + 7 * (size_t)sc->image_frame[image1];
            const double* b = sc->rig_from_world + 7 * (size_t)f;
            double Ra[9], Rb[9], ci[3], base[3];
            ba_quat_to_R(a, Ra); ba_quat_to_R(b, Rb);
            for (int r = 0; r < 3; ++r) ci[r] = -(Rb[r] * b[4] + Rb[3 + r] * b[5] + Rb[6 + r] * b[6]);
            for (int r = 0; r < 3; ++r) base[r] = Ra[3 * r] * ci[0] + Ra[3 * r + 1] * ci[1] + Ra[3 * r + 2] * ci[2] + a[4 + r];
            int mi = 0;
            for (int r = 1; r < 3; ++r) if (fabs(base[r]) > fabs(base[mi])) mi = r;
            if (fabs(base[mi]) > 1e-9) { image2 = i; dim2 = mi; break; }
          }
        }
        if (image1 < 0 || image2 < 0) three_points = true;   // "Falling back to fixing Gauge with three points" (:390-394)
        else {
          A->pose_constant[sc->image_frame[image1]] = 1;
          if (!flag(cfg->frame_constant_pose, sc->image_frame[image2])) A->pose_fixed_dim[sc->image_frame[image2]] = (int8_t)dim2;
        }
      }
    }
  }
  // FixGauge (:270-417), TWO_CAMS_FROM_WORLD, trivial frames: the search runs over the config's images in ascending image id
  if (!rigs && cfg->fixed_gauge == 1 && o->refine_rig_from_world) {
    std::vector<int> idx;
    for (int i = 0; i < NI; ++i) if (flag(cfg->image_in_config, i) && image_parameterized[i]) idx.push_back(i);   // parameterized_image_ids_
    std::vector<double> sp(7 * idx.size());
    std::vector<uint8_t> sc_in(idx.size()), sc_out(idx.size());
    std::vector<int8_t> sd_in(idx.size(), -1), sd_out(idx.size());
    for (size_t k = 0; k < idx.size(); ++k) { memcpy(sp.data() + 7 * k, A->poses.data() + 7 * (size_t)idx[k], 56); sc_in[k] = A->pose_constant[idx[k]]; }
    b200ba_problem sub;
    memset(&sub, 0, sizeof(sub));
    sub.num_poses = (int)idx.size(); sub.poses = sp.data(); sub.pose_constant = sc_in.data(); sub.pose_fixed_translation_dim = sd_in.data();
    if (b200ba_fix_gauge_two_cams_from_world(&sub, o, sc_out.data(), sd_out.data()) == 1) {
      three_points = true;   // "Failed to fix Gauge with two cameras. Falling back to fixing Gauge with three points." (:390-394)
    } else {
      for (size_t k = 0; k < idx.size(); ++k) { A->pose_constant[idx[k]] = sc_out[k]; A->pose_fixed_dim[idx[k]] = sd_out[k]; }
    }
  }
  // FixGaugeWithThreePoints (:270-306): three points whose coordinate vectors are linearly independent stay fixed; points
  // that are already constant count first.  The reference walks a hash map (unspecified order); here ascending point id.
  if (three_points) {
    double basis[9];
    int nfixed = 0;
    double max_pivot = 0.0;
    auto maybe_add = [&](const double* X) {   // rank test of [fixed points | X] by Gram-Schmidt, Eigen's default threshold
      if (nfixed >= 3) return false;
      double r[3] = {X[0], X[1], X[2]};
      for (int b = 0; b < nfixed; ++b) {
        const double* q = basis + 3 * b;
        const double d = r[0] * q[0] + r[1] * q[1] + r[2] * q[2];
        for (int c = 0; c < 3; ++c) r[c] -= d * q[c];
      }
      const double nr = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
      const double nx = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
      if (!(nr > 3.0 * 2.220446049250313e-16 * std::max(max_pivot, nx))) return false;
      for (int c = 0; c < 3; ++c) basis[3 * nfixed + c] = r[c] / nr;
      max_pivot = std::max(max_pivot, nx);
      ++nfixed;
      return true;
    };
    for (int64_t pid = 0; pid < NPT && nfixed < 3; ++pid)
      if (point_num_obs[pid] > 0 && A->point_constant[pid]) maybe_add(A->points.data() + 3 * pid);
    for (int64_t pid = 0; pid < NPT && nfixed < 3; ++pid)
      if (point_num_obs[pid] > 0 && !A->point_constant[pid] && maybe_add(A->points.data() + 3 * pid)) A->point_constant[pid] = 1;
    if (nfixed < 3) g_ba_error = "Failed to fix Gauge due to insufficient number of fixed points";   // warning, like the reference
  }
  *out = A;
  return 0;
}
b200ba_problem* b200ba_assembly_problem(b200ba_assembly_t a) { return a ? &a->problem : nullptr; }
void b200ba_assembly_free(b200ba_assembly_t a) { delete a; }

}  // extern "C"
