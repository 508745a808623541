// policy.cu — the host-side policy around the hot path (SURVEY.md §8f rank 4): keyframe admission, keyframe subset selection for
// one bundle adjustment, and the closed-form initial pose.  Scalar O(K^2) work on 4x4 matrices: plain host code, no kernels, no
// CUDA calls (these entry points work without a GPU).  Restated from
//   Utils::rotationGeodesicDistance          /root/reference/src/Utils.cpp:42-47
//   Bundler::checkAndAddKeyframe             /root/reference/src/Bundler.cpp:185-221
//   Bundler::selectKeyFramesForBA            /root/reference/src/Bundler.cpp:224-274   ("greedy_rot")
//   Utils::solveRigidTransformBetweenPoints  /root/reference/src/Utils.cpp:180-214      (used by SiftManager::procrustesByCorrespondence)
// Poses are row-major 4x4 cam->model like everywhere in this ABI.
#include <math.h>
#include <algorithm>
#include <limits>
#include <vector>
#include <string>
#include <stdio.h>
#include <string.h>
#include "bt_common.cuh"
#include "rigid.cuh"

namespace {

// acos((trace(R1 R2^T) - 1) / 2), clamped, in float like the reference
float geodesic(const float* A, const float* B) {
	float tr = 0.f;
	for (int r = 0; r < 3; r++)
		for (int c = 0; c < 3; c++) tr += A[r * 4 + c] * B[r * 4 + c];      // trace(R1 R2^T) = sum_rc R1(r,c) R2(r,c)
	float t = (tr - 1.f) / 2.0f;
	t = std::max(std::min(1.0f, t), -1.0f);
	return acosf(t);
}

}  // namespace

extern "C" float bt_rotation_geodesic(const float* pose_a, const float* pose_b) {
	if (!pose_a || !pose_b) return std::numeric_limits<float>::quiet_NaN();
	return geodesic(pose_a, pose_b);
}

extern "C" int bt_keyframe_check(const float* pose_new, int frame_id, int n_keypts, const float* keyframe_poses, int n_keyframes, int min_feat_num, float min_rot_deg) {
	if (frame_id == 0) return 1;                         // the first frame always becomes a keyframe
	if (!pose_new || (n_keyframes > 0 && !keyframe_poses)) return 0;
	if (n_keypts < min_feat_num) return 0;
	for (int i = 0; i < n_keyframes; i++) {
		const float rot_deg = geodesic(pose_new, keyframe_poses + 16 * (size_t)i) * 180 / (float)M_PI;
		if (rot_deg < min_rot_deg) return 0;             // too close in rotation to an existing keyframe
	}
	return 1;
}

extern "C" int bt_select_keyframes(const float* pose_new, const float* keyframe_poses, int n_keyframes, int max_BA_frames, int32_t* chosen_out, int* n_chosen_out) {
	BT_REQUIRE(pose_new && chosen_out && n_chosen_out && n_keyframes >= 0 && (n_keyframes == 0 || keyframe_poses) && max_BA_frames >= 1, BT_ERR_INVALID_ARG,
	           "bt_select_keyframes: bad arguments");
	std::vector<char> in(n_keyframes, 0);
	int n_in = 1;                                        // the new frame is always part of the window
	if (n_keyframes + 1 <= max_BA_frames) {
		for (int i = 0; i < n_keyframes; i++) in[i] = 1;
	} else {
		in[0] = 1; n_in = 2;                             // keyframe 0 anchors the model frame
		// greedy_rot: repeatedly add the keyframe with the smallest summed rotation distance to the frames chosen so far.  The
		// reference walks a std::set of shared_ptr (pointer order); here the chosen set is walked new frame first, then keyframes in
		// index order, and ties go to the lower index.
		while (n_in < max_BA_frames) {
			float best = std::numeric_limits<float>::max();
			int best_i = -1;
			for (int i = 0; i < n_keyframes; i++) {
				if (in[i]) continue;
				const float* kf = keyframe_poses + 16 * (size_t)i;
				float cum = geodesic(kf, pose_new);
				for (int j = 0; j < n_keyframes; j++) if (in[j]) cum += geodesic(kf, keyframe_poses + 16 * (size_t)j);
				if (cum < best) { best = cum; best_i = i; }
			}
			if (best_i < 0) break;                       // every distance was NaN / nothing left
			in[best_i] = 1; n_in++;
		}
	}
	int n = 0;
	for (int i = 0; i < n_keyframes; i++) if (in[i]) chosen_out[n++] = i;
	*n_chosen_out = n;
	return BT_OK;
}

extern "C" int bt_rigid_transform(const float* pts1, const float* pts2, int n, float* pose_out) {
	BT_REQUIRE(pts1 && pts2 && pose_out && n >= 3, BT_ERR_INVALID_ARG, "bt_rigid_transform: needs two arrays of >= 3 points");
	bt::RigidSums r;                                     // the same fit k_pose_init runs on the device (rigid.cuh)
	bt::rigid_init(r);
	for (int i = 0; i < n; i++) bt::rigid_add_means(r, pts1 + 3 * (size_t)i, pts2 + 3 * (size_t)i);
	bt::rigid_means(r, n);
	for (int i = 0; i < n; i++) bt::rigid_add_cov(r, pts1 + 3 * (size_t)i, pts2 + 3 * (size_t)i);
	bt::rigid_solve(r, pose_out);
	return BT_OK;
}

// ---- LF-Net reply (SURVEY.md §8f rank 3): Lfnet::detectFeature, /root/reference/src/FeatureManager.cpp:876-907, for rot_deg = 0 (the only
// value Bundler::processNewFrame passes, /root/reference/src/Bundler.cpp:104-107).  Wire format of the server's reply
// (lf-net-release/run_server.py:171-177): part 0 = int32 (n, dim), part 1 = float32 n x 2 keypoints (x, y) in the 400 x 400 network input,
// part 2 = float32 n x dim descriptors (row-major: exactly the matrix bt_knn_match_pairs takes, no repacking).  Keypoints go back to
// image pixels through forward^-1, forward = scale(400/side) * translate(-umin, -vmin), side = max(roi height, roi width).
extern "C" int bt_ba_gate(int n_edges_newframe, int min_fm_edges_newframe) {
	return n_edges_newframe > min_fm_edges_newframe ? 1 : 0;      // `if (n_edges_newframe<=min_fm_edges_newframe) { NO_BA; return; }`, Bundler.cpp:343
}

// inverse of a 4x4 in float, by cofactors (what Eigen's Matrix4f::inverse() evaluates); row-major in and out.  bt_pose_format and
// bt_pose_overlay (overlay.cu) share it, so the overlay draws with the ob_in_cam the pose file holds.
bool bt::inverse4(const float* m, float* inv) {
	float t[16];
	t[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
	t[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
	t[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
	t[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
	t[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
	t[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
	t[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
	t[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
	t[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
	t[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
	t[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
	t[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
	t[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
	t[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
	t[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
	t[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
	const float det = m[0] * t[0] + m[1] * t[4] + m[2] * t[8] + m[3] * t[12];
	if (!(det != 0.f)) return false;
	const float id = 1.0f / det;
	for (int i = 0; i < 16; i++) inv[i] = t[i] * id;
	return true;
}

extern "C" int bt_pose_format(const float* cur_in_model, char* text, int cap) {
	BT_REQUIRE(cur_in_model && text && cap > 0, BT_ERR_INVALID_ARG, "bt_pose_format: NULL argument");
	float ob[16];
	BT_REQUIRE(bt::inverse4(cur_in_model, ob), BT_ERR_INVALID_ARG, "bt_pose_format: the pose is singular");
	// Eigen's default IOFormat with the stream's precision: every coefficient printed like `os << std::setprecision(10) << float`
	// (= %.10g), padded on the left to the widest one, coefficients separated by one blank, rows by a newline, `endl` after the matrix
	char cell[16][40];
	size_t width = 0;
	for (int i = 0; i < 16; i++) { snprintf(cell[i], sizeof cell[i], "%.10g", (double)ob[i]); width = std::max(width, strlen(cell[i])); }
	std::string out;
	for (int r = 0; r < 4; r++) {
		for (int c = 0; c < 4; c++) {
			if (c) out += ' ';
			out.append(width - strlen(cell[r * 4 + c]), ' ');
			out += cell[r * 4 + c];
		}
		out += '\n';
	}
	BT_REQUIRE((int)out.size() + 1 <= cap, BT_ERR_CAPACITY, "bt_pose_format: %zu bytes needed, %d given", out.size() + 1, cap);
	memcpy(text, out.c_str(), out.size() + 1);
	return BT_OK;
}

extern "C" int bt_pose_write_txt(const char* path, const float* cur_in_model) {
	BT_REQUIRE(path, BT_ERR_INVALID_ARG, "bt_pose_write_txt: NULL path");
	char text[1024];
	const int rc = bt_pose_format(cur_in_model, text, (int)sizeof text);
	if (rc != BT_OK) return rc;
	FILE* f = fopen(path, "w");
	BT_REQUIRE(f != nullptr, BT_ERR_INVALID_ARG, "bt_pose_write_txt: cannot open %s", path);
	const size_t n = strlen(text);
	const bool ok = fwrite(text, 1, n, f) == n;
	BT_REQUIRE(fclose(f) == 0 && ok, BT_ERR_INVALID_ARG, "bt_pose_write_txt: short write to %s", path);
	return BT_OK;
}

extern "C" int bt_lfnet_parse_reply(const void* info, size_t info_bytes, const void* kpts, size_t kpts_bytes, size_t desc_bytes, const int* roi,
                                    float* kpts_out, int kpts_capacity, int* n_out, int* dim_out) {
	BT_REQUIRE(info && roi && n_out && dim_out, BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: NULL argument");
	BT_REQUIRE(info_bytes == 2 * sizeof(int32_t), BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: the first part must be 2 x int32 (n, dim), got %zu bytes", info_bytes);
	int32_t nd[2];
	memcpy(nd, info, sizeof nd);
	const int n = nd[0], dim = nd[1];
	BT_REQUIRE(n >= 0 && dim > 0, BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: bad header (n=%d, dim=%d)", n, dim);
	BT_REQUIRE(kpts_bytes == sizeof(float) * 2 * (size_t)n, BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: keypoint part has %zu bytes, %d keypoints need %zu", kpts_bytes, n, sizeof(float) * 2 * (size_t)n);
	BT_REQUIRE(desc_bytes == sizeof(float) * (size_t)n * dim, BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: descriptor part has %zu bytes, %d x %d floats need %zu", desc_bytes, n, dim, sizeof(float) * (size_t)n * dim);
	BT_REQUIRE(n == 0 || (kpts && kpts_out), BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: NULL keypoint buffer");
	BT_REQUIRE(n <= kpts_capacity, BT_ERR_CAPACITY, "bt_lfnet_parse_reply: %d keypoints > capacity %d", n, kpts_capacity);
	const int W = roi[1] - roi[0], H = roi[3] - roi[2];
	BT_REQUIRE(W > 0 && H > 0, BT_ERR_INVALID_ARG, "bt_lfnet_parse_reply: empty roi");
	const int side = std::max(H, W);
	// forward = [[a, 0, a*(-umin)], [0, b, b*(-vmin)], [0, 0, 1]]; its inverse as Eigen's 3x3 inverse forms it (cofactors times 1/det, float)
	const float a = 400 / float(side), b = 400 / float(side);
	const float f02 = a * (float)(-roi[0]), f12 = b * (float)(-roi[2]);
	const float invdet = 1.0f / (a * b);
	const float i00 = b * invdet, i11 = a * invdet, i02 = (0.f * f12 - f02 * b) * invdet, i12 = -(a * f12 - f02 * 0.f) * invdet;
	const float* k = (const float*)kpts;
	for (int i = 0; i < n; i++) {
		float xy[2];
		memcpy(xy, k + 2 * (size_t)i, sizeof xy);        // the message buffer need not be aligned
		kpts_out[2 * (size_t)i] = i00 * xy[0] + 0.f * xy[1] + i02 * 1.f;
		kpts_out[2 * (size_t)i + 1] = 0.f * xy[0] + i11 * xy[1] + i12 * 1.f;
	}
	*n_out = n; *dim_out = dim;
	return BT_OK;
}
