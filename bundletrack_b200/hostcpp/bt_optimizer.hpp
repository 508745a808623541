// bt_optimizer.hpp — C++ host shim with the REFERENCE'S signatures on top of the C-ABI (include/bundletrack_b200.h).
//
// Drop-in for what BundleTrack's host code talks to on the hot path:
//   * OptimizerGpu::optimizeFrames      (/root/reference/src/cuda/LossGPU.h:50, called from Bundler::optimizeGPU,
//                                        /root/reference/src/Bundler.cpp:350-351)
//   * ransacMultiPairGPU                (/root/reference/src/cuda/cuda_ransac.h:50, called from
//                                        SiftManager::runRansacMultiPairGPU, /root/reference/src/FeatureManager.cpp:713)
//   * knnMatchBothDirections            (the two cv::cuda::DescriptorMatcher::knnMatch calls of SiftManager::findCorresbyNN,
//                                        /root/reference/src/FeatureManager.cpp:271-273)
//   * processDepthAndNormals            (Frame::processDepth + Frame::depthToCloudAndNormals, /root/reference/src/Frame.cpp:152-233)
// Header-only, no Eigen/yaml-cpp/OpenCV dependency of its own: the pose and intrinsics types are template parameters
// that only need operator()(row, col) (Eigen::Matrix4f / Matrix3f satisfy it), and the yml values arrive through
// BtSolverConfig, which the caller fills from the UNCHANGED config_*.yml keys (see INTEGRATION.md for the 6-line
// yaml-cpp version).  Errors are thrown as std::runtime_error with bt_last_error(); nothing exits or hangs.
#pragma once
#include <cmath>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>
#include "../../include/bundletrack_b200.h"

struct BtSolverConfig {            // bundle.* / p2p.* of config_nocs.yml, same names
	int num_iter_outter = 7;
	int num_iter_inner = 5;
	float robust_delta = 0.005f;
	float image_downscale = 4.f;
	float p2p_max_dist = 0.02f;
	float p2p_max_normal_angle = 45.f;   // degrees, converted like CUDASolverBundling.cpp:94
	bt_solver_params to_params() const {
		bt_solver_params p;
		p.num_iter_outer = num_iter_outter; p.num_iter_inner = num_iter_inner; p.robust_delta = robust_delta; p.image_downscale = image_downscale;
		p.dense_dist_thresh = p2p_max_dist; p.dense_cos_normal_thresh = std::cos(p2p_max_normal_angle / 180.0 * M_PI);
		p.depth_min = 0.1f; p.depth_max = 9999.f; p.w_sparse = 1.f; p.w_dense = 1.f;
		return p;
	}
};

// Layout-compatible with the reference's EntryJ (SIFTImageManager.h:44-59); BundleTrack code can pass its own
// std::vector<EntryJ> through reinterpret_cast<const bt_entryj*>.
static_assert(sizeof(bt_entryj) == 32, "EntryJ layout");

class OptimizerGpu {
public:
	// max_windows > 1 lets optimizeWindows() solve several independent windows in ONE call (one launch sequence for the batch).
	explicit OptimizerGpu(const BtSolverConfig& cfg, int device = 0, int max_frames = 15, int max_corr = 1 << 16, int H = 480, int W = 640, int max_windows = 1)
	    : cfg_(cfg) {
		check(bt_ctx_create(&ctx_, device), "bt_ctx_create");
		bt_solver_limits lim = { max_windows, max_frames, max_corr, H, W, cfg.image_downscale };
		check(bt_solver_reserve(ctx_, &lim), "bt_solver_reserve");
	}
	~OptimizerGpu() { bt_ctx_destroy(ctx_); }
	OptimizerGpu(const OptimizerGpu&) = delete;
	OptimizerGpu& operator=(const OptimizerGpu&) = delete;

	// Same argument list as the reference.  colors_gpu is unused there too (LossGPU.cu:53, SBA.cpp:28-32); n_match_per_pair is unused there and optional here.
	// `poses` is in-out: every frame of the window is overwritten with its optimised cam->model pose.
	template <class EntryJT, class Uchar4T, class Float4T, class Mat4, class Alloc, class Mat3>
	void optimizeFrames(const std::vector<EntryJT>& global_corres, const std::vector<int>& n_match_per_pair, int n_frames, int H, int W,
	                    const std::vector<float*>& depths_gpu, const std::vector<Uchar4T*>& /*colors_gpu*/, const std::vector<Float4T*>& normals_gpu,
	                    std::vector<Mat4, Alloc>& poses, const Mat3& K, void* stream = nullptr) {
		static_assert(sizeof(EntryJT) == sizeof(bt_entryj), "EntryJ must be the 32-byte reference struct");
		std::vector<const float*> dptr(n_frames), nptr(n_frames);
		std::vector<float> flat(16 * (size_t)n_frames);
		for (int f = 0; f < n_frames; f++) {
			dptr[f] = depths_gpu[f];
			nptr[f] = reinterpret_cast<const float*>(normals_gpu[f]);
			for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) flat[16 * f + 4 * r + c] = poses[f](r, c);   // Eigen is column-major; the ABI is row-major
		}
		bt_window win{};
		win.n_frames = n_frames; win.H = H; win.W = W;
		win.n_corr = (int)global_corres.size();
		win.corr = reinterpret_cast<const bt_entryj*>(global_corres.data());
		win.depth_dev = dptr.data(); win.normal_dev = nptr.data();
		win.fx = K(0, 0); win.fy = K(1, 1); win.cx = K(0, 2); win.cy = K(1, 2);
		win.dense_pairs = nullptr; win.n_dense_pairs = 0; win.compat_flip = 1;
		// Bundler::optimizeGPU pushes one count per frame pair next to the entries it emits pair by pair (Bundler.cpp:298-324): when the
		// counts cover the list they save the library its own grouping pass over the entries
		long long covered = 0;
		for (int v : n_match_per_pair) covered += v;
		if (!n_match_per_pair.empty() && covered == (long long)global_corres.size()) { win.n_blocks = (int)n_match_per_pair.size(); win.block_n = n_match_per_pair.data(); }
		const bt_solver_params prm = cfg_.to_params();
		check(bt_solve_windows(ctx_, 1, &win, &prm, flat.data(), stream), "bt_solve_windows");
		for (int f = 0; f < n_frames; f++)
			for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) poses[f](r, c) = flat[16 * f + 4 * r + c];
	}
	// Bundler::optimizeGPU from the gate onwards (/root/reference/src/Bundler.cpp:343-358): `n_edges_newframe` = the number of emitted
	// correspondences with the new frame on either side.  Returns false (the caller sets _newframe->_status = Frame::NO_BA) without
	// touching the GPU when the new frame has too few edges, true after optimizeFrames has rewritten `poses`.
	template <class EntryJT, class Uchar4T, class Float4T, class Mat4, class Alloc, class Mat3>
	bool optimizeGPU(const std::vector<EntryJT>& global_corres, const std::vector<int>& n_match_per_pair, int n_edges_newframe, int min_fm_edges_newframe,
	                 int n_frames, int H, int W, const std::vector<float*>& depths_gpu, const std::vector<Uchar4T*>& colors_gpu,
	                 const std::vector<Float4T*>& normals_gpu, std::vector<Mat4, Alloc>& poses, const Mat3& K, void* stream = nullptr) {
		if (!bt_ba_gate(n_edges_newframe, min_fm_edges_newframe)) return false;
		optimizeFrames(global_corres, n_match_per_pair, n_frames, H, W, depths_gpu, colors_gpu, normals_gpu, poses, K, stream);
		return true;
	}
	// Batched form: the windows of several tracked objects (or several frames' worth of work) in one call.  Every element of `windows`
	// carries what one optimizeFrames call takes; poses[w] is in-out like above.
	template <class EntryJT, class Float4T, class Mat4, class Alloc, class Mat3>
	struct WindowArgs {
		const std::vector<EntryJT>* global_corres; int n_frames, H, W;
		const std::vector<float*>* depths_gpu; const std::vector<Float4T*>* normals_gpu;
		std::vector<Mat4, Alloc>* poses; const Mat3* K;
	};
	template <class EntryJT, class Float4T, class Mat4, class Alloc, class Mat3>
	void optimizeWindows(const std::vector<WindowArgs<EntryJT, Float4T, Mat4, Alloc, Mat3>>& windows, void* stream = nullptr) {
		static_assert(sizeof(EntryJT) == sizeof(bt_entryj), "EntryJ must be the 32-byte reference struct");
		const size_t nw = windows.size();
		if (nw == 0) return;
		std::vector<bt_window> wins(nw);
		std::vector<std::vector<const float*>> dptr(nw), nptr(nw);
		std::vector<float> flat;
		for (size_t w = 0; w < nw; w++) {
			const auto& a = windows[w];
			dptr[w].resize(a.n_frames); nptr[w].resize(a.n_frames);
			for (int f = 0; f < a.n_frames; f++) {
				dptr[w][f] = (*a.depths_gpu)[f]; nptr[w][f] = reinterpret_cast<const float*>((*a.normals_gpu)[f]);
				for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) flat.push_back((*a.poses)[f](r, c));
			}
			bt_window win{};
			win.n_frames = a.n_frames; win.H = a.H; win.W = a.W;
			win.n_corr = (int)a.global_corres->size(); win.corr = reinterpret_cast<const bt_entryj*>(a.global_corres->data());
			win.depth_dev = dptr[w].data(); win.normal_dev = nptr[w].data();
			win.fx = (*a.K)(0, 0); win.fy = (*a.K)(1, 1); win.cx = (*a.K)(0, 2); win.cy = (*a.K)(1, 2);
			win.compat_flip = 1;
			wins[w] = win;
		}
		const bt_solver_params prm = cfg_.to_params();
		check(bt_solve_windows(ctx_, (int)nw, wins.data(), &prm, flat.data(), stream), "bt_solve_windows");
		size_t o = 0;
		for (size_t w = 0; w < nw; w++)
			for (int f = 0; f < windows[w].n_frames; f++, o += 16)
				for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) (*windows[w].poses)[f](r, c) = flat[o + 4 * r + c];
	}
	bt_ctx* ctx() { return ctx_; }

private:
	static void check(int rc, const char* what) {
		if (rc != BT_OK) throw std::runtime_error(std::string(what) + ": " + bt_last_error());
	}
	BtSolverConfig cfg_;
	bt_ctx* ctx_ = nullptr;
};

// Bundler::saveNewframeResult's pose record (/root/reference/src/Bundler.cpp:362-378): <pose_out_dir>/<id_str>.txt holds ob_in_cam =
// cur_in_model^-1 printed with 10 significant digits the way Eigen prints a Matrix4f.  The caller creates the directory, as the reference does.
template <class Mat4>
inline void saveNewframePose(const std::string& path, const Mat4& cur_in_model) {
	float flat[16];
	for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) flat[4 * r + c] = cur_in_model(r, c);
	if (bt_pose_write_txt(path.c_str(), flat) != BT_OK) throw std::runtime_error(std::string("bt_pose_write_txt: ") + bt_last_error());
}

// scripts/Utils.py add / adi for a whole sequence in one device call: ADD and ADD-S per frame (metres) into add_gpu / adds_gpu (device double
// [n_frames]), asynchronous on `stream`.  model_pts_gpu: device double n_pts x 3 (points.xyz); pred / gt: ob_in_cam per frame as the
// reference's poses/<id>.txt hold them.  The context needs bt_metrics_reserve(ctx, >= n_pts, >= pred.size()).
template <class Mat4>
inline void poseMetrics(bt_ctx* ctx, const double* model_pts_gpu, int n_pts, const std::vector<Mat4>& pred, const std::vector<Mat4>& gt, double* add_gpu,
                        double* adds_gpu, void* stream = nullptr) {
	if (pred.size() != gt.size()) throw std::runtime_error("poseMetrics: pred and gt differ in length");
	std::vector<double> p(16 * pred.size()), g(16 * gt.size());
	for (size_t f = 0; f < pred.size(); f++)
		for (int r = 0; r < 4; r++)
			for (int c = 0; c < 4; c++) { p[16 * f + 4 * r + c] = pred[f](r, c); g[16 * f + 4 * r + c] = gt[f](r, c); }
	if (bt_pose_metrics(ctx, model_pts_gpu, n_pts, p.data(), g.data(), (int)pred.size(), add_gpu, adds_gpu, stream) != BT_OK)
		throw std::runtime_error(std::string("bt_pose_metrics: ") + bt_last_error());
}

// eval_ycbineoat.py's VOCap: the AUC of the errors up to max_err (0.1 m), divided by max_err; x 100 is the number the paper's table prints.
inline double voCap(const std::vector<double>& err, double max_err = 0.1) {
	double auc = 0.0;
	if (bt_vocap(err.data(), (int)err.size(), max_err, &auc) != BT_OK) throw std::runtime_error(std::string("bt_vocap: ") + bt_last_error());
	return auc;
}

// scripts/benchmark.py (6-PACK, NOCS-REAL275) per record in one device call: theta (degrees), shift and IoU into device double [n] arrays,
// asynchronous on `stream`.  pred / gt as the benchmark compares them (translations in mm); corners: 24 doubles per record (the 8 rows of
// model_scales/<model>.txt); symmetric: bottle, bowl and can.  The context needs bt_nocs_reserve(ctx, >= pred.size()).
template <class Mat4>
inline void nocsMetrics(bt_ctx* ctx, const std::vector<Mat4>& pred, const std::vector<Mat4>& gt, const std::vector<double>& corners,
                        const std::vector<int32_t>& symmetric, double* theta_gpu, double* shift_gpu, double* iou_gpu, void* stream = nullptr) {
	if (pred.size() != gt.size() || symmetric.size() != pred.size() || corners.size() != 24 * pred.size())
		throw std::runtime_error("nocsMetrics: pred, gt, corners and symmetric differ in length");
	std::vector<double> p(16 * pred.size()), g(16 * gt.size());
	for (size_t f = 0; f < pred.size(); f++)
		for (int r = 0; r < 4; r++)
			for (int c = 0; c < 4; c++) { p[16 * f + 4 * r + c] = pred[f](r, c); g[16 * f + 4 * r + c] = gt[f](r, c); }
	if (bt_nocs_metrics(ctx, p.data(), g.data(), corners.data(), symmetric.data(), (int)pred.size(), theta_gpu, shift_gpu, iou_gpu, stream) != BT_OK)
		throw std::runtime_error(std::string("bt_nocs_metrics: ") + bt_last_error());
}

// benchmark.py's aggregation: per class (bottle .. mug) and overall {5 deg 5 cm fraction, IoU25 fraction, mean theta, mean shift (mm)}.
struct NocsScore { double per_class[6][4]; double overall[4]; };
inline NocsScore nocsScore(const std::vector<int32_t>& cls, const std::vector<int32_t>& scored, const std::vector<double>& theta_deg,
                           const std::vector<double>& shift, const std::vector<double>& iou) {
	const size_t n = cls.size();
	if (scored.size() != n || theta_deg.size() != n || shift.size() != n || iou.size() != n) throw std::runtime_error("nocsScore: lengths differ");
	NocsScore s;
	if (bt_nocs_score(cls.data(), scored.data(), theta_deg.data(), shift.data(), iou.data(), (int)n, &s.per_class[0][0], s.overall) != BT_OK)
		throw std::runtime_error(std::string("bt_nocs_score: ") + bt_last_error());
	return s;
}

// ransacMultiPairGPU with the reference's argument list (device float4 arrays per pair, host result vectors).  The device result
// buffers and the library's scratch belong to the object: nothing is allocated per call (the reference allocates six arrays and a
// stream per pair per call, cuda_ransac.cu:1240-1275).
class RansacGpu {
public:
	RansacGpu(bt_ctx* ctx, int max_pairs, int max_pts_per_pair, int max_trials) : ctx_(ctx), max_pairs_(max_pairs), max_total_((size_t)max_pairs * max_pts_per_pair) {
		check(bt_ransac_reserve(ctx, max_pairs, max_pts_per_pair, max_trials), "bt_ransac_reserve");
		check(bt_dev_alloc(&d_ids_, sizeof(int32_t) * max_total_), "bt_dev_alloc");
		check(bt_dev_alloc(&d_cnt_, sizeof(int32_t) * (size_t)max_pairs), "bt_dev_alloc");
		ids_.resize(max_total_); cnt_.resize(max_pairs);
	}
	~RansacGpu() { bt_dev_free(d_ids_); bt_dev_free(d_cnt_); }
	RansacGpu(const RansacGpu&) = delete;
	RansacGpu& operator=(const RansacGpu&) = delete;
	template <class Float4T>
	void ransacMultiPairGPU(const std::vector<Float4T*>& ptsA, const std::vector<Float4T*>& ptsB, const std::vector<int>& n_pts,
	                        int n_trials, float dist_thres, std::vector<std::vector<int>>& inlier_ids, void* stream = nullptr) {
		const int n = (int)ptsA.size();
		inlier_ids.assign(n, {});
		if (n == 0) return;
		size_t total = 0;
		for (int v : n_pts) total += (size_t)v;
		if (n > max_pairs_ || total > max_total_) throw std::runtime_error("RansacGpu: more pairs / points than the object was created for");
		a_.resize(n); b_.resize(n);
		for (int p = 0; p < n; p++) { a_[p] = reinterpret_cast<const float*>(ptsA[p]); b_[p] = reinterpret_cast<const float*>(ptsB[p]); }
		check(bt_ransac_pairs(ctx_, n, a_.data(), b_.data(), n_pts.data(), n_trials, dist_thres, 0, (int32_t*)d_ids_, (int32_t*)d_cnt_, stream), "bt_ransac_pairs");
		check(bt_memcpy_d2h(cnt_.data(), d_cnt_, sizeof(int32_t) * n, stream), "bt_memcpy_d2h");
		if (total) check(bt_memcpy_d2h(ids_.data(), d_ids_, sizeof(int32_t) * total, stream), "bt_memcpy_d2h");
		size_t off = 0;
		for (int p = 0; p < n; p++) { inlier_ids[p].assign(ids_.begin() + off, ids_.begin() + off + cnt_[p]); off += (size_t)n_pts[p]; }
	}
private:
	static void check(int rc, const char* what) { if (rc != BT_OK) throw std::runtime_error(std::string(what) + ": " + bt_last_error()); }
	bt_ctx* ctx_; int max_pairs_; size_t max_total_;
	void *d_ids_ = nullptr, *d_cnt_ = nullptr;
	std::vector<int32_t> ids_, cnt_;
	std::vector<const float*> a_, b_;
};
// Free-function form with exactly the reference's name: creates a RansacGpu sized for this call (convenient, but it allocates - hold
// a RansacGpu in SiftManager instead, INTEGRATION.md).
template <class Float4T>
inline void ransacMultiPairGPU(bt_ctx* ctx, const std::vector<Float4T*>& ptsA, const std::vector<Float4T*>& ptsB, const std::vector<int>& n_pts,
                               int n_trials, float dist_thres, std::vector<std::vector<int>>& inlier_ids, void* stream = nullptr) {
	inlier_ids.assign(ptsA.size(), {});
	if (ptsA.empty()) return;
	int maxp = 1;
	for (int v : n_pts) if (v > maxp) maxp = v;
	RansacGpu r(ctx, (int)ptsA.size(), maxp, n_trials);
	r.ransacMultiPairGPU(ptsA, ptsB, n_pts, n_trials, dist_thres, inlier_ids, stream);
}

// ---- Frame::processDepth + Frame::depthToCloudAndNormals (/root/reference/src/Frame.cpp:152-233) ----------------------------------
struct BtDepthConfig {            // depth_processing.* of config_nocs.yml, same names
	float erode_radius = 1, erode_diff = 0.001f, erode_ratio = 0.8f;
	int bf_radius = 2; float sigma_D = 2.f, sigma_R = 100000.f;
	bt_depth_params to_params() const { bt_depth_params p; p.erode_radius = (int)erode_radius; p.erode_diff = erode_diff; p.erode_ratio = erode_ratio;
		p.bf_radius = bf_radius; p.sigma_D = sigma_D; p.sigma_R = sigma_R; return p; }
};
// raw depth (device, metres) -> Frame::_depth_gpu, Frame::_normal_gpu and, if wanted, the camera-space point map that the
// reference copies to the host for its PCL cloud (xyz_gpu may be nullptr).  One fused kernel; depth_gpu != depth_raw_gpu.
template <class Float4T, class Mat3>
inline void processDepthAndNormals(bt_ctx* ctx, const float* depth_raw_gpu, float* depth_gpu, Float4T* normal_gpu, Float4T* xyz_gpu, int H, int W, const Mat3& K,
                                   const BtDepthConfig& cfg, void* stream = nullptr) {
	const bt_depth_params prm = cfg.to_params();
	const float* in[1] = { depth_raw_gpu }; float* out[1] = { depth_gpu };
	float* nrm[1] = { reinterpret_cast<float*>(normal_gpu) }; float* xyz[1] = { reinterpret_cast<float*>(xyz_gpu) };
	if (bt_frames_preprocess(ctx, 1, in, H, W, K(0, 0), K(1, 1), K(0, 2), K(1, 2), &prm, out, xyz_gpu ? xyz : nullptr, nrm, stream) != BT_OK)
		throw std::runtime_error(std::string("bt_frames_preprocess: ") + bt_last_error());
}

// ---- Frame::segmentationByMaskFile + invalidatePixelsByMask (Frame.cpp:236-374) on top of the front end -----------------------------
// mask_gpu: the mask PNG's bytes (device uint8 H*W); mode: BT_MASK_LARGEST_HULL when data_dir contains "NOCS", else BT_MASK_AS_IS.
// Writes the masked maps, fg_gpu (= Frame::_fg_mask, device uint8 H*W, not mask_gpu) and roi_gpu (device int32[4], kept for
// lfnetRequest), then reads the ROI back into roi (Vector4-like: roi(0..3) = umin, umax, vmin, vmax; waits for the stream).
template <class Float4T, class Mat3, class Vec4>
inline void processDepthNormalsAndMask(bt_ctx* ctx, const float* depth_raw_gpu, const uint8_t* mask_gpu, int mode, float* depth_gpu, Float4T* normal_gpu,
                                       Float4T* xyz_gpu, uint8_t* fg_gpu, int32_t* roi_gpu, int H, int W, const Mat3& K, const BtDepthConfig& cfg, Vec4& roi,
                                       void* stream = nullptr) {
	const bt_depth_params prm = cfg.to_params();
	const float* in[1] = { depth_raw_gpu }; float* out[1] = { depth_gpu };
	float* nrm[1] = { reinterpret_cast<float*>(normal_gpu) }; float* xyz[1] = { reinterpret_cast<float*>(xyz_gpu) };
	const uint8_t* msk[1] = { mask_gpu }; uint8_t* fg[1] = { fg_gpu };
	if (bt_frames_preprocess_masked(ctx, 1, in, msk, mode, H, W, K(0, 0), K(1, 1), K(0, 2), K(1, 2), &prm, out, xyz_gpu ? xyz : nullptr, nrm, fg, roi_gpu, stream) != BT_OK)
		throw std::runtime_error(std::string("bt_frames_preprocess_masked: ") + bt_last_error());
	int32_t r[4];
	if (bt_memcpy_d2h(r, roi_gpu, sizeof r, stream) != BT_OK) throw std::runtime_error(std::string("bt_memcpy_d2h: ") + bt_last_error());
	for (int i = 0; i < 4; i++) roi(i) = r[i];
}
// Lfnet::detectFeature's request image (FeatureManager.cpp:813-858, rot_deg = 0) from processDepthNormalsAndMask's fg / roi:
// request_gpu (device uint8 400*400*3) receives the BGR bytes of the second message part; untouched when the ROI fails the gate.
inline void lfnetRequest(bt_ctx* ctx, const uint8_t* color_gpu, const uint8_t* fg_gpu, const int32_t* roi_gpu, int H, int W, uint8_t* request_gpu,
                         void* stream = nullptr) {
	const uint8_t* col[1] = { color_gpu }; const uint8_t* fg[1] = { fg_gpu }; uint8_t* out[1] = { request_gpu };
	if (bt_lfnet_request(ctx, 1, col, fg, roi_gpu, H, W, out, stream) != BT_OK)
		throw std::runtime_error(std::string("bt_lfnet_request: ") + bt_last_error());
}

// ---- the two knnMatch calls of SiftManager::findCorresbyNN (/root/reference/src/FeatureManager.cpp:271-273) in one call --------
// desA/desB: device CV_32F descriptor matrices (GpuMat::data, rows, step).  DMatchT needs queryIdx, trainIdx, distance (cv::DMatch).
// The device result buffers belong to the object (sized once for max_feats x k), nothing is allocated per call.
class KnnMatcherGpu {
public:
	KnnMatcherGpu(bt_ctx* ctx, int max_feats, int dim = 256, int k = 5) : ctx_(ctx), max_feats_(max_feats), dim_(dim), k_(k) {
		check(bt_matcher_reserve(ctx, 1, max_feats, dim), "bt_matcher_reserve");
		const size_t e = (size_t)max_feats * k;
		check(bt_dev_alloc(&iab_, 4 * e), "bt_dev_alloc"); check(bt_dev_alloc(&dab_, 4 * e), "bt_dev_alloc");
		check(bt_dev_alloc(&iba_, 4 * e), "bt_dev_alloc"); check(bt_dev_alloc(&dba_, 4 * e), "bt_dev_alloc");
		hi_[0].resize(e); hi_[1].resize(e); hd_[0].resize(e); hd_[1].resize(e);
	}
	~KnnMatcherGpu() { bt_dev_free(iab_); bt_dev_free(dab_); bt_dev_free(iba_); bt_dev_free(dba_); }
	KnnMatcherGpu(const KnnMatcherGpu&) = delete;
	KnnMatcherGpu& operator=(const KnnMatcherGpu&) = delete;
	template <class DMatchT>
	void knnMatchBothDirections(const float* desA, int nA, size_t stepA, const float* desB, int nB, size_t stepB,
	                            std::vector<std::vector<DMatchT>>& matchesAB, std::vector<std::vector<DMatchT>>& matchesBA, void* stream = nullptr) {
		if (nA > max_feats_ || nB > max_feats_) throw std::runtime_error("KnnMatcherGpu: more features than the object was created for");
		bt_desc_view A{}; A.dev = desA; A.n = nA; A.dim = dim_; A.pitch_bytes = stepA;
		bt_desc_view B{}; B.dev = desB; B.n = nB; B.dim = dim_; B.pitch_bytes = stepB;
		check(bt_knn_match_pairs(ctx_, 1, &A, &B, k_, (int32_t*)iab_, (float*)dab_, (int32_t*)iba_, (float*)dba_, stream), "bt_knn_match_pairs");
		if (nA) { check(bt_memcpy_d2h(hi_[0].data(), iab_, 4 * (size_t)nA * k_, stream), "bt_memcpy_d2h"); check(bt_memcpy_d2h(hd_[0].data(), dab_, 4 * (size_t)nA * k_, stream), "bt_memcpy_d2h"); }
		if (nB) { check(bt_memcpy_d2h(hi_[1].data(), iba_, 4 * (size_t)nB * k_, stream), "bt_memcpy_d2h"); check(bt_memcpy_d2h(hd_[1].data(), dba_, 4 * (size_t)nB * k_, stream), "bt_memcpy_d2h"); }
		fill(nA, hi_[0], hd_[0], matchesAB); fill(nB, hi_[1], hd_[1], matchesBA);
	}
private:
	static void check(int rc, const char* what) { if (rc != BT_OK) throw std::runtime_error(std::string(what) + ": " + bt_last_error()); }
	template <class DMatchT>
	void fill(int n, const std::vector<int32_t>& idx, const std::vector<float>& dist, std::vector<std::vector<DMatchT>>& out) const {
		out.assign(n, {});
		for (int q = 0; q < n; q++)
			for (int j = 0; j < k_; j++) {
				if (idx[(size_t)q * k_ + j] < 0) break;          // fewer than k train rows
				DMatchT m{}; m.queryIdx = q; m.trainIdx = idx[(size_t)q * k_ + j]; m.distance = dist[(size_t)q * k_ + j];
				out[q].push_back(m);
			}
	}
	bt_ctx* ctx_; int max_feats_, dim_, k_;
	void *iab_ = nullptr, *dab_ = nullptr, *iba_ = nullptr, *dba_ = nullptr;
	std::vector<int32_t> hi_[2]; std::vector<float> hd_[2];
};
// Free-function form: creates a KnnMatcherGpu sized for this call (it allocates - hold a KnnMatcherGpu in SiftManager instead).
template <class DMatchT>
inline void knnMatchBothDirections(bt_ctx* ctx, const float* desA, int nA, size_t stepA, const float* desB, int nB, size_t stepB, int dim, int k,
                                   std::vector<std::vector<DMatchT>>& matchesAB, std::vector<std::vector<DMatchT>>& matchesBA, void* stream = nullptr) {
	KnnMatcherGpu m(ctx, (nA > nB ? nA : nB) > 0 ? (nA > nB ? nA : nB) : 1, dim, k);
	m.knnMatchBothDirections(desA, nA, stepA, desB, nB, stepB, matchesAB, matchesBA, stream);
}

// ---- Bundler::processNewFrame (the reference's src/Bundler.cpp:56-183) as one object over bt_tracker_* -------------------------------------
// The reference's call is split where it asks the LF-Net server for features (Lfnet::detectFeature, Bundler.cpp:108): beginFrame segments the
// frame and returns the request image, the caller does the ZMQ round trip (bt_lfnet_parse_reply maps the keypoints back) and calls endFrame,
// or dropFrame when detection threw.  Statuses are Frame::_status values (BT_FRAME_OTHER / FAIL / NO_BA); poses are cam->model through
// operator()(row, col) (Eigen::Matrix4f works); endFrame's pose is what Bundler::saveNewframeResult records for the frame.
class BundlerGpu {
public:
	explicit BundlerGpu(const bt_tracker_params& p, int device = 0) { check(bt_tracker_create(&t_, device, &p), "bt_tracker_create"); }
	~BundlerGpu() { bt_tracker_destroy(t_); }
	BundlerGpu(const BundlerGpu&) = delete;
	BundlerGpu& operator=(const BundlerGpu&) = delete;

	// loader_id / first_pose (nullptr: identity) name the frame when the tracker holds none.  roi (optional): Frame::_roi.
	template <class Mat4>
	int beginFrame(int loader_id, const Mat4* first_pose, const float* depth_raw_gpu, const uint8_t* mask_gpu, const uint8_t* color_gpu, uint8_t* request_gpu,
	               int32_t* roi = nullptr, void* stream = nullptr) {
		float fp[16];
		if (first_pose) to_flat(*first_pose, fp);
		int st = -1;
		check(bt_tracker_begin_frame(t_, loader_id, first_pose ? fp : nullptr, depth_raw_gpu, mask_gpu, color_gpu, request_gpu, roi, &st, stream), "bt_tracker_begin_frame");
		return st;
	}
	// kpts: n x (x, y) image pixels; desc_gpu: n x 256 device floats, desc_step bytes per row (GpuMat::step; 0 = packed)
	template <class Mat4>
	int endFrame(const float* kpts, int n, const float* desc_gpu, size_t desc_step, Mat4& pose, void* stream = nullptr) {
		bt_desc_view d{}; d.dev = desc_gpu; d.n = n; d.dim = 256; d.pitch_bytes = desc_step;
		float fp[16];
		int st = -1;
		check(bt_tracker_end_frame(t_, kpts, n, &d, fp, &st, stream), "bt_tracker_end_frame");
		from_flat(fp, pose);
		return st;
	}
	template <class Mat4>
	void dropFrame(Mat4& pose) {
		float fp[16];
		check(bt_tracker_drop_frame(t_, fp), "bt_tracker_drop_frame");
		from_flat(fp, pose);
	}
	// every frame alive, oldest first
	template <class Mat4, class Alloc>
	void state(std::vector<int>& ids, std::vector<Mat4, Alloc>& poses, std::vector<bool>& is_keyframe) {
		int n = 0;
		const int rc = bt_tracker_state(t_, nullptr, nullptr, nullptr, 0, &n);      // the count (BT_ERR_CAPACITY unless no frame is alive)
		if (rc != BT_ERR_CAPACITY) check(rc, "bt_tracker_state");
		std::vector<int32_t> id(n), kf(n);
		std::vector<float> p(16 * (size_t)n);
		check(bt_tracker_state(t_, id.data(), p.data(), kf.data(), n, &n), "bt_tracker_state");
		ids.assign(id.begin(), id.end());
		poses.resize(n);
		is_keyframe.resize(n);
		for (int k = 0; k < n; k++) { from_flat(&p[16 * (size_t)k], poses[k]); is_keyframe[k] = kf[k] != 0; }
	}
	bt_tracker* handle() { return t_; }

private:
	static void check(int rc, const char* what) { if (rc != BT_OK) throw std::runtime_error(std::string(what) + ": " + bt_last_error()); }
	template <class Mat4> static void to_flat(const Mat4& m, float* f) { for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) f[4 * r + c] = m(r, c); }
	template <class Mat4> static void from_flat(const float* f, Mat4& m) { for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) m(r, c) = f[4 * r + c]; }
	bt_tracker* t_ = nullptr;
};
