// Drives BundlerGpu (bundletrack_b200/hostcpp/bt_optimizer.hpp) over a sequence written by tests/test_tracker_gpu.py, with the NOCS
// configuration and a column-major Mat4, and writes per frame: status (int32), pose (16 floats, row-major), the 400x400x3 request image.
#include "bundletrack_b200/hostcpp/bt_optimizer.hpp"
#include <cstdio>
#include <cmath>

struct Mat4 { float m[16]; float& operator()(int r, int c) { return m[c * 4 + r]; } float operator()(int r, int c) const { return m[c * 4 + r]; } };

template <class T> static void rd(FILE* f, T* p, size_t n) { if (fread(p, sizeof(T), n, f) != n) throw std::runtime_error("short input"); }

int main(int argc, char** argv) {
	try {
		FILE* in = fopen(argv[1], "rb");
		FILE* out = fopen(argv[2], "wb");
		if (!in || !out) return 2;
		int32_t hdr[4]; rd(in, hdr, 4);
		const int n_frames = hdr[0], H = hdr[1], W = hdr[2], max_feats = hdr[3];
		float K[4]; rd(in, K, 4);
		bt_tracker_params p{};                       // config_nocs.yml (the library's defaults when no yml is given)
		p.H = H; p.W = W; p.fx = K[0]; p.fy = K[1]; p.cx = K[2]; p.cy = K[3];
		p.max_feats = max_feats; p.max_frames_alive = 24; p.mask_mode = BT_MASK_LARGEST_HULL;
		p.depth = BtDepthConfig().to_params(); p.solver = BtSolverConfig().to_params();
		p.prune.max_dist_no_neighbor = 0.02f; p.prune.cos_max_normal_no_neighbor = (float)std::cos(45.0 / 180.0 * M_PI);
		p.prune.max_dist_neighbor = 10000.f; p.prune.cos_max_normal_neighbor = (float)std::cos(180.0 / 180.0 * M_PI);
		p.ransac_trials = 2000; p.ransac_inlier_dist = 0.005f;
		p.window_size = 2; p.max_BA_frames = 15; p.min_fm_edges_newframe = 10; p.min_feat_num = 0; p.min_rot_deg = 10.f;
		BundlerGpu bundler(p);
		const size_t hw = (size_t)H * W;
		std::vector<float> depth(hw), kpts(2 * (size_t)max_feats), desc(256 * (size_t)max_feats);
		std::vector<uint8_t> mask(hw), colour(3 * hw), request(400 * 400 * 3);
		void *d_depth, *d_mask, *d_colour, *d_req, *d_desc;
		bt_dev_alloc(&d_depth, 4 * hw); bt_dev_alloc(&d_mask, hw); bt_dev_alloc(&d_colour, 3 * hw); bt_dev_alloc(&d_req, request.size());
		bt_dev_alloc(&d_desc, 4 * desc.size());
		for (int k = 0; k < n_frames; k++) {
			rd(in, depth.data(), hw); rd(in, mask.data(), hw); rd(in, colour.data(), 3 * hw);
			int32_t n; rd(in, &n, 1);
			if (n >= 0) { rd(in, kpts.data(), 2 * (size_t)n); rd(in, desc.data(), 256 * (size_t)n); }
			bt_memcpy_h2d(d_depth, depth.data(), 4 * hw, nullptr); bt_memcpy_h2d(d_mask, mask.data(), hw, nullptr);
			bt_memcpy_h2d(d_colour, colour.data(), 3 * hw, nullptr);
			std::vector<uint8_t> zero(request.size(), 0);
			bt_memcpy_h2d(d_req, zero.data(), zero.size(), nullptr);
			Mat4 pose{}; for (int i = 0; i < 4; i++) pose(i, i) = 1.f;
			int st = bundler.beginFrame<Mat4>(0, nullptr, (const float*)d_depth, (const uint8_t*)d_mask, (const uint8_t*)d_colour, (uint8_t*)d_req);
			if (st == BT_FRAME_OTHER) {
				if (n < 0) { bundler.dropFrame(pose); st = BT_FRAME_FAIL; }
				else {
					bt_memcpy_h2d(d_desc, desc.data(), 4 * 256 * (size_t)n, nullptr);
					st = bundler.endFrame(kpts.data(), n, (const float*)d_desc, 0, pose);
				}
			}
			bt_memcpy_d2h(request.data(), d_req, request.size(), nullptr);
			float flat[16];
			for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) flat[4 * r + c] = pose(r, c);
			fwrite(&st, 4, 1, out); fwrite(flat, 4, 16, out); fwrite(request.data(), 1, request.size(), out);
		}
		std::vector<int> ids; std::vector<Mat4> poses; std::vector<bool> kf;
		bundler.state(ids, poses, kf);
		bt_dev_free(d_depth); bt_dev_free(d_mask); bt_dev_free(d_colour); bt_dev_free(d_req); bt_dev_free(d_desc);
		fclose(in); fclose(out);
	} catch (const std::exception& e) { std::fprintf(stderr, "%s\n", e.what()); return 1; }
	return 0;
}
