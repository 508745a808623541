// Tracks a sequence with BundlerGpu and LfnetGpu (bundletrack_b200/hostcpp/bt_optimizer.hpp), the C++ loop of INTEGRATION.md §7:
// beginFrame -> LfnetGpu::detectFeature -> endFrame, or dropFrame when detection throws.  Written by tests/test_lfnet_file_gpu.py.
// argv: input file, output directory (with poses/), weights file, second weights file (used for the frames the input marks).
// Input: int32 n_frames, H, W, sizeof(bt_tracker_params), the params; per frame: int32 id length, the id, int32 use_second, float first_pose[16]
// (row-major), uint16 depth H x W (millimetres), uint8 mask H x W, uint8 colour H x W x 3.  Output: <out>/poses/<id>.txt per frame
// (saveNewframePose) and <out>/status.bin, one int32 status per frame.
#include "bundletrack_b200/hostcpp/bt_optimizer.hpp"
#include <cstdio>

struct Mat4 { float m[16]; float& operator()(int r, int c) { return m[c * 4 + r]; } float operator()(int r, int c) const { return m[c * 4 + r]; } };
struct KeyPoint { struct { float x, y; } pt; float size; };        // cv::KeyPoint's members that LfnetGpu sets

template <class T> static void rd(FILE* f, T* p, size_t n) { if (fread(p, sizeof(T), n, f) != n) throw std::runtime_error("short input"); }

int main(int argc, char** argv) {
	try {
		if (argc != 5) return 2;
		FILE* in = fopen(argv[1], "rb");
		const std::string out_dir = argv[2];
		FILE* st_out = fopen((out_dir + "/status.bin").c_str(), "wb");
		if (!in || !st_out) return 2;
		int32_t hdr[4]; rd(in, hdr, 4);
		const int n_frames = hdr[0], H = hdr[1], W = hdr[2];
		if (hdr[3] != (int32_t)sizeof(bt_tracker_params)) throw std::runtime_error("bt_tracker_params size differs");
		bt_tracker_params p; rd(in, &p, 1);
		BundlerGpu bundler(p);
		LfnetGpu lfnet(argv[3]), lfnet_second(argv[4]);
		const size_t hw = (size_t)H * W;
		std::vector<uint16_t> depth(hw);
		std::vector<uint8_t> mask(hw), colour(3 * hw);
		void *d_depth, *d_mask, *d_colour, *d_req;
		bt_dev_alloc(&d_depth, 2 * hw); bt_dev_alloc(&d_mask, hw); bt_dev_alloc(&d_colour, 3 * hw); bt_dev_alloc(&d_req, 400 * 400 * 3);
		std::vector<KeyPoint> kpts;
		std::vector<float> xy;
		for (int k = 0; k < n_frames; k++) {
			int32_t len; rd(in, &len, 1);
			std::string id(len, ' '); rd(in, &id[0], len);
			int32_t second; rd(in, &second, 1);
			float fp[16]; rd(in, fp, 16);
			Mat4 first{};
			for (int r = 0; r < 4; r++) for (int c = 0; c < 4; c++) first(r, c) = fp[4 * r + c];
			rd(in, depth.data(), hw); rd(in, mask.data(), hw); rd(in, colour.data(), 3 * hw);
			bt_memcpy_h2d(d_depth, depth.data(), 2 * hw, nullptr); bt_memcpy_h2d(d_mask, mask.data(), hw, nullptr);
			bt_memcpy_h2d(d_colour, colour.data(), 3 * hw, nullptr);
			Mat4 pose{};
			int frame_id = -1;
			int32_t roi[4];
			int st = bundler.beginFrame<Mat4>(k, &first, (const uint16_t*)d_depth, (const uint8_t*)d_mask, (const uint8_t*)d_colour, (uint8_t*)d_req,
			                                  frame_id, pose, roi);
			if (st == BT_FRAME_OTHER) {
				bt_desc_view desc{};
				int n = 0;
				try {
					n = (second ? lfnet_second : lfnet).detectFeature((const uint8_t*)d_req, roi, kpts, desc);
				} catch (const std::exception& e) {
					std::fprintf(stderr, "frame %s: %s\n", id.c_str(), e.what());
				}
				if (n == 0) { bundler.dropFrame(pose); st = BT_FRAME_FAIL; }
				else {
					xy.resize(2 * (size_t)n);
					for (int j = 0; j < n; j++) { xy[2 * j] = kpts[j].pt.x; xy[2 * j + 1] = kpts[j].pt.y; }
					st = bundler.endFrame(xy.data(), n, desc.dev, desc.pitch_bytes, pose);
				}
			}
			saveNewframePose(out_dir + "/poses/" + id + ".txt", pose);
			fwrite(&st, 4, 1, st_out);
		}
		bt_dev_free(d_depth); bt_dev_free(d_mask); bt_dev_free(d_colour); bt_dev_free(d_req);
		fclose(in); fclose(st_out);
	} catch (const std::exception& e) { std::fprintf(stderr, "%s\n", e.what()); return 1; }
	return 0;
}
