// Stand-in for stb_image_write (absent submodule) for the reference's PNG slice writers (marching_cubes.cu:898-1015): stbi_write_png
// records the file name, size, channel count and pixels instead of writing a file; ref_slices_driver_cuda.cu hands the records out.
// TEST INFRASTRUCTURE ONLY.
#pragma once
#include <cstdint>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

struct StbPngRecord {
	std::string filename;
	int w, h, comp;
	std::vector<uint8_t> pixels;  // w * h * comp bytes, rows packed
};
inline std::vector<StbPngRecord>& stb_png_records() { static std::vector<StbPngRecord> r; return r; }
inline std::mutex& stb_png_mutex() { static std::mutex m; return m; }

inline int stbi_write_png(const char* filename, int w, int h, int comp, const void* data, int stride_in_bytes) {
	StbPngRecord r{filename, w, h, comp, std::vector<uint8_t>((size_t)w * h * comp)};
	for (int y = 0; y < h; ++y) std::memcpy(r.pixels.data() + (size_t)y * w * comp, (const uint8_t*)data + (size_t)y * stride_in_bytes, (size_t)w * comp);
	std::lock_guard<std::mutex> lock(stb_png_mutex());
	stb_png_records().push_back(std::move(r));
	return 1;
}
