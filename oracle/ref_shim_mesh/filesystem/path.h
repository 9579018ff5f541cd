// Stand-in for the filesystem/path.h submodule (absent here), for the reference's save_mesh (marching_cubes.cu:760-896): only what it
// calls — fs::path(name).extension() (the text after the file name's last '.', without the dot) and with_extension().str(). TEST ONLY.
#pragma once
#include <string>

namespace filesystem {
class path {
	std::string s_;

public:
	path(const std::string& s) : s_(s) {}
	path(const char* s) : s_(s) {}
	std::string filename() const { const size_t k = s_.find_last_of('/'); return k == std::string::npos ? s_ : s_.substr(k + 1); }
	std::string extension() const { const std::string n = filename(); const size_t k = n.find_last_of('.'); return k == std::string::npos ? "" : n.substr(k + 1); }
	path with_extension(const std::string& ext) const { const size_t k = s_.find_last_of('.'); return path((k == std::string::npos ? s_ : s_.substr(0, k)) + ext); }
	std::string str() const { return s_; }
};
}  // namespace filesystem
