// TEST INFRASTRUCTURE ONLY (oracle/_ref): the reference's logger for its PNG slice writers. info() keeps the text it is given (the
// counts save_density_grid_to_png logs, marching_cubes.cu:968-971) in tlog::info_text(); everything else is a sink.
#pragma once
#include <cstddef>
#include <sstream>
#include <string>
namespace tlog {
inline std::string& info_text() { static std::string s; return s; }
struct Sink { template <typename T> Sink& operator<<(const T&) { return *this; } };
struct Info {
	std::ostringstream os;
	template <typename T> Info& operator<<(const T& v) { os << v; return *this; }
	~Info() { info_text() += os.str() + "\n"; }
};
inline Info info() { return {}; }
inline Sink warning() { return {}; } inline Sink error() { return {}; } inline Sink success() { return {}; } inline Sink debug() { return {}; } inline Sink none() { return {}; }
struct Progress { void update(size_t) {} };
inline Progress progress(size_t) { return {}; }
}  // namespace tlog
