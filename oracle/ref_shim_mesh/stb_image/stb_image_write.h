// Stand-in for stb_image_write (absent submodule): save_mesh only calls stbi_write_tga for the UV-unwrap texture, which the parity
// tests do not request. Writing nothing is reported as failure (0), like stb on an I/O error. TEST ONLY.
#pragma once
inline int stbi_write_tga(const char*, int, int, int, const void*) { return 0; }
