// The saved pose-graph format of savePoseGraph / loadPoseGraph (pose_graph/src/pose_graph.cpp:697-870), read and written
// by vp_save / vp_load (pose_graph.cpp) and, compiled with g++, by tests/hostlib/pg_map_host.cpp.  For a prefix P:
//   P + "pose_graph.txt"           one line per key frame, " %d %f x14 %d %f x8 %d\n": index, stamp, VIO T, PG T,
//                                  VIO Q (w x y z), PG Q (w x y z), loop_index, loop_info (8), keypoint count
//   P + <index> + "_keypoints.txt" "%f %f %f %f\n" per corner: pixel x y, normalised x y
//   P + <index> + "_briefdes.dat"  one line per descriptor as boost::dynamic_bitset's operator<< writes it: 256 '0' / '1'
//                                  characters, the highest bit first (character j is bit 255 - j), then '\n'
// Bit i of a descriptor is BRIEF pattern pair i, in word i / 64 (lv_layout.h).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace vb {

struct MapKeyFrame {
    int index = 0;
    double stamp = 0;
    double vio_T[3] = {}, pg_T[3] = {}, vio_Q[4] = {}, pg_Q[4] = {};  // quaternions w x y z
    int loop_index = -1;
    double loop_info[8] = {};
    int n_kp = 0;                 // the keypoint count of the pose_graph.txt row
    std::vector<float> kp, kpn;   // 2 n_kp each (only when the points are read or written)
    std::vector<uint64_t> desc;   // 4 n_kp
};

// Writes the key frames under prefix.  with_points = false writes every key frame with a count of 0 and two empty
// files.  Returns 0, or VP_ERR_INVALID with err naming the file that could not be written.
int map_write(const std::string& prefix, const std::vector<MapKeyFrame>& kfs, bool with_points, std::string* err);

// Reads the key frames under prefix; with_points also reads each key frame's keypoints and descriptors.  Rows must be
// numbered 0, 1, 2, ... and every loop_index must name an earlier row.  More than max_keyframes rows, or (with_points) a
// count above max_corners, is VP_ERR_CAPACITY; a missing file, a truncated or unparsable line, a descriptor line that is
// not 256 '0' / '1' characters or a count that does not match its files is VP_ERR_INVALID.  err names the file and line.
// On error *out is left as it was.
int map_read(const std::string& prefix, bool with_points, int max_keyframes, int max_corners, std::vector<MapKeyFrame>* out,
             std::string* err);

}  // namespace vb
