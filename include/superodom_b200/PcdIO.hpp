// =============================================================================
// superodom_b200/PcdIO.hpp -- dependency-free reader for the prior-map file of
// localization mode.  Upstream: utils::readPointCloud(config_.map_dir, laserCloudPrior)
// (super_odometry/src/utils/superodom_utils.cpp:16-33, a thin wrapper over
// pcl::PCDReader::read) followed by slam.localMap.addSurfPointCloud(*laserCloudPrior)
// (src/LaserMapping/laserMapping.cpp:161-173).  PCL is not a dependency of this
// library, so the PCD v0.5-v0.7 container (the published file-format description:
// header keywords VERSION FIELDS SIZE TYPE COUNT WIDTH HEIGHT VIEWPOINT POINTS
// DATA; DATA ascii | binary | binary_compressed, the latter LZF-compressed and
// stored field by field) is parsed here.  Fields are matched by name: x, y, z and
// intensity are taken (any of the PCD scalar types, converted to float), every
// other field is skipped, a missing intensity reads as 0 -- what PCDReader does
// for pcl::PointXYZI.  Same return convention as upstream: true / false + a
// message on stderr, never throws.
// =============================================================================
#pragma once
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <type_traits>
#include <vector>

namespace super_odometry {
namespace b200 {
namespace pcd_detail {

struct Field { std::string name; int size = 4; char type = 'F'; int count = 1; size_t offset = 0; };

inline double read_scalar(const unsigned char* p, char type, int size) {
    switch (type) {
        case 'F': if (size == 4) { float v; std::memcpy(&v, p, 4); return v; } if (size == 8) { double v; std::memcpy(&v, p, 8); return v; } break;
        case 'U': if (size == 1) return *p; if (size == 2) { uint16_t v; std::memcpy(&v, p, 2); return v; } if (size == 4) { uint32_t v; std::memcpy(&v, p, 4); return v; }
                  if (size == 8) { uint64_t v; std::memcpy(&v, p, 8); return double(v); } break;
        case 'I': if (size == 1) return *reinterpret_cast<const int8_t*>(p); if (size == 2) { int16_t v; std::memcpy(&v, p, 2); return v; }
                  if (size == 4) { int32_t v; std::memcpy(&v, p, 4); return v; } if (size == 8) { int64_t v; std::memcpy(&v, p, 8); return double(v); } break;
        default: break;
    }
    return 0.0;
}

// LZF decompression (the format PCL's lzfDecompress reads: control byte < 32 = literal run of ctrl+1 bytes, otherwise a
// back-reference of length (ctrl >> 5) + 2 (7 = extended by the next byte) at distance ((ctrl & 31) << 8 | next) + 1).
inline bool lzf_decompress(const unsigned char* in, size_t in_len, unsigned char* out, size_t out_len) {
    size_t ip = 0, op = 0;
    while (ip < in_len) {
        unsigned ctrl = in[ip++];
        if (ctrl < 32) {
            ++ctrl;
            if (op + ctrl > out_len || ip + ctrl > in_len) return false;
            std::memcpy(out + op, in + ip, ctrl);
            ip += ctrl; op += ctrl;
        } else {
            unsigned len = ctrl >> 5;
            if (len == 7) { if (ip >= in_len) return false; len += in[ip++]; }
            if (ip >= in_len) return false;
            const size_t dist = (size_t(ctrl & 31) << 8 | in[ip++]) + 1;
            len += 2;
            if (dist > op || op + len > out_len) return false;
            for (unsigned k = 0; k < len; ++k, ++op) out[op] = out[op - dist];      // may overlap: byte by byte
        }
    }
    return op == out_len;
}

}  // namespace pcd_detail

// Reads `file_path` into *cloud_out (cleared first).  CloudPtr: anything with ->points (std::vector of a point holding float
// x, y, z, intensity) -- pcl::PointCloud<pcl::PointXYZI>::Ptr upstream.  Unorganised or organised files alike end up as a flat
// list of WIDTH*HEIGHT (or POINTS) points, non-finite ones included (PCDReader keeps them; the map insert drops them).
template <class CloudPtr>
inline bool readPointCloud(const std::string& file_path, CloudPtr cloud_out) {
    using namespace pcd_detail;
    using PointT = typename std::decay<decltype(cloud_out->points[0])>::type;
    std::ifstream f(file_path.c_str(), std::ios::binary);
    if (!f.good()) { std::cerr << "Error: File does not exist: " << file_path << std::endl; return false; }
    std::vector<Field> fields;
    size_t width = 0, height = 1, points = 0;
    bool have_points = false;
    std::string data_mode, line;
    while (std::getline(f, line)) {
        if (!line.empty() && line.back() == '\r') line.pop_back();
        if (line.empty() || line[0] == '#') continue;
        std::istringstream ls(line);
        std::string key;
        ls >> key;
        if (key == "FIELDS" || key == "COLUMNS") { std::string n; while (ls >> n) { Field fl; fl.name = n; fields.push_back(fl); } }
        else if (key == "SIZE") { for (auto& fl : fields) ls >> fl.size; }
        else if (key == "TYPE") { for (auto& fl : fields) ls >> fl.type; }
        else if (key == "COUNT") { for (auto& fl : fields) ls >> fl.count; }
        else if (key == "WIDTH") ls >> width;
        else if (key == "HEIGHT") ls >> height;
        else if (key == "POINTS") { ls >> points; have_points = true; }
        else if (key == "DATA") { ls >> data_mode; break; }
    }
    if (fields.empty() || data_mode.empty()) { std::cerr << "Error reading PCD file: " << file_path << " (no FIELDS / DATA header)" << std::endl; return false; }
    if (!have_points) points = width * height;
    if (points > (size_t(1) << 31)) { std::cerr << "Error reading PCD file: " << file_path << " (implausible point count)" << std::endl; return false; }
    size_t rec = 0;
    for (auto& fl : fields) {
        // untrusted header: element sizes PCL knows (1/2/4/8), at least one element per field (a COUNT 0 field would add no bytes to
        // the record while read_scalar still reads `size` bytes from it), bounded counts so that the record size cannot wrap
        if (!(fl.size == 1 || fl.size == 2 || fl.size == 4 || fl.size == 8) || fl.count < 1 || fl.count > 4096) {
            std::cerr << "Error reading PCD file: " << file_path << " (bad SIZE / COUNT)" << std::endl; return false;
        }
        fl.offset = rec; rec += size_t(fl.size) * size_t(fl.count);
    }
    if (rec == 0 || rec > (size_t(1) << 20) || points > (size_t(1) << 40) / rec) { std::cerr << "Error reading PCD file: " << file_path << " (implausible record / cloud size)" << std::endl; return false; }
    // the body cannot be larger than what is left of the file: checked before any allocation sized from the header
    const std::streampos body_pos = f.tellg();
    f.seekg(0, std::ios::end);
    const std::streampos end_pos = f.tellg();
    f.seekg(body_pos);
    const size_t remaining = (body_pos >= 0 && end_pos >= body_pos) ? size_t(end_pos - body_pos) : 0;
    if (data_mode == "binary" && points * rec > remaining) { std::cerr << "Error reading PCD file: " << file_path << " (truncated)" << std::endl; return false; }
    if (data_mode == "ascii" && points > remaining) { std::cerr << "Error reading PCD file: " << file_path << " (truncated)" << std::endl; return false; }
    int ix = -1, iy = -1, iz = -1, ii = -1;
    for (size_t k = 0; k < fields.size(); ++k) {
        if (fields[k].name == "x") ix = int(k); else if (fields[k].name == "y") iy = int(k); else if (fields[k].name == "z") iz = int(k);
        else if (fields[k].name == "intensity") ii = int(k);
    }
    if (ix < 0 || iy < 0 || iz < 0) { std::cerr << "Error reading PCD file: " << file_path << " (no x/y/z fields)" << std::endl; return false; }
    cloud_out->points.clear();
    try { cloud_out->points.resize(points); }
    catch (const std::exception&) { std::cerr << "Error reading PCD file: " << file_path << " (out of memory)" << std::endl; cloud_out->points.clear(); return false; }
    auto set = [&](size_t i, double x, double y, double z, double it) {
        PointT p{};
        p.x = float(x); p.y = float(y); p.z = float(z); p.intensity = float(it);
        cloud_out->points[i] = p;
    };
    if (data_mode == "ascii") {
        for (size_t i = 0; i < points; ++i) {
            if (!std::getline(f, line)) { std::cerr << "Error reading PCD file: " << file_path << " (truncated)" << std::endl; return false; }
            std::istringstream ls(line);
            double v[4] = {0, 0, 0, 0};
            for (size_t k = 0; k < fields.size(); ++k)
                for (int c = 0; c < fields[k].count; ++c) {
                    std::string tok;
                    if (!(ls >> tok)) { std::cerr << "Error reading PCD file: " << file_path << " (short row)" << std::endl; return false; }
                    if (c != 0) continue;
                    double val;
                    if (tok == "nan" || tok == "NaN" || tok == "-nan") val = std::nan("");
                    else { try { val = std::stod(tok); } catch (...) { std::cerr << "Error reading PCD file: " << file_path << " (bad number)" << std::endl; return false; } }
                    if (int(k) == ix) v[0] = val; else if (int(k) == iy) v[1] = val; else if (int(k) == iz) v[2] = val; else if (int(k) == ii) v[3] = val;
                }
            set(i, v[0], v[1], v[2], v[3]);
        }
        return true;
    }
    std::vector<unsigned char> raw;
    const bool soa = data_mode == "binary_compressed";
    if (data_mode == "binary") {
        raw.resize(points * rec);
        f.read(reinterpret_cast<char*>(raw.data()), std::streamsize(raw.size()));
        if (size_t(f.gcount()) != raw.size()) { std::cerr << "Error reading PCD file: " << file_path << " (truncated)" << std::endl; return false; }
    } else if (soa) {
        uint32_t csize = 0, usize = 0;
        f.read(reinterpret_cast<char*>(&csize), 4);
        f.read(reinterpret_cast<char*>(&usize), 4);
        if (!f.good() || size_t(usize) != points * rec || remaining < 8 || size_t(csize) > remaining - 8) {
            std::cerr << "Error reading PCD file: " << file_path << " (bad compressed header)" << std::endl; return false;
        }
        std::vector<unsigned char> comp(csize);
        f.read(reinterpret_cast<char*>(comp.data()), std::streamsize(csize));
        if (size_t(f.gcount()) != size_t(csize)) { std::cerr << "Error reading PCD file: " << file_path << " (truncated)" << std::endl; return false; }
        raw.resize(usize);
        if (!lzf_decompress(comp.data(), comp.size(), raw.data(), raw.size())) { std::cerr << "Error reading PCD file: " << file_path << " (LZF)" << std::endl; return false; }
    } else { std::cerr << "Error reading PCD file: " << file_path << " (DATA " << data_mode << ")" << std::endl; return false; }
    // binary: records back to back; binary_compressed: field by field (all x, then all y, ...), each field `points` entries of size*count bytes
    std::vector<size_t> soa_base(fields.size(), 0);
    if (soa) { size_t b = 0; for (size_t k = 0; k < fields.size(); ++k) { soa_base[k] = b; b += size_t(fields[k].size) * size_t(fields[k].count) * points; } }
    auto get = [&](int k, size_t i) -> double {
        if (k < 0) return 0.0;
        const Field& fl = fields[size_t(k)];
        const unsigned char* p = soa ? raw.data() + soa_base[size_t(k)] + i * size_t(fl.size) * size_t(fl.count) : raw.data() + i * rec + fl.offset;
        return read_scalar(p, fl.type, fl.size);
    };
    for (size_t i = 0; i < points; ++i) set(i, get(ix, i), get(iy, i), get(iz, i), get(ii, i));
    return true;
}

// Writes `cloud` (anything with .points, a std::vector of a point holding float x, y, z, intensity) to `file_path` as an
// unorganised binary PCD v0.7 file of float fields x y z intensity -- what pcl::io::savePCDFileBinary writes for pcl::PointXYZI, and
// what readPointCloud reads back bit for bit (non-finite points included).  With LocalMap::getWholeMap it saves a session's map as
// the next session's prior map.  true / false + a message on stderr, never throws.
template <class Cloud>
inline bool writePointCloud(const std::string& file_path, const Cloud& cloud) {
    std::ofstream f(file_path.c_str(), std::ios::binary | std::ios::trunc);
    if (!f.good()) { std::cerr << "Error: cannot open for writing: " << file_path << std::endl; return false; }
    const size_t n = cloud.points.size();
    f << "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
      << "WIDTH " << n << "\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS " << n << "\nDATA binary\n";
    std::vector<float> rec(4 * n);
    for (size_t i = 0; i < n; ++i) {
        const auto& p = cloud.points[i];
        rec[4 * i] = p.x; rec[4 * i + 1] = p.y; rec[4 * i + 2] = p.z; rec[4 * i + 3] = p.intensity;
    }
    f.write(reinterpret_cast<const char*>(rec.data()), std::streamsize(rec.size() * sizeof(float)));
    if (!f.good()) { std::cerr << "Error writing PCD file: " << file_path << std::endl; return false; }
    return true;
}

}  // namespace b200
}  // namespace super_odometry
